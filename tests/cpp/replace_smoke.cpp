// cudf/replace.hpp through the cudf:: C++ surface (over the C ABI): replace_nans with a column and a scalar, the in-place
// normalize_nans_and_zeros on a mutable_column_view, both fill policies, clamp and find_and_replace_all, with the reference's
// exception types.
#include <cudf/replace.hpp>
#include <cudf/types.hpp>

#include <cuda_runtime_api.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <vector>

template <typename T>
struct dev_vec {
  T* p = nullptr;
  size_t n;
  explicit dev_vec(std::vector<T> const& h) : n(h.size()) { cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T) + 64); cudaMemcpy(p, h.data(), n * sizeof(T), cudaMemcpyHostToDevice); }
  ~dev_vec() { cudaFree(p); }
};
template <typename T>
std::vector<T> to_host(cudf::column_view const& v)
{
  std::vector<T> h(v.size());
  cudaDeviceSynchronize();
  if (!h.empty()) cudaMemcpy(h.data(), v.data<T>(), h.size() * sizeof(T), cudaMemcpyDeviceToHost);
  return h;
}
uint32_t mask_word(cudf::column_view const& v)
{
  uint32_t w = 0;
  cudaDeviceSynchronize();
  cudaMemcpy(&w, v.null_mask(), 4, cudaMemcpyDeviceToHost);
  return w;
}
uint64_t bits(double x)
{
  uint64_t u;
  std::memcpy(&u, &x, 8);
  return u;
}
#define EXPECT(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main()
{
  using namespace cudf;
  double const nan = std::numeric_limits<double>::quiet_NaN();
  // replace_nans with a column: a NaN row takes the replacement's value and validity
  dev_vec<double> x({1.0, nan, 3.0, nan, 5.0}), r({10, 20, 30, 40, 50});
  dev_vec<uint32_t> rmask({0b11101u});  // row 1 of the replacement is null
  column_view xv{data_type{type_id::FLOAT64}, 5, x.p};
  column_view rv{data_type{type_id::FLOAT64}, 5, r.p, rmask.p, 1};
  auto a = replace_nans(xv, rv);
  EXPECT(a->null_count() == 1);
  EXPECT(mask_word(a->view()) == 0b11101u);
  auto ah = to_host<double>(a->view());
  EXPECT(ah[0] == 1.0 && ah[2] == 3.0 && ah[3] == 40.0 && ah[4] == 5.0);
  // replace_nans with a scalar: the output always has a mask
  numeric_scalar<double> s(-1.0);
  auto b = replace_nans(xv, s);
  EXPECT(b->null_count() == 0 && b->view().nullable());
  EXPECT((to_host<double>(b->view()) == std::vector<double>{1.0, -1.0, 3.0, -1.0, 5.0}));
  // a non-float input and a type mismatch are logic_error
  dev_vec<int32_t> k({5, 1, 7, 2});
  column_view kv{data_type{type_id::INT32}, 4, k.p};
  bool threw = false;
  try { replace_nans(kv, s); } catch (cudf::logic_error const&) { threw = true; }
  EXPECT(threw);

  // normalize_nans_and_zeros in place on a mutable_column_view: -NaN and -0.0 become quiet NaN and +0.0, bit for bit
  dev_vec<double> z({-0.0, -nan, 2.0, 0.0});
  mutable_column_view zv{data_type{type_id::FLOAT64}, 4, z.p};
  normalize_nans_and_zeros(zv);
  auto zh = to_host<double>(zv);
  EXPECT(bits(zh[0]) == bits(0.0) && bits(zh[1]) == bits(nan) && zh[2] == 2.0 && bits(zh[3]) == bits(0.0));
  // the reference's idiom on an owned column: `cudf::mutable_column_view v = col;` (a no-null replace_nulls is a copy)
  dev_vec<double> w({-0.0, -nan, 7.0});
  auto owned = replace_nulls(column_view{data_type{type_id::FLOAT64}, 3, w.p}, s);
  cudf::mutable_column_view ov = *owned;
  normalize_nans_and_zeros(ov);
  auto wh = to_host<double>(owned->view());
  EXPECT(bits(wh[0]) == bits(0.0) && bits(wh[1]) == bits(nan) && wh[2] == 7.0);
  auto zc = normalize_nans_and_zeros(column_view{data_type{type_id::FLOAT64}, 4, z.p});
  EXPECT(bits(to_host<double>(zc->view())[1]) == bits(nan));

  // replace_nulls: PRECEDING / FOLLOWING (replace_nulls_tests.cpp's policy answers), a leading / trailing run stays null
  dev_vec<int32_t> p({1, 2, 3, 4, 5, 6});
  dev_vec<uint32_t> pm({0b011010u});  // valid rows 1, 3, 4
  column_view pv{data_type{type_id::INT32}, 6, p.p, pm.p, 3};
  auto pre = replace_nulls(pv, replace_policy::PRECEDING);
  EXPECT(pre->null_count() == 1 && mask_word(pre->view()) == 0b111110u);
  auto ph = to_host<int32_t>(pre->view());
  EXPECT(ph[1] == 2 && ph[2] == 2 && ph[3] == 4 && ph[4] == 5 && ph[5] == 5);
  auto fol = replace_nulls(pv, replace_policy::FOLLOWING);
  EXPECT(fol->null_count() == 1 && mask_word(fol->view()) == 0b011111u);
  auto fh = to_host<int32_t>(fol->view());
  EXPECT(fh[0] == 2 && fh[1] == 2 && fh[2] == 4 && fh[3] == 4 && fh[4] == 5);

  // clamp (lo / hi as their own replacements) and find_and_replace_all (first duplicate wins)
  numeric_scalar<int32_t> lo(2), hi(6);
  EXPECT((to_host<int32_t>(clamp(kv, lo, hi)->view()) == std::vector<int32_t>{5, 2, 6, 2}));
  dev_vec<int32_t> old({7, 1, 7}), neu({70, 10, 71});
  auto f = find_and_replace_all(kv, column_view{data_type{type_id::INT32}, 3, old.p}, column_view{data_type{type_id::INT32}, 3, neu.p});
  EXPECT((to_host<int32_t>(f->view()) == std::vector<int32_t>{5, 10, 70, 2}));
  numeric_scalar<int64_t> wide(1);
  threw = false;
  try { clamp(kv, wide, wide); } catch (cudf::data_type_error const&) { threw = true; }
  EXPECT(threw);
  std::printf("REPLACE_CPP_OK\n");
  return 0;
}

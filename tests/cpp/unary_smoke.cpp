// Known answers of cpp/tests/unary/math_ops_test.cpp, unary_ops_test.cpp and cast_tests.cpp (reference tree) through the cudf::
// C++ surface (include/cudf/unary.hpp over the C ABI).
#include <cudf/unary.hpp>
#include <cudf/types.hpp>

#include <cuda_runtime_api.h>

#include <cmath>
#include <cstdio>
#include <limits>
#include <stdexcept>
#include <vector>

template <typename T>
struct dev_vec {
  T* p = nullptr;
  size_t n;
  explicit dev_vec(std::vector<T> const& h) : n(h.size()) { cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T) + 64); cudaMemcpy(p, h.data(), n * sizeof(T), cudaMemcpyHostToDevice); }
  ~dev_vec() { cudaFree(p); }
};
template <typename T>
std::vector<T> to_host(cudf::column const& c)
{
  b2_column_view v = c.view().native();
  std::vector<T> h(v.size);
  cudaDeviceSynchronize();
  if (!h.empty()) cudaMemcpy(h.data(), v.data, h.size() * sizeof(T), cudaMemcpyDeviceToHost);
  return h;
}
#define EXPECT(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main()
{
  using namespace cudf;
  // SimpleNEGATE (math_ops_test.cpp:37)
  dev_vec<int32_t> a({0, 1, 2, 3});
  column_view av{data_type{type_id::INT32}, 4, a.p};
  EXPECT((to_host<int32_t>(*unary_operation(av, unary_operator::NEGATE)) == std::vector<int32_t>{0, -1, -2, -3}));
  // SimpleSQRT (:276) and SimpleRINT (:458)
  dev_vec<double> s({1, 4, 9, 16}), r({1.5, 3.5, -1.5, -3.5});
  column_view sv{data_type{type_id::FLOAT64}, 4, s.p}, rv{data_type{type_id::FLOAT64}, 4, r.p};
  EXPECT((to_host<double>(*unary_operation(sv, unary_operator::SQRT)) == std::vector<double>{1, 2, 3, 4}));
  EXPECT((to_host<double>(*unary_operation(rv, unary_operator::RINT)) == std::vector<double>{2, 4, -2, -4}));
  // BitCount (:105): 0 .. 3 -> 0, 1, 1, 2 in INT32
  auto bc = unary_operation(column_view{data_type{type_id::INT32}, 4, a.p}, unary_operator::BIT_COUNT);
  EXPECT(bc->view().type().id() == type_id::INT32);
  EXPECT((to_host<int32_t>(*bc) == std::vector<int32_t>{0, 1, 1, 2}));
  // RINTNonFloatingFail and NegateUnsupportedTypesFail
  dev_vec<uint32_t> u({1, 2, 3});
  column_view uv{data_type{type_id::UINT32}, 3, u.p};
  try { (void)unary_operation(av, unary_operator::RINT); EXPECT(false); } catch (cudf::logic_error const&) {}
  try { (void)unary_operation(uv, unary_operator::NEGATE); EXPECT(false); } catch (cudf::logic_error const&) {}
  // IsNull WithInvalids (unary_ops_test.cpp:69): rows 1 and 3 null
  uint32_t const mask_host = 0b0101u;
  dev_vec<uint32_t> mask({mask_host, 0u});
  column_view nv{data_type{type_id::INT32}, 4, a.p, mask.p, 2};
  EXPECT((to_host<uint8_t>(*is_null(nv)) == std::vector<uint8_t>{0, 1, 0, 1}));
  EXPECT((to_host<uint8_t>(*is_valid(nv)) == std::vector<uint8_t>{1, 0, 1, 0}));
  // IsNAN WithNull (:167)
  dev_vec<float> f({1.0f, NAN, NAN, 4.0f});
  column_view fv{data_type{type_id::FLOAT32}, 4, f.p, mask.p, 2};
  EXPECT((to_host<uint8_t>(*is_nan(fv)) == std::vector<uint8_t>{0, 0, 1, 0}));
  EXPECT((to_host<uint8_t>(*is_not_nan(fv)) == std::vector<uint8_t>{1, 1, 0, 1}));
  try { (void)is_nan(av); EXPECT(false); } catch (cudf::logic_error const&) {}
  // DownCastingFloorsValues (cast_tests.cpp:315): milliseconds before the epoch floor to seconds and days
  dev_vec<int64_t> ms({-131968727238LL, 1530705600000LL, 1674631932929LL});
  column_view msv{data_type{type_id::TIMESTAMP_MILLISECONDS}, 3, ms.p};
  EXPECT((to_host<int64_t>(*cast(msv, data_type{type_id::TIMESTAMP_SECONDS})) ==
          std::vector<int64_t>{-131968728LL, 1530705600LL, 1674631932LL}));
  EXPECT((to_host<int32_t>(*cast(msv, data_type{type_id::TIMESTAMP_DAYS})) == std::vector<int32_t>{-1528, 17716, 19382}));
  try { (void)cast(msv, data_type{type_id::INT64}); EXPECT(false); } catch (cudf::logic_error const&) {}
  try { (void)cast(av, data_type{type_id::DECIMAL64}); EXPECT(false); } catch (cudf::data_type_error const&) {}
  EXPECT((to_host<double>(*cast(av, data_type{type_id::FLOAT64})) == std::vector<double>{0, 1, 2, 3}));
  EXPECT(is_supported_cast(data_type{type_id::INT32}, data_type{type_id::DURATION_DAYS}));
  EXPECT(!is_supported_cast(data_type{type_id::INT32}, data_type{type_id::TIMESTAMP_DAYS}));
  EXPECT(!is_supported_cast(data_type{type_id::DECIMAL32}, data_type{type_id::INT32}));
  EXPECT(!is_supported_cast(data_type{type_id::NUM_TYPE_IDS}, data_type{type_id::INT32}));  // noexcept: false, not a throw
  // bit_cast: a view of the same bits; different widths are not bit-castable
  EXPECT(is_bit_castable(data_type{type_id::INT32}, data_type{type_id::FLOAT32}));
  EXPECT(!is_bit_castable(data_type{type_id::INT32}, data_type{type_id::INT64}));
  column_view bv = bit_cast(av, data_type{type_id::UINT32});
  EXPECT(bv.type().id() == type_id::UINT32 && bv.head<void>() == av.head<void>());
  try { (void)bit_cast(av, data_type{type_id::INT64}); EXPECT(false); } catch (cudf::logic_error const&) {}
  std::printf("UNARY_CPP_OK\n");
  return 0;
}

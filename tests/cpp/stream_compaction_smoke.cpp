// Known answers of cpp/tests/stream_compaction/*_tests.cpp (reference tree) through the cudf:: C++ surface
// (include/cudf/stream_compaction.hpp over the C ABI).
#include <cudf/stream_compaction.hpp>
#include <cudf/types.hpp>

#include <cuda_runtime_api.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
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
  auto v = c.view();
  std::vector<T> h(static_cast<size_t>(v.size()));
  cudaDeviceSynchronize();
  if (!h.empty()) cudaMemcpy(h.data(), v.data<T>(), h.size() * sizeof(T), cudaMemcpyDeviceToHost);
  return h;
}
#define EXPECT(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main()
{
  using namespace cudf;
  // apply_boolean_mask_tests.cpp:36-52 (col2 only): {10, 40, 70, 5, 2, 10} with {T, F, T, F, T, F} -> {10, 70, 2}
  dev_vec<int32_t> c2({10, 40, 70, 5, 2, 10});
  dev_vec<uint8_t> m({1, 0, 1, 0, 1, 0});
  column_view c2v{data_type{type_id::INT32}, 6, c2.p}, mv{data_type{type_id::BOOL8}, 6, m.p};
  auto kept = apply_boolean_mask(table_view{{c2v}}, mv);
  EXPECT((to_host<int32_t>(kept->get_column(0)) == std::vector<int32_t>{10, 70, 2}));
  auto del = apply_deletion_mask(table_view{{c2v}}, mv);
  EXPECT((to_host<int32_t>(del->get_column(0)) == std::vector<int32_t>{40, 5, 10}));
  try { apply_boolean_mask(table_view{{c2v}}, c2v); EXPECT(false); } catch (cudf::logic_error const&) {}

  // drop_nulls_tests.cpp:21-43 (col1): validity {1, 1, 0, 1, 1, 0} on key 0 -> rows 0, 1, 3, 4
  dev_vec<uint32_t> valid({0b011011u});
  column_view c2n{data_type{type_id::INT32}, 6, c2.p, valid.p, 2};
  EXPECT((to_host<int32_t>(drop_nulls(table_view{{c2n}}, {0})->get_column(0)) == std::vector<int32_t>{10, 40, 5, 2}));
  EXPECT(drop_nulls(table_view{{c2n, c2v}}, {0, 1}, 1)->num_rows() == 6);

  // drop_nans: a NaN key drops the row, a null one does not
  dev_vec<double> f({1.0, NAN, 3.0, NAN});
  dev_vec<uint32_t> fvalid({0b0111u});
  column_view fv{data_type{type_id::FLOAT64}, 4, f.p, fvalid.p, 1};
  EXPECT((to_host<double>(drop_nans(table_view{{fv}}, {0})->get_column(0)).size() == 3));
  try { drop_nans(table_view{{c2v}}, {0}); EXPECT(false); } catch (cudf::logic_error const&) {}

  // unique / distinct / stable_distinct / distinct_indices on {5, 4, 4, 5, 5, 8}
  dev_vec<int64_t> k({5, 4, 4, 5, 5, 8});
  column_view kv{data_type{type_id::INT64}, 6, k.p};
  EXPECT((to_host<int64_t>(unique(table_view{{kv}}, {0}, duplicate_keep_option::KEEP_FIRST)->get_column(0)) ==
          std::vector<int64_t>{5, 4, 5, 8}));
  EXPECT((to_host<int64_t>(stable_distinct(table_view{{kv}}, {0})->get_column(0)) == std::vector<int64_t>{5, 4, 8}));
  auto d = to_host<int64_t>(distinct(table_view{{kv}}, {0}, duplicate_keep_option::KEEP_NONE)->get_column(0));
  EXPECT((d == std::vector<int64_t>{8}));
  auto idx = distinct_indices(table_view{{kv}}, duplicate_keep_option::KEEP_LAST, null_equality::EQUAL, nan_equality::UNEQUAL);
  EXPECT((to_host<int32_t>(*idx) == std::vector<int32_t>{2, 4, 5}));
  try { distinct(table_view{{kv}}, {3}); EXPECT(false); } catch (std::out_of_range const&) {}
  std::printf("STREAM_COMPACTION_CPP_OK\n");
  return 0;
}

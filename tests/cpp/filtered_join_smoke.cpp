// Known answers of cpp/tests/join/semi_anti_join_tests.cpp and the examples of cpp/include/cudf/join/filtered_join.hpp
// (reference tree) through the cudf:: C++ surface (include/cudf/join/filtered_join.hpp over the C ABI).
#include <cudf/join/filtered_join.hpp>
#include <cudf/types.hpp>

#include <cuda_runtime_api.h>

#include <cstdio>
#include <stdexcept>
#include <vector>

template <typename T>
struct dev_vec {
  T* p = nullptr;
  size_t n;
  explicit dev_vec(std::vector<T> const& h) : n(h.size()) { cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T) + 64); cudaMemcpy(p, h.data(), n * sizeof(T), cudaMemcpyHostToDevice); }
  ~dev_vec() { cudaFree(p); }
};
std::vector<int32_t> to_host(rmm::device_uvector<cudf::size_type> const& v)
{
  std::vector<int32_t> h(v.size());
  cudaDeviceSynchronize();
  if (!h.empty()) cudaMemcpy(h.data(), v.data(), h.size() * sizeof(int32_t), cudaMemcpyDeviceToHost);
  return h;
}
#define EXPECT(c) do { if (!(c)) { std::printf("FAILED: %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main()
{
  using namespace cudf;
  auto stream = cudf::get_default_stream();
  // filtered_join.hpp:107-111,132-136: right (filter) {1, 2, 3}, left {0, 1, 2} -> semi {1, 2}, anti {0}
  dev_vec<int32_t> r({1, 2, 3}), l({0, 1, 2});
  column_view rv{data_type{type_id::INT32}, 3, r.p}, lv{data_type{type_id::INT32}, 3, l.p};
  filtered_join fj(table_view{{rv}}, null_equality::EQUAL, stream);
  EXPECT((to_host(*fj.semi_join(table_view{{lv}})) == std::vector<int32_t>{1, 2}));
  EXPECT((to_host(*fj.anti_join(table_view{{lv}})) == std::vector<int32_t>{0}));

  // PrefilterNullableColumnsNullsEqual (:456-487): left {1, N, 3, 4, N}, right {N, 3, 5, 6}
  dev_vec<int32_t> l2({1, 2, 3, 4, 5}), r2({2, 3, 5, 6});
  dev_vec<uint32_t> l2v({0b01101u}), r2v({0b1110u});
  column_view l2c{data_type{type_id::INT32}, 5, l2.p, l2v.p, 2}, r2c{data_type{type_id::INT32}, 4, r2.p, r2v.p, 1};
  filtered_join eq(table_view{{r2c}}, null_equality::EQUAL, 0.5, stream);
  EXPECT((to_host(*eq.semi_join(table_view{{l2c}})) == std::vector<int32_t>{1, 2, 4}));
  EXPECT((to_host(*eq.anti_join(table_view{{l2c}})) == std::vector<int32_t>{0, 3}));
  filtered_join ne(table_view{{r2c}}, null_equality::UNEQUAL, 1.0, stream);
  EXPECT((to_host(*ne.semi_join(table_view{{l2c}})) == std::vector<int32_t>{2}));
  EXPECT((to_host(*ne.anti_join(table_view{{l2c}})) == std::vector<int32_t>{0, 1, 3, 4}));

  // InvalidLoadFactor (:520-532)
  for (double lf : {-0.1, 0.0, 1.1}) {
    try { filtered_join bad(table_view{{rv}}, null_equality::EQUAL, lf, stream); EXPECT(false); } catch (std::invalid_argument const&) {}
  }
  // a key type differing from the right table's
  dev_vec<int64_t> w({0, 1, 2});
  column_view wv{data_type{type_id::INT64}, 3, w.p};
  try { (void)fj.semi_join(table_view{{wv}}); EXPECT(false); } catch (std::invalid_argument const&) {}
  std::printf("FILTERED_JOIN_CPP_OK\n");
  return 0;
}

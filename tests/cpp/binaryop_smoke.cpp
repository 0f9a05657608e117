// Known answers of cpp/tests/binaryop/binop-compiled-test.cpp, binop-null-test.cpp and binop-verify-input-test.cpp (reference
// tree) through the cudf:: C++ surface (include/cudf/binaryop.hpp over the C ABI).
#include <cudf/binaryop.hpp>
#include <cudf/types.hpp>

#include <cuda_runtime_api.h>

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
  // IntPow_SpecialCases (binop-compiled-test.cpp:390-407)
  dev_vec<int64_t> l({3, -3, 8, -8}), r({1, 1, 7, 7});
  column_view lv{data_type{type_id::INT64}, 4, l.p}, rv{data_type{type_id::INT64}, 4, r.p};
  auto p = binary_operation(lv, rv, binary_operator::INT_POW, data_type{type_id::INT64});
  EXPECT((to_host<int64_t>(*p) == std::vector<int64_t>{3, -3, 2097152, -2097152}));
  // FloorDivInt64RoundNegativeInf (:432-453)
  constexpr int64_t lo = std::numeric_limits<int64_t>::min();
  dev_vec<int64_t> fl({lo, lo + 10, lo + 100}), ten({10, 10, 10});
  column_view flv{data_type{type_id::INT64}, 3, fl.p}, tenv{data_type{type_id::INT64}, 3, ten.p};
  auto fd = binary_operation(flv, tenv, binary_operator::FLOOR_DIV, data_type{type_id::INT64});
  EXPECT((to_host<int64_t>(*fd) == std::vector<int64_t>{lo / 10 - 1, (lo + 10) / 10 - 1, (lo + 100) / 10 - 1}));
  // Scalar_Null_Vector_Valid (binop-null-test.cpp:32-45): every row null
  dev_vec<int32_t> seq({0, 1, 2, 3, 4, 5, 6, 7, 8, 9});
  column_view sv{data_type{type_id::INT32}, 10, seq.p};
  numeric_scalar<int32_t> null_s(0, false), one(1);
  EXPECT(binary_operation(null_s, sv, binary_operator::ADD, data_type{type_id::INT32})->view().native().null_count == 10);
  EXPECT((to_host<int32_t>(*binary_operation(sv, one, binary_operator::ADD, data_type{type_id::INT32})) ==
          std::vector<int32_t>{1, 2, 3, 4, 5, 6, 7, 8, 9, 10}));
  // comparison against a scalar writes BOOL8
  auto gt = binary_operation(sv, numeric_scalar<int32_t>(4), binary_operator::GREATER, data_type{type_id::BOOL8});
  EXPECT((to_host<uint8_t>(*gt) == std::vector<uint8_t>{0, 0, 0, 0, 0, 1, 1, 1, 1, 1}));
  EXPECT(binops::is_supported_operation(data_type{type_id::FLOAT64}, data_type{type_id::INT32}, data_type{type_id::INT32},
                                        binary_operator::BITWISE_AND));
  EXPECT(!binops::is_supported_operation(data_type{type_id::FLOAT64}, data_type{type_id::FLOAT64}, data_type{type_id::FLOAT64},
                                         binary_operator::BITWISE_AND));
  // binop-verify-input-test.cpp: an output type id outside type_id, differing column sizes; and an unsupported combination
  numeric_scalar<int64_t> s64(1);
  try { (void)binary_operation(s64, lv, binary_operator::ADD, data_type{type_id::NUM_TYPE_IDS}); EXPECT(false); } catch (cudf::logic_error const&) {}
  try { (void)binary_operation(lv, tenv, binary_operator::ADD, data_type{type_id::INT64}); EXPECT(false); } catch (std::invalid_argument const&) {}
  try { (void)binary_operation(lv, rv, binary_operator::GREATER, data_type{type_id::INT64}); EXPECT(false); } catch (cudf::data_type_error const&) {}
  std::printf("BINARYOP_CPP_OK\n");
  return 0;
}

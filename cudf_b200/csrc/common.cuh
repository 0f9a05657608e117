// common.cuh — shared host/device plumbing of the H100-native hot path.
// Error taxonomy follows cpp/include/cudf/utilities/error.hpp:35-118 of the reference; the data model
// follows column_view.hpp:237-244 / column.hpp:36-334 (see include/cudf_b200.h).
#pragma once

#include "../../include/cudf_b200.h"

#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

namespace b2 {

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
struct error : std::exception {
  b2_status code;
  std::string msg;
  error(b2_status c, std::string m) : code(c), msg(std::move(m)) {}
  const char* what() const noexcept override { return msg.c_str(); }
};

#define B2_STR2(x) #x
#define B2_STR(x) B2_STR2(x)
#define B2_EXPECTS(cond, code, message)                                                    \
  do {                                                                                     \
    if (!(cond)) throw ::b2::error((code), std::string(message) + " [" __FILE__ ":" B2_STR(__LINE__) "]"); \
  } while (0)
#define B2_FAIL(code, message) throw ::b2::error((code), std::string(message) + " [" __FILE__ ":" B2_STR(__LINE__) "]")
#define B2_CUDA_TRY(call)                                                                  \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      cudaGetLastError();                                                                  \
      throw ::b2::error(e__ == cudaErrorMemoryAllocation ? B2_ERR_BAD_ALLOC : B2_ERR_CUDA, \
                        std::string("CUDA error ") + cudaGetErrorName(e__) + ": " +        \
                          cudaGetErrorString(e__) + " at " __FILE__ ":" B2_STR(__LINE__)); \
    }                                                                                      \
  } while (0)

void set_last_error(const char* msg);

// NVTX range over every C-ABI entry point (role of CUDF_FUNC_RANGE, cpp/include/cudf/detail/nvtx/ranges.hpp:50): header-only
// NVTX v3, a no-op unless a profiler is attached.
#ifndef B2_EMU
}  // namespace b2
#include <nvtx3/nvToolsExt.h>
namespace b2 {
struct nvtx_range {
  explicit nvtx_range(const char* name) { nvtxRangePushA(name); }
  ~nvtx_range() { nvtxRangePop(); }
};
#else
struct nvtx_range {
  explicit nvtx_range(const char*) {}
};
#endif

// One-time per-device setup (function attributes, pool / limit settings): `done` is a bit mask over device ordinals.
template <typename F>
inline void once_per_device(std::atomic<uint64_t>& done, F&& f)
{
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return;
  const uint64_t bit = 1ull << (dev & 63);
  if (done.load(std::memory_order_acquire) & bit) return;
  f();
  done.fetch_or(bit, std::memory_order_release);
}

// The extern "C" boundary: every entry point body sits between these two (status code + thread-local message).
#define B2_TRY_BEGIN try { ::b2::nvtx_range b2_nvtx_range__(__func__);
#define B2_TRY_END                                                                           \
  }                                                                                          \
  catch (const ::b2::error& e) { ::b2::set_last_error(e.what()); return e.code; }            \
  catch (const std::bad_alloc& e) { ::b2::set_last_error(e.what()); return B2_ERR_BAD_ALLOC; } \
  catch (const std::exception& e) { ::b2::set_last_error(e.what()); return B2_ERR_LOGIC; }   \
  return B2_OK;
inline std::vector<uint8_t> vec_u8(const uint8_t* p, int32_t n) { return (p && n > 0) ? std::vector<uint8_t>(p, p + n) : std::vector<uint8_t>{}; }

// every kernel launch goes through this so bench.py can report gpu_launches
extern std::atomic<uint64_t> g_launch_count;
#ifdef B2_EMU  // tests/emu: the kernels run on the CPU emulator (test infrastructure, never part of the product build)
#define B2_LAUNCH(kernel, grid, block, smem, stream, ...)                                               \
  do {                                                                                                  \
    ::emu::launch(#kernel, dim3(grid), dim3(block), (size_t)(smem), [&]() { kernel(__VA_ARGS__); });    \
    ::b2::g_launch_count.fetch_add(1, std::memory_order_relaxed);                                       \
  } while (0)
#define B2_DYNAMIC_SMEM(name) unsigned char* name = ::emu::dynamic_smem()
#else
#define B2_LAUNCH(kernel, grid, block, smem, stream, ...)                \
  do {                                                                   \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);          \
    ::b2::g_launch_count.fetch_add(1, std::memory_order_relaxed);        \
    B2_CUDA_TRY(cudaGetLastError());                                     \
  } while (0)
#define B2_DYNAMIC_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

// optional event timing of a kernel family (see b2_profile_* in the C ABI)
extern std::atomic<int> g_profile_on;
struct prof_scope {
  const char* name;
  cudaStream_t s;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  prof_scope(const char* n, cudaStream_t stream);
  ~prof_scope();
};

// ---------------------------------------------------------------------------------------------
// device memory: stream-ordered pool (cudaMallocAsync) — stands in for rmm::device_buffer / mr
// ---------------------------------------------------------------------------------------------
void* dev_alloc(size_t bytes, cudaStream_t stream);
void dev_free(void* p, cudaStream_t stream) noexcept;

struct dbuf {  // RAII device buffer
  void* ptr      = nullptr;
  size_t bytes   = 0;
  cudaStream_t s = nullptr;
  dbuf() = default;
  dbuf(size_t n, cudaStream_t stream) : ptr(n ? dev_alloc(n, stream) : nullptr), bytes(n), s(stream) {}
  dbuf(dbuf&& o) noexcept : ptr(o.ptr), bytes(o.bytes), s(o.s) { o.ptr = nullptr; o.bytes = 0; }
  dbuf& operator=(dbuf&& o) noexcept
  {
    if (this != &o) { reset(); ptr = o.ptr; bytes = o.bytes; s = o.s; o.ptr = nullptr; o.bytes = 0; }
    return *this;
  }
  dbuf(const dbuf&)            = delete;
  dbuf& operator=(const dbuf&) = delete;
  ~dbuf() { reset(); }
  void reset() noexcept
  {
    if (ptr) dev_free(ptr, s);
    ptr = nullptr; bytes = 0;
  }
  void* release() noexcept { void* p = ptr; ptr = nullptr; bytes = 0; return p; }
  template <typename T> T* as() const { return static_cast<T*>(ptr); }
};

// ---------------------------------------------------------------------------------------------
// type helpers
// ---------------------------------------------------------------------------------------------
inline int type_width(int32_t id)
{
  switch (id) {
    case B2_INT8: case B2_UINT8: case B2_BOOL8: return 1;
    case B2_INT16: case B2_UINT16: return 2;
    case B2_INT32: case B2_UINT32: case B2_FLOAT32: case B2_TIMESTAMP_DAYS: case B2_DURATION_DAYS: return 4;
    case B2_INT64: case B2_UINT64: case B2_FLOAT64:
    case B2_TIMESTAMP_SECONDS: case B2_TIMESTAMP_MILLISECONDS: case B2_TIMESTAMP_MICROSECONDS:
    case B2_TIMESTAMP_NANOSECONDS: case B2_DURATION_SECONDS: case B2_DURATION_MILLISECONDS:
    case B2_DURATION_MICROSECONDS: case B2_DURATION_NANOSECONDS: return 8;
    default: return 0;
  }
}
inline bool is_fixed_width(int32_t id) { return type_width(id) != 0; }
// f(T{}) with the unsigned integer type of `width` bytes (the kernels move fixed-width values as plain bits)
template <typename F>
inline void dispatch_width(int width, F&& f)
{
  switch (width) {
    case 1: f(uint8_t{}); break;
    case 2: f(uint16_t{}); break;
    case 4: f(uint32_t{}); break;
    case 8: f(uint64_t{}); break;
    default: throw ::b2::error(B2_ERR_DATA_TYPE, "unsupported (non fixed-width) column type");
  }
}
// storage type of chrono ids (dispatch_storage_type): timestamps/durations are signed ints
inline int32_t storage_type(int32_t id)
{
  switch (id) {
    case B2_TIMESTAMP_DAYS: case B2_DURATION_DAYS: return B2_INT32;
    case B2_TIMESTAMP_SECONDS: case B2_TIMESTAMP_MILLISECONDS: case B2_TIMESTAMP_MICROSECONDS:
    case B2_TIMESTAMP_NANOSECONDS: case B2_DURATION_SECONDS: case B2_DURATION_MILLISECONDS:
    case B2_DURATION_MICROSECONDS: case B2_DURATION_NANOSECONDS: return B2_INT64;
    default: return id;
  }
}
inline bool is_numeric(int32_t id) { return id >= B2_INT8 && id <= B2_BOOL8; }
inline bool is_integral_id(int32_t id) { return (id >= B2_INT8 && id <= B2_UINT64) || id == B2_BOOL8; }
inline bool is_float_id(int32_t id) { return id == B2_FLOAT32 || id == B2_FLOAT64; }
inline bool is_signed_id(int32_t id) { return id >= B2_INT8 && id <= B2_INT64; }

inline size_t bitmask_bytes(int64_t bits) { return ((size_t)((bits + 31) / 32) * 4 + 63) / 64 * 64; }
inline int64_t num_words(int64_t bits) { return (bits + 31) / 32; }

inline bool has_nulls(const b2_column_view& c) { return c.null_mask != nullptr && c.null_count > 0; }

// ---------------------------------------------------------------------------------------------
// owning objects behind the opaque handles
// ---------------------------------------------------------------------------------------------
}  // namespace b2

struct b2_buffer {
  b2::dbuf buf;
};

struct b2_column {
  int32_t type_id    = B2_EMPTY;
  int32_t size       = 0;
  // null_count < 0: still being counted on the device (`pending` holds an unsigned long long that
  // the producing kernel accumulates into); resolved lazily so that producers stay asynchronous.
  mutable int32_t null_count = 0;
  b2::dbuf data;
  b2::dbuf mask;
  mutable b2::dbuf pending;
  cudaStream_t pending_stream = nullptr;
  bool pending_is_valid_count = false;  // pending counts valid rows instead of nulls
  int32_t resolve_null_count() const;
  b2_column_view view() const
  {
    int32_t nc = resolve_null_count();
    return b2_column_view{type_id, size, data.ptr, static_cast<const uint32_t*>(mask.ptr), nc, 0};
  }
};

struct b2_table {
  std::vector<std::unique_ptr<b2_column>> cols;
};

struct b2_scalar {
  int32_t type_id = B2_EMPTY;
  b2::dbuf data;   // 8 bytes value + 4 bytes validity flag (int32) at offset 8
};

namespace b2 {

using column_ptr = std::unique_ptr<b2_column>;
using table_ptr  = std::unique_ptr<b2_table>;

column_ptr make_column(int32_t type_id, int32_t size, bool with_mask, cudaStream_t stream);
void validate_column(const b2_column_view& c);
void validate_table(const b2_table_view* t, std::vector<b2_column_view>& cols);

// ---- implemented in the individual .cu files ------------------------------------------------
// bitmask.cu
int32_t count_set_bits(const uint32_t* mask, int64_t start, int64_t stop, cudaStream_t stream);
void set_null_mask(uint32_t* mask, int64_t begin, int64_t end, bool valid, cudaStream_t stream);
dbuf copy_bitmask(const uint32_t* mask, int64_t begin, int64_t end, cudaStream_t stream);
// AND of nullable columns' masks; returns empty dbuf if none nullable
dbuf bitmask_and(const std::vector<b2_column_view>& cols, int32_t rows, int32_t* null_count, cudaStream_t stream);

// gather.cu
column_ptr gather_column(const b2_column_view& src, const int32_t* map, int32_t n, bool nullify_oob,
                         cudaStream_t stream);
table_ptr gather_table(const std::vector<b2_column_view>& cols, const int32_t* map, int32_t n,
                       bool nullify_oob, cudaStream_t stream);

// radix_sort.cu
column_ptr sorted_order(const std::vector<b2_column_view>& keys, const std::vector<uint8_t>& order,
                        const std::vector<uint8_t>& null_prec, bool stable, cudaStream_t stream);
column_ptr sort_single_column(const b2_column_view& col, bool ascending, cudaStream_t stream);
bool is_radix_sortable(const b2_column_view& c);
bool sort_carry_applicable(const b2_column_view& keys, const b2_column_view& values, bool ascending);
column_ptr sort_by_key_carry(const b2_column_view& keys, const b2_column_view& values, bool ascending, cudaStream_t stream);
void radix_partition_top16_mix(const uint64_t* packed_keys, int64_t n, uint64_t* keys_out, int32_t* idx_out, cudaStream_t stream);

void radix_partition_mix_carry(const uint64_t* keys, const void* vals, int val_bytes, int64_t n, uint64_t* mixed_keys_out, void* vals_out,
                               uint32_t* part_base, cudaStream_t stream);
// histogram-free variant (estimated partition bases; radix_sort.cu)
uint32_t radix_partition_est_capacity(const uint64_t* keys, int64_t n, cudaStream_t stream);
bool radix_partition_mix_carry_est(const uint64_t* keys, const void* vals, int val_bytes, int64_t n, uint32_t cap, uint64_t* mixed_keys_out,
                                   void* vals_out, uint32_t* part_base, uint32_t* part_end, cudaStream_t stream);

void range_partition_counts(const b2_column_view& keys, const void* splitters, int P, int64_t* out_counts, cudaStream_t stream);
void range_partition_scatter(const b2_column_view& keys, const b2_column_view* values, const void* splitters, int P, void* const* key_dst,
                             void* const* val_dst, cudaStream_t stream);

// radix_join.cu (the free-function join when both sides have >= 2^24 null-free rows; B2_JOIN_RADIX_ROWS moves the limit)
bool radix_join_applicable(const std::vector<b2_column_view>& a, const std::vector<b2_column_view>& b);
void radix_join(const std::vector<b2_column_view>& build, const std::vector<b2_column_view>& probe, bool left, cudaStream_t stream,
                column_ptr& out_probe, column_ptr& out_build);
// hash_join.cu: concatenates partial full-join results and appends (JoinNoMatch, r) for every unmatched build row r
void hash_join_finalize_full(const std::vector<b2_column_view>& lparts, const std::vector<b2_column_view>& rparts, int32_t left_rows,
                             int32_t right_rows, cudaStream_t stream, column_ptr& out_left, column_ptr& out_right);

// scan_reduce.cu
std::unique_ptr<b2_scalar> reduce(const b2_column_view& col, int32_t kind, int32_t out_type,
                                  const b2_scalar* init, cudaStream_t stream);
column_ptr segmented_reduce(const b2_column_view& col, const int32_t* offsets, int32_t num_offsets,
                            int32_t kind, int32_t out_type, int32_t null_handling, const b2_scalar* init,
                            cudaStream_t stream);
column_ptr scan(const b2_column_view& col, int32_t kind, int32_t scan_type, int32_t null_handling,
                cudaStream_t stream);
std::unique_ptr<b2_scalar> make_scalar(int32_t type_id, const void* host_value, bool valid, cudaStream_t stream);

}  // namespace b2

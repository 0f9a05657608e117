// scan_reduce.cu — device-wide reduce, decoupled look-back scan and segmented reduce (no cub/thrust).
//
// Replaces, with reference semantics:
//   cudf::reduce            cpp/src/reductions/reductions.cpp:474-536, simple.cuh:47-85 + dispatcher
//                           :373-447 (accumulate in the output type when it equals the input type, else
//                           int64 / double and cast), compound.cuh (MEAN), K22 cub::DeviceReduce
//   cudf::scan              cpp/src/reductions/scan/scan.cpp:13-54, scan_inclusive.cu:36-145,198-240,
//                           scan_exclusive.cu:32-104 (output type == input type, null policies), K24/K25
//   cudf::segmented_reduce  cpp/src/reductions/segmented/reductions.cpp:112-168, simple.cuh:57-104,
//                           validity rule cpp/include/cudf/detail/null_mask.cuh:785-843, K23/K27
#include "common.cuh"
#include "device_utils.cuh"

#include <algorithm>
#include <limits>

namespace b2 {
namespace {

enum { OP_SUM = 0, OP_PRODUCT = 1, OP_MIN = 2, OP_MAX = 3 };

// MIN / MAX order floats with NaN above +inf, whatever its sign (the order of sorted_order): MIN is NaN only when every
// value is NaN, MAX as soon as one is, whatever the order of evaluation. The top of that order, NaN, is MIN's identity;
// where the identity itself is a result (an exclusive scan's empty prefix) scan() writes the reference's +inf instead.
template <typename A, int OP>
struct binop {
  static __host__ __device__ __forceinline__ A identity()
  {
    if constexpr (OP == OP_SUM) return A(0);
    else if constexpr (OP == OP_PRODUCT) return A(1);
    else if constexpr (OP == OP_MIN) {
      if constexpr (std::numeric_limits<A>::has_quiet_NaN) return std::numeric_limits<A>::quiet_NaN();
      else return std::numeric_limits<A>::max();
    } else {
      if constexpr (std::numeric_limits<A>::has_infinity) return -std::numeric_limits<A>::infinity();
      else return std::numeric_limits<A>::lowest();
    }
  }
  static __host__ __device__ __forceinline__ A apply(A a, A b)
  {
    if constexpr (OP == OP_SUM) return a + b;
    else if constexpr (OP == OP_PRODUCT) return a * b;
    else if constexpr (OP == OP_MIN) return (b < a || a != a) ? b : a;  // a != a: a is NaN (false for integers)
    else return (a < b || b != b) ? b : a;
  }
};

template <typename T, typename A>
__device__ __forceinline__ A load_as(const T* p, int64_t i, bool is_bool)
{
  T v = p[i];
  if (is_bool) return A(v != T(0));
  return static_cast<A>(v);
}

template <typename A, int OP>
__device__ __forceinline__ A warp_reduce_op(A v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = binop<A, OP>::apply(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// write accumulator `a` as type `out_type` at dst
template <typename A>
__device__ __forceinline__ void store_as(void* dst, int64_t i, int32_t out_type, A a)
{
  switch (out_type) {
    case B2_INT8: static_cast<int8_t*>(dst)[i] = (int8_t)a; break;
    case B2_INT16: static_cast<int16_t*>(dst)[i] = (int16_t)a; break;
    case B2_INT32: static_cast<int32_t*>(dst)[i] = (int32_t)a; break;
    case B2_INT64: static_cast<int64_t*>(dst)[i] = (int64_t)a; break;
    case B2_UINT8: static_cast<uint8_t*>(dst)[i] = (uint8_t)a; break;
    case B2_UINT16: static_cast<uint16_t*>(dst)[i] = (uint16_t)a; break;
    case B2_UINT32: static_cast<uint32_t*>(dst)[i] = (uint32_t)a; break;
    case B2_UINT64: static_cast<uint64_t*>(dst)[i] = (uint64_t)a; break;
    case B2_FLOAT32: static_cast<float*>(dst)[i] = (float)a; break;
    case B2_FLOAT64: static_cast<double*>(dst)[i] = (double)a; break;
    case B2_BOOL8: static_cast<uint8_t*>(dst)[i] = (a != A(0)) ? 1 : 0; break;
    default: break;
  }
}
template <typename A>
__device__ __forceinline__ A load_scalar_as(const void* src, int32_t type)
{
  switch (type) {
    case B2_INT8: return (A) * static_cast<const int8_t*>(src);
    case B2_INT16: return (A) * static_cast<const int16_t*>(src);
    case B2_INT32: return (A) * static_cast<const int32_t*>(src);
    case B2_INT64: return (A) * static_cast<const int64_t*>(src);
    case B2_UINT8: return (A) * static_cast<const uint8_t*>(src);
    case B2_UINT16: return (A) * static_cast<const uint16_t*>(src);
    case B2_UINT32: return (A) * static_cast<const uint32_t*>(src);
    case B2_UINT64: return (A) * static_cast<const uint64_t*>(src);
    case B2_FLOAT32: return (A) * static_cast<const float*>(src);
    case B2_FLOAT64: return (A) * static_cast<const double*>(src);
    case B2_BOOL8: return (A)(*static_cast<const uint8_t*>(src) != 0);
    default: return A(0);
  }
}

// ------------------------------------------------------------------------------------------------
// reduce
// ------------------------------------------------------------------------------------------------
struct reduce_tail {
  void* partials;           // A[grid]
  unsigned int* ticket;     // zeroed
  void* out_value;          // scalar storage (8 B value + int32 valid at +8)
  int32_t out_type;
  int32_t in_type;
  const void* init_value;   // device scalar storage or null
  int32_t mean;             // divide by valid_count
  int64_t valid_count;
  int32_t is_bool;
};

template <typename T, typename A, int OP, bool NULLS>
__global__ void __launch_bounds__(256) reduce_kernel(const T* __restrict__ data, const uint32_t* __restrict__ mask,
                                                     int64_t bit_offset, int64_t n, reduce_tail t)
{
  using B = binop<A, OP>;
  A acc = B::identity();
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  if constexpr (!NULLS) {
    constexpr int VEC = 16 / sizeof(T);
    const uintptr_t addr = reinterpret_cast<uintptr_t>(data);
    int64_t head = ((16 - (addr & 15)) & 15) / sizeof(T);
    if (head > n) head = n;
    const int64_t nvec = (n - head) / VEC;
    const int4* v4 = reinterpret_cast<const int4*>(data + head);
    for (int64_t v = tid; v < nvec; v += stride) {
      int4 q = ld_nc_v4(v4 + v);
      T tmp[VEC];
      memcpy(tmp, &q, 16);
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc = B::apply(acc, t.is_bool ? A(tmp[j] != T(0)) : static_cast<A>(tmp[j]));
    }
    const int64_t tail_start = head + nvec * VEC;
    const int64_t nscalar = head + (n - tail_start);
    for (int64_t j = tid; j < nscalar; j += stride) {
      int64_t e = j < head ? j : tail_start + (j - head);
      acc = B::apply(acc, load_as<T, A>(data, e, t.is_bool));
    }
  } else {
    for (int64_t i = tid; i < n; i += stride) {
      if (bit_is_set(mask, bit_offset + i)) acc = B::apply(acc, load_as<T, A>(data, i, t.is_bool));
    }
  }
  // block reduce
  __shared__ A sh[8];
  __shared__ bool is_last;
  acc = warp_reduce_op<A, OP>(acc);
  if (lane_id() == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    A b = sh[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) b = B::apply(b, sh[w]);
    static_cast<A*>(t.partials)[blockIdx.x] = b;
    __threadfence();
    unsigned int prev = atomicAdd(t.ticket, 1u);
    is_last = prev == gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x < 32) {
    __threadfence();
    A r = B::identity();
    for (unsigned i = threadIdx.x; i < gridDim.x; i += 32) r = B::apply(r, static_cast<volatile A*>(t.partials)[i]);
    r = warp_reduce_op<A, OP>(r);
    if (threadIdx.x == 0) {
      int32_t valid = 1;
      if (t.init_value) {
        const int32_t iv = *reinterpret_cast<const int32_t*>(static_cast<const char*>(t.init_value) + 8);
        if (iv) r = B::apply(r, load_scalar_as<A>(t.init_value, t.in_type));
        valid = iv != 0;
      }
      if (t.mean) r = r / A(t.valid_count);
      store_as<A>(t.out_value, 0, t.out_type, r);
      *reinterpret_cast<int32_t*>(static_cast<char*>(t.out_value) + 8) = valid;
    }
  }
}

template <typename T, typename A, int OP>
void launch_reduce(const b2_column_view& col, reduce_tail& t, cudaStream_t stream)
{
  const int64_t n = col.size;
  int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 256 * 16 - 1) / (256 * 16), num_sms() * 8));
  dbuf partials(sizeof(A) * grid + 16, stream);
  dbuf ticket(sizeof(unsigned int), stream);
  B2_CUDA_TRY(cudaMemsetAsync(ticket.ptr, 0, sizeof(unsigned int), stream));
  t.partials = partials.ptr;
  t.ticket   = ticket.as<unsigned int>();
  const T* data = static_cast<const T*>(col.data) + col.offset;
  if (has_nulls(col)) {
    B2_LAUNCH((reduce_kernel<T, A, OP, true>), grid, 256, 0, stream, data, col.null_mask, (int64_t)col.offset, n, t);
  } else {
    B2_LAUNCH((reduce_kernel<T, A, OP, false>), grid, 256, 0, stream, data, (const uint32_t*)nullptr, (int64_t)0, n, t);
  }
}

template <typename T, typename A>
void dispatch_reduce_op(int op, const b2_column_view& col, reduce_tail& t, cudaStream_t stream)
{
  switch (op) {
    case OP_SUM: launch_reduce<T, A, OP_SUM>(col, t, stream); break;
    case OP_PRODUCT: launch_reduce<T, A, OP_PRODUCT>(col, t, stream); break;
    case OP_MIN: launch_reduce<T, A, OP_MIN>(col, t, stream); break;
    case OP_MAX: launch_reduce<T, A, OP_MAX>(col, t, stream); break;
  }
}

// unsigned input: accumulate in uint64 when the output is the input type (MIN / MAX need its order), else in int64 as the
// reference does (simple.cuh:407-419): the bits are the same, but a result with bit 63 set converts to a negative float
template <typename T>
void dispatch_reduce_unsigned(bool widen, int op, const b2_column_view& col, reduce_tail& t, cudaStream_t stream)
{
  if (widen) {
    if (op == OP_SUM) launch_reduce<T, int64_t, OP_SUM>(col, t, stream);
    else launch_reduce<T, int64_t, OP_PRODUCT>(col, t, stream);  // MIN / MAX: output type == input type
  } else {
    dispatch_reduce_op<T, uint64_t>(op, col, t, stream);
  }
}

// widen: true -> the output type differs from the input type: integers accumulate in int64, floats in double
void dispatch_reduce(int32_t in_type, bool widen, bool to_float32_acc, int op, const b2_column_view& col, reduce_tail& t,
                     cudaStream_t stream)
{
  switch (in_type) {
    // integer accumulation in 64 bits truncates to the same bits as narrow wrap-around arithmetic
    case B2_INT8: dispatch_reduce_op<int8_t, int64_t>(op, col, t, stream); break;
    case B2_INT16: dispatch_reduce_op<int16_t, int64_t>(op, col, t, stream); break;
    case B2_INT32: dispatch_reduce_op<int32_t, int64_t>(op, col, t, stream); break;
    case B2_INT64: dispatch_reduce_op<int64_t, int64_t>(op, col, t, stream); break;
    case B2_UINT8: case B2_BOOL8: dispatch_reduce_unsigned<uint8_t>(widen, op, col, t, stream); break;
    case B2_UINT16: dispatch_reduce_unsigned<uint16_t>(widen, op, col, t, stream); break;
    case B2_UINT32: dispatch_reduce_unsigned<uint32_t>(widen, op, col, t, stream); break;
    case B2_UINT64: dispatch_reduce_unsigned<uint64_t>(widen, op, col, t, stream); break;
    case B2_FLOAT32:
      if (to_float32_acc) dispatch_reduce_op<float, float>(op, col, t, stream);
      else dispatch_reduce_op<float, double>(op, col, t, stream);
      break;
    case B2_FLOAT64: dispatch_reduce_op<double, double>(op, col, t, stream); break;
    default: B2_FAIL(B2_ERR_DATA_TYPE, "Reduction operator not supported for this type");
  }
}

// MEAN on integer inputs accumulates in the floating result type (compound.cuh): convert on load
template <typename T, typename A>
void mean_launch(const b2_column_view& col, reduce_tail& t, cudaStream_t stream)
{
  launch_reduce<T, A, OP_SUM>(col, t, stream);
}
template <typename A>
void dispatch_mean(int32_t in_type, const b2_column_view& col, reduce_tail& t, cudaStream_t stream)
{
  switch (in_type) {
    case B2_INT8: mean_launch<int8_t, A>(col, t, stream); break;
    case B2_INT16: mean_launch<int16_t, A>(col, t, stream); break;
    case B2_INT32: mean_launch<int32_t, A>(col, t, stream); break;
    case B2_INT64: mean_launch<int64_t, A>(col, t, stream); break;
    case B2_UINT8: case B2_BOOL8: mean_launch<uint8_t, A>(col, t, stream); break;
    case B2_UINT16: mean_launch<uint16_t, A>(col, t, stream); break;
    case B2_UINT32: mean_launch<uint32_t, A>(col, t, stream); break;
    case B2_UINT64: mean_launch<uint64_t, A>(col, t, stream); break;
    case B2_FLOAT32: mean_launch<float, A>(col, t, stream); break;
    case B2_FLOAT64: mean_launch<double, A>(col, t, stream); break;
    default: B2_FAIL(B2_ERR_DATA_TYPE, "Reduction operator not supported for this type");
  }
}

int op_of(int32_t kind)
{
  switch (kind) {
    case B2_AGG_SUM: return OP_SUM;
    case B2_AGG_PRODUCT: return OP_PRODUCT;
    case B2_AGG_MIN: return OP_MIN;
    case B2_AGG_MAX: return OP_MAX;
    default: return -1;
  }
}

}  // namespace

std::unique_ptr<b2_scalar> make_scalar(int32_t type_id, const void* host_value, bool valid, cudaStream_t stream)
{
  B2_EXPECTS(is_fixed_width(type_id), B2_ERR_DATA_TYPE, "scalar type must be fixed width");
  auto s = std::make_unique<b2_scalar>();
  s->type_id = type_id;
  s->data    = dbuf(16, stream);
  unsigned char h[16] = {0};
  if (host_value) memcpy(h, host_value, type_width(type_id));
  int32_t v = valid ? 1 : 0;
  memcpy(h + 8, &v, 4);
  // pageable source: the runtime stages it before returning, so `h` may go out of scope
  B2_CUDA_TRY(cudaMemcpyAsync(s->data.ptr, h, 16, cudaMemcpyHostToDevice, stream));
  return s;
}

std::unique_ptr<b2_scalar> reduce(const b2_column_view& col, int32_t kind, int32_t out_type, const b2_scalar* init,
                                  cudaStream_t stream)
{
  validate_column(col);
  const int32_t in_type = storage_type(col.type_id);
  B2_EXPECTS(!init || init->type_id == col.type_id, B2_ERR_DATA_TYPE, "column and initial value must be the same type");
  B2_EXPECTS(!init || (kind == B2_AGG_SUM || kind == B2_AGG_PRODUCT || kind == B2_AGG_MIN || kind == B2_AGG_MAX),
             B2_ERR_INVALID_ARGUMENT, "Initial value is only supported for SUM, PRODUCT, MIN, MAX aggregation types");
  B2_EXPECTS(kind == B2_AGG_MEAN || op_of(kind) >= 0, B2_ERR_INVALID_ARGUMENT, "Unsupported reduction operator");
  B2_EXPECTS(is_fixed_width(out_type), B2_ERR_DATA_TYPE, "Unsupported output data type");

  // no data: invalid default-constructed scalar of the output type (reductions.cpp:498-500)
  if (col.size == col.null_count) {
    if (kind == B2_AGG_MIN || kind == B2_AGG_MAX)
      B2_EXPECTS(col.type_id == out_type, B2_ERR_LOGIC, "min/max operation requires matching output type");
    return make_scalar(out_type, nullptr, false, stream);
  }
  auto out = std::make_unique<b2_scalar>();
  out->type_id = out_type;
  out->data    = dbuf(16, stream);
  B2_CUDA_TRY(cudaMemsetAsync(out->data.ptr, 0, 16, stream));
  reduce_tail t{};
  t.out_value   = out->data.ptr;
  t.out_type    = storage_type(out_type);
  t.in_type     = in_type;
  t.init_value  = init ? init->data.ptr : nullptr;
  t.valid_count = (int64_t)col.size - col.null_count;
  t.is_bool     = col.type_id == B2_BOOL8;

  if (kind == B2_AGG_MEAN) {
    B2_EXPECTS(is_numeric(col.type_id), B2_ERR_DATA_TYPE,
               "Reduction operators other than `min` and `max` are not supported for non-arithmetic types");
    B2_EXPECTS(is_float_id(out_type), B2_ERR_DATA_TYPE, "Unsupported output data type");
    t.mean = 1;
    if (out_type == B2_FLOAT32) dispatch_mean<float>(in_type, col, t, stream);
    else dispatch_mean<double>(in_type, col, t, stream);
    return out;
  }
  if (kind == B2_AGG_MIN || kind == B2_AGG_MAX) {
    B2_EXPECTS(col.type_id == out_type, B2_ERR_LOGIC, "min/max operation requires matching output type");
  } else {
    B2_EXPECTS(is_numeric(col.type_id), B2_ERR_DATA_TYPE, "Reduction operator not supported for this type");
    B2_EXPECTS(is_numeric(out_type), B2_ERR_DATA_TYPE, "Unsupported output data type");
  }
  const bool same = out_type == col.type_id;
  dispatch_reduce(in_type, !same, same && in_type == B2_FLOAT32, op_of(kind), col, t, stream);
  return out;
}

// ------------------------------------------------------------------------------------------------
// scan: single pass, decoupled look-back (flag/aggregate/inclusive arrays with release/acquire)
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int SC_THREADS = 512;  // two CTAs per SM
// 16-byte vectors per lane per tile: 64 KB tiles for 8-byte types (8192 elements), 32 KB otherwise. The look-back consumes
// SC_LB * 32 predecessor records per global-memory round trip, so tiles/us <= SC_LB * 32 / latency: larger tiles and a
// wider window lift that ceiling above the HBM rate.
template <typename T> constexpr int sc_k() { return sizeof(T) == 8 ? 8 : 4; }
constexpr int SC_LB = 4;  // predecessor records per look-back lane and round

__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v)
{
#ifdef B2_EMU
  *reinterpret_cast<volatile uint32_t*>(p) = v;
#else
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p)
{
#ifdef B2_EMU
  return *reinterpret_cast<const volatile uint32_t*>(p);
#else
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}

// valid bits of rows [r, r+cnt) (cnt <= 16) at absolute bit position
__device__ __forceinline__ uint32_t valid_bits_at(const uint32_t* mask, int64_t bit, int64_t last_word)
{
  return load_mask_word_unaligned(mask, bit, last_word);
}

template <typename T, int OP, bool COUNT>
__global__ void __launch_bounds__(SC_THREADS, 2) scan_kernel(const T* __restrict__ in, const uint32_t* __restrict__ mask,
                                                          int64_t bit_offset, int64_t n, bool exclusive, bool in_aligned,
                                                          T* __restrict__ out, scan_state st)
{
  using B = binop<T, OP>;
  constexpr int V = 16 / sizeof(T);
  constexpr int SC_K = sc_k<T>();
  constexpr int NW = SC_THREADS / 32;
  constexpr int64_t WARP_ELEMS = 32 * V * SC_K;
  constexpr int64_t TILE = WARP_ELEMS * NW;
  __shared__ T s_wtot[NW];
  __shared__ T s_prefix;
  __shared__ uint32_t s_tile;
  if (threadIdx.x == 0) s_tile = atomicAdd(st.ticket, 1u);
  __syncthreads();
  const int64_t tile = s_tile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wbase = tile * TILE + warp * WARP_ELEMS;
  const int64_t last_word = mask ? ((bit_offset + n - 1) >> 5) : 0;

  T v[SC_K][V];
  // ---- load ----
#pragma unroll
  for (int k = 0; k < SC_K; ++k) {
    const int64_t e0 = wbase + ((int64_t)k * 32 + lane) * V;
    if constexpr (COUNT) {
#pragma unroll
      for (int j = 0; j < V; ++j) v[k][j] = (e0 + j < n) ? T(1) : T(0);
    } else if (in_aligned && e0 + V <= n) {
      int4 q = ld_nc_v4(in + e0);
      memcpy(&v[k][0], &q, 16);
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j) v[k][j] = (e0 + j < n) ? in[e0 + j] : B::identity();
    }
    if (mask) {
      if (e0 < n) {
        uint32_t bits = valid_bits_at(mask, bit_offset + e0, last_word);
#pragma unroll
        for (int j = 0; j < V; ++j)
          if (!((bits >> j) & 1u) || e0 + j >= n) v[k][j] = COUNT ? T(0) : B::identity();
      }
    }
  }
  // ---- warp-local scan over K steps ----
  T carry = B::identity();
#pragma unroll
  for (int k = 0; k < SC_K; ++k) {
    // inclusive scan inside the vector
#pragma unroll
    for (int j = 1; j < V; ++j) v[k][j] = B::apply(v[k][j - 1], v[k][j]);
    T tot = v[k][V - 1];
    T inc = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      T nb = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc = B::apply(nb, inc);
    }
    T excl_lane = __shfl_up_sync(0xffffffffu, inc, 1);
    T pre = lane == 0 ? carry : B::apply(carry, excl_lane);
#pragma unroll
    for (int j = 0; j < V; ++j) v[k][j] = B::apply(pre, v[k][j]);
    carry = B::apply(carry, __shfl_sync(0xffffffffu, inc, 31));
  }
  if (lane == 0) s_wtot[warp] = carry;
  __syncthreads();
  // ---- block aggregate + look-back (warp 0) ----
  if (warp == 0) {
    T block_tot = s_wtot[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) block_tot = B::apply(block_tot, s_wtot[w]);
    if (tile == 0) {
      if (lane == 0) {
        publish_rec<T>(st.rec, 2u, block_tot);
        s_prefix = B::identity();
      }
    } else {
      if (lane == 0) publish_rec<T>(st.rec + tile, 1u, block_tot);
      T excl = B::identity();
      int64_t base = tile - 1;  // nearest predecessor not folded yet
      while (true) {
        // lane l holds the SC_LB records at distances l * SC_LB + r from `base` (lane 0 = the nearest ones), fetched with
        // independent 16-byte loads; tiles before the first one act as an inclusive identity
        uint32_t f[SC_LB];
        T c[SC_LB];
#pragma unroll
        for (int r = 0; r < SC_LB; ++r) {
          const int64_t idx = base - ((int64_t)lane * SC_LB + r);
          f[r] = 2u;
          c[r] = B::identity();
          if (idx >= 0) f[r] = read_rec<T>(st.rec + idx, c[r]);
        }
        // leading ready records of this lane, the first inclusive one among them, and their fold (nearest first)
        int nr = 0, fi = SC_LB;
        T part = B::identity();
#pragma unroll
        for (int r = 0; r < SC_LB; ++r) {
          if (nr == r && fi == SC_LB && f[r] != 0u) {
            ++nr;
            part = B::apply(c[r], part);
            if (f[r] == 2u) fi = r;
          }
        }
        const bool has_incl = fi < SC_LB;
        const bool blocked  = !has_incl && nr < SC_LB;  // a record that is still needed has not been published yet
        const unsigned incl_mask = __ballot_sync(0xffffffffu, has_incl);
        const unsigned blk_mask  = __ballot_sync(0xffffffffu, blocked);
        const int first_incl = incl_mask ? (__ffs(incl_mask) - 1) : 32;
        const int first_blk  = blk_mask ? (__ffs(blk_mask) - 1) : 32;
        if (first_blk < first_incl) continue;  // poll again (the loads above are volatile)
        if (lane > first_incl) part = B::identity();
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part = B::apply(__shfl_xor_sync(0xffffffffu, part, o), part);
        excl = B::apply(part, excl);
        if (incl_mask) break;
        base -= 32 * SC_LB;
      }
      if (lane == 0) {
        publish_rec<T>(st.rec + tile, 2u, B::apply(excl, block_tot));
        s_prefix = excl;
      }
    }
  }
  __syncthreads();
  T pre = s_prefix;
  for (int w = 0; w < warp; ++w) pre = B::apply(pre, s_wtot[w]);
  // ---- store ----
#pragma unroll
  for (int k = 0; k < SC_K; ++k) {
    const int64_t e0 = wbase + ((int64_t)k * 32 + lane) * V;
    T o[V];
    if (!exclusive) {
#pragma unroll
      for (int j = 0; j < V; ++j) o[j] = B::apply(pre, v[k][j]);
    } else {
      // exclusive: element j gets the inclusive value of its predecessor
      // inclusive value of the last element of the previous lane; lane 0 takes the last element of
      // the previous step (k is unrolled, so the branch below is compile-time)
      const T last = B::apply(pre, v[k][V - 1]);
      const T up   = __shfl_up_sync(0xffffffffu, last, 1);
      T prev_step_last = pre;  // first element of the warp segment: prefix of earlier warps / tiles
      if (k > 0) prev_step_last = __shfl_sync(0xffffffffu, B::apply(pre, v[k > 0 ? k - 1 : 0][V - 1]), 31);
      o[0] = lane == 0 ? prev_step_last : up;
#pragma unroll
      for (int j = 1; j < V; ++j) o[j] = B::apply(pre, v[k][j - 1]);
    }
    if (e0 + V <= n) {
      int4 q;
      memcpy(&q, &o[0], 16);
      st_na_v4(out + e0, q);
    } else {
#pragma unroll
      for (int j = 0; j < V; ++j)
        if (e0 + j < n) out[e0 + j] = o[j];
    }
  }
}

template <typename T, int OP, bool COUNT>
void launch_scan(const T* in, const uint32_t* mask, int64_t bit_offset, int64_t n, bool exclusive, T* out, cudaStream_t stream)
{
  constexpr int V = 16 / sizeof(T);
  constexpr int64_t TILE = (int64_t)32 * V * sc_k<T>() * (SC_THREADS / 32);
  const int64_t ntiles = (n + TILE - 1) / TILE;
  dbuf work(sizeof(uint4) * (ntiles + 1), stream);
  B2_CUDA_TRY(cudaMemsetAsync(work.ptr, 0, work.bytes, stream));
  scan_state st;
  st.rec    = work.as<uint4>();
  st.ticket = reinterpret_cast<uint32_t*>(work.as<uint4>() + ntiles);
  const bool aligned = in == nullptr || (reinterpret_cast<uintptr_t>(in) & 15) == 0;
  B2_LAUNCH((scan_kernel<T, OP, COUNT>), (unsigned)ntiles, SC_THREADS, 0, stream, in, mask, bit_offset, n, exclusive, aligned,
            out, st);
}

template <typename T>
void dispatch_scan_op(int op, const b2_column_view& col, const uint32_t* mask, bool exclusive, void* out, cudaStream_t stream)
{
  const T* in = static_cast<const T*>(col.data) + col.offset;
  switch (op) {
    case OP_SUM: launch_scan<T, OP_SUM, false>(in, mask, col.offset, col.size, exclusive, static_cast<T*>(out), stream); break;
    case OP_PRODUCT: launch_scan<T, OP_PRODUCT, false>(in, mask, col.offset, col.size, exclusive, static_cast<T*>(out), stream); break;
    case OP_MIN: launch_scan<T, OP_MIN, false>(in, mask, col.offset, col.size, exclusive, static_cast<T*>(out), stream); break;
    case OP_MAX: launch_scan<T, OP_MAX, false>(in, mask, col.offset, col.size, exclusive, static_cast<T*>(out), stream); break;
  }
}

// first null position (INCLUDE policy: everything from the first null on is null) — mask_scan,
// scan_inclusive.cu:36-61; flip = 0 finds the first valid position instead
__global__ void first_null_kernel(const uint32_t* __restrict__ mask, int64_t bit_offset, int64_t n, uint32_t flip, unsigned long long* first)
{
  const int64_t nwords = (n + 31) / 32;
  const int64_t last_word = (bit_offset + n - 1) >> 5;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long best = ~0ull;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += stride) {
    uint32_t bits = load_mask_word_unaligned(mask, bit_offset + w * 32, last_word);
    int64_t rem = n - w * 32;
    uint32_t live = rem < 32 ? ((1u << rem) - 1u) : 0xffffffffu;
    uint32_t nulls = (bits ^ flip) & live;
    if (nulls) {
      unsigned long long p = (unsigned long long)(w * 32 + __ffs(nulls) - 1);
      if (p < best) best = p;
      break;  // later words of this thread are farther
    }
  }
  if (best != ~0ull) atomicMin(first, best);
}

__global__ void mask_from_first_null_kernel(uint32_t* __restrict__ out, int64_t n, const unsigned long long* first, int excl_off,
                                            unsigned long long* valid_count)
{
  unsigned long long f = *first;
  int64_t pos = f == ~0ull ? n : (int64_t)min((unsigned long long)n, f + (unsigned long long)excl_off);
  const int64_t nwords = (n + 31) / 32;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += stride) {
    int64_t lo = w * 32;
    uint32_t bits = pos >= lo + 32 ? 0xffffffffu : (pos <= lo ? 0u : ((1u << (pos - lo)) - 1u));
    out[w] = bits;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *valid_count = (unsigned long long)pos;
}

// rows [0, first valid row] of an exclusive float MIN scan: their prefix holds no valid row
template <typename T>
__global__ void fill_empty_prefix_kernel(T* __restrict__ out, int64_t n, const unsigned long long* first)
{
  const unsigned long long f = *first;  // ~0: no valid row
  const int64_t end = f >= (unsigned long long)n ? n : (int64_t)f + 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) out[i] = std::numeric_limits<T>::infinity();
}

}  // namespace

column_ptr scan(const b2_column_view& col, int32_t kind, int32_t scan_type, int32_t null_handling, cudaStream_t stream)
{
  validate_column(col);
  const bool exclusive = scan_type == B2_SCAN_EXCLUSIVE;
  const bool count = kind == B2_AGG_COUNT_VALID || kind == B2_AGG_COUNT_ALL;
  const int op = op_of(kind);
  B2_EXPECTS(count || op >= 0, B2_ERR_LOGIC, "Unsupported aggregation operator for scan");
  const int32_t sid = storage_type(col.type_id);
  B2_EXPECTS(count || is_numeric(sid) || is_fixed_width(col.type_id), B2_ERR_DATA_TYPE, "unsupported type for scan");
  const int64_t n = col.size;
  const bool nullable = col.null_mask != nullptr;

  auto out = make_column(count ? B2_INT32 : col.type_id, col.size, false, stream);
  if (n == 0) return out;

  // ---- output mask (scan_inclusive.cu:204-212 / scan_exclusive.cu:90-98) ----
  const uint32_t* scan_mask = nullptr;  // mask used to replace nulls by the identity
  int64_t scan_mask_offset = 0;
  if (null_handling == B2_NULL_EXCLUDE) {
    if (has_nulls(col) || nullable) {
      out->mask       = copy_bitmask(col.null_mask, col.offset, (int64_t)col.offset + n, stream);
      out->null_count = col.null_count;
    }
  } else if (nullable) {
    out->mask = dbuf(bitmask_bytes(n), stream);
    B2_CUDA_TRY(cudaMemsetAsync(out->mask.ptr, 0, out->mask.bytes, stream));
    dbuf first(sizeof(unsigned long long), stream);
    B2_CUDA_TRY(cudaMemsetAsync(first.ptr, 0xff, sizeof(unsigned long long), stream));
    int grid = (int)std::max<int64_t>(1, std::min<int64_t>((num_words(n) + 255) / 256, num_sms() * 4));
    B2_LAUNCH(first_null_kernel, grid, 256, 0, stream, col.null_mask, (int64_t)col.offset, n, 0xffffffffu, first.as<unsigned long long>());
    out->pending = dbuf(sizeof(unsigned long long), stream);
    out->pending_stream = stream;
    out->pending_is_valid_count = true;
    out->null_count = -1;
    B2_LAUNCH(mask_from_first_null_kernel, grid, 256, 0, stream, out->mask.as<uint32_t>(), n, first.as<unsigned long long>(),
              exclusive ? 1 : 0, out->pending.as<unsigned long long>());
  }
  if (has_nulls(col)) {
    scan_mask = col.null_mask;
    scan_mask_offset = col.offset;
  }

  if (count) {
    // COUNT_VALID counts the OUTPUT mask bits (scan_inclusive.cu:117-145); COUNT_ALL counts rows
    const uint32_t* cm = nullptr;
    int64_t cm_off = 0;
    if (kind == B2_AGG_COUNT_VALID && out->mask.ptr) { cm = out->mask.as<uint32_t>(); cm_off = 0; }
    launch_scan<int32_t, OP_SUM, true>(nullptr, cm, cm_off, n, exclusive, out->data.as<int32_t>(), stream);
    return out;
  }
  b2_column_view c2 = col;
  c2.null_mask = scan_mask;
  (void)scan_mask_offset;
  // a running SUM of BOOL8 is true from the first true row on (the reference adds bools as ints and stores bool): MAX of the
  // 0 / 1 bytes, which a uint8 + would wrap back to 0 after 256 true rows
  const int sop = sid == B2_BOOL8 && op == OP_SUM ? OP_MAX : op;
  switch (sid) {
    case B2_INT8: dispatch_scan_op<int8_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_INT16: dispatch_scan_op<int16_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_INT32: dispatch_scan_op<int32_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_INT64: dispatch_scan_op<int64_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_UINT8: case B2_BOOL8: dispatch_scan_op<uint8_t>(sop, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_UINT16: dispatch_scan_op<uint16_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_UINT32: dispatch_scan_op<uint32_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_UINT64: dispatch_scan_op<uint64_t>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_FLOAT32: dispatch_scan_op<float>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    case B2_FLOAT64: dispatch_scan_op<double>(op, c2, scan_mask, exclusive, out->data.ptr, stream); break;
    default: B2_FAIL(B2_ERR_DATA_TYPE, "unsupported type for scan");
  }
  if (exclusive && op == OP_MIN && is_float_id(sid)) {
    // an empty prefix holds MIN's identity, NaN (binop); the reference's identity there is +inf
    dbuf first(sizeof(unsigned long long), stream);
    B2_CUDA_TRY(cudaMemsetAsync(first.ptr, scan_mask ? 0xff : 0, sizeof(unsigned long long), stream));
    int grid = 1;
    if (scan_mask) {
      grid = (int)std::max<int64_t>(1, std::min<int64_t>((num_words(n) + 255) / 256, num_sms() * 4));
      B2_LAUNCH(first_null_kernel, grid, 256, 0, stream, scan_mask, (int64_t)col.offset, n, 0u, first.as<unsigned long long>());
    }
    if (sid == B2_FLOAT32) B2_LAUNCH(fill_empty_prefix_kernel<float>, grid, 256, 0, stream, out->data.as<float>(), n, first.as<unsigned long long>());
    else B2_LAUNCH(fill_empty_prefix_kernel<double>, grid, 256, 0, stream, out->data.as<double>(), n, first.as<unsigned long long>());
  }
  return out;
}

// ------------------------------------------------------------------------------------------------
// segmented reduce: one warp per segment
// ------------------------------------------------------------------------------------------------
namespace {

template <typename T, typename A, int OP>
__global__ void __launch_bounds__(256) segreduce_kernel(const T* __restrict__ data, const uint32_t* __restrict__ mask,
                                                        int64_t bit_offset, const int32_t* __restrict__ offsets,
                                                        int64_t nseg, int32_t out_type, bool is_bool, int null_include,
                                                        const void* init, int32_t in_type, int mean, void* __restrict__ out,
                                                        uint32_t* __restrict__ out_mask, unsigned long long* valid_segments)
{
  using B = binop<A, OP>;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const unsigned lane = lane_id();
  bool has_init = init != nullptr;
  bool init_valid = false;
  A init_v = B::identity();
  if (has_init) {
    init_valid = *reinterpret_cast<const int32_t*>(static_cast<const char*>(init) + 8) != 0;
    if (init_valid) init_v = load_scalar_as<A>(init, in_type);
  }
  unsigned long long nvalid_seg = 0;
  // process 32 segments per warp iteration so that one lane can assemble a full mask word
  const int64_t ngroups = (nseg + 31) / 32;
  for (int64_t g = warp_global; g < ngroups; g += nwarps) {
    uint32_t word = 0;
    for (int s = 0; s < 32; ++s) {
      const int64_t seg = g * 32 + s;
      if (seg >= nseg) break;
      const int64_t b = offsets[seg], e = offsets[seg + 1];
      A acc = B::identity();
      int64_t vc = 0;
      for (int64_t i = b + lane; i < e; i += 32) {
        bool valid = mask == nullptr || bit_is_set(mask, bit_offset + i);
        if (valid) {
          acc = B::apply(acc, load_as<T, A>(data, i, is_bool));
          ++vc;
        }
      }
      acc = warp_reduce_op<A, OP>(acc);
      vc = warp_sum(vc);
      const int64_t len = e - b;
      bool seg_valid;
      if (mask == nullptr) seg_valid = has_init ? init_valid : len > 0;
      else if (!null_include) seg_valid = init_valid || vc > 0;
      else seg_valid = (has_init ? init_valid : len > 0) && vc == len;
      if (lane == 0) {
        A r = B::apply(init_v, acc);
        if (mean) r = vc > 0 ? r / A(vc) : r;
        store_as<A>(out, seg, out_type, r);
      }
      word |= (seg_valid ? 1u : 0u) << s;
    }
    if (lane == 0) {
      out_mask[g] = word;
      nvalid_seg += __popc(word);
    }
  }
  if (lane == 0 && nvalid_seg) atomicAdd(valid_segments, nvalid_seg);
}

template <typename T, typename A>
void dispatch_seg_op(int op, bool mean, const b2_column_view& col, const int32_t* offsets, int64_t nseg, int32_t out_type,
                     int null_include, const b2_scalar* init, b2_column& out, cudaStream_t stream)
{
  const T* data = static_cast<const T*>(col.data) + col.offset;
  const uint32_t* mask = col.null_mask;  // the reference keys the validity rule on nullable(), not on null_count
  const int64_t groups = (nseg + 31) / 32;
  int grid = (int)std::max<int64_t>(1, std::min<int64_t>((groups * 32 + 255) / 256, num_sms() * 8));
  const bool is_bool = col.type_id == B2_BOOL8;
  const void* iv = init ? init->data.ptr : nullptr;
  const int32_t in_type = storage_type(col.type_id);
  auto go = [&](auto opc) {
    constexpr int OP = decltype(opc)::value;
    B2_LAUNCH((segreduce_kernel<T, A, OP>), grid, 256, 0, stream, data, mask, (int64_t)col.offset, offsets, nseg,
              storage_type(out_type), is_bool, null_include, iv, in_type, mean ? 1 : 0, out.data.ptr, out.mask.as<uint32_t>(),
              out.pending.as<unsigned long long>());
  };
  switch (op) {
    case OP_SUM: go(std::integral_constant<int, OP_SUM>{}); break;
    case OP_PRODUCT: go(std::integral_constant<int, OP_PRODUCT>{}); break;
    case OP_MIN: go(std::integral_constant<int, OP_MIN>{}); break;
    case OP_MAX: go(std::integral_constant<int, OP_MAX>{}); break;
  }
}

}  // namespace

column_ptr segmented_reduce(const b2_column_view& col, const int32_t* offsets, int32_t num_offsets, int32_t kind,
                            int32_t out_type, int32_t null_handling, const b2_scalar* init, cudaStream_t stream)
{
  validate_column(col);
  B2_EXPECTS(!init || init->type_id == col.type_id, B2_ERR_DATA_TYPE, "column and initial value must be the same type");
  B2_EXPECTS(!init || (kind == B2_AGG_SUM || kind == B2_AGG_PRODUCT || kind == B2_AGG_MIN || kind == B2_AGG_MAX),
             B2_ERR_LOGIC, "Initial value is only supported for SUM, PRODUCT, MIN, MAX aggregation types");
  if (col.size == 0 && num_offsets == 0) return make_column(out_type, 0, false, stream);
  B2_EXPECTS(num_offsets > 0, B2_ERR_LOGIC, "`offsets` should have at least 1 element.");
  const bool mean = kind == B2_AGG_MEAN;
  const int op = mean ? OP_SUM : op_of(kind);
  B2_EXPECTS(op >= 0, B2_ERR_LOGIC, "Unsupported aggregation type.");
  if (kind == B2_AGG_MIN || kind == B2_AGG_MAX)
    B2_EXPECTS(col.type_id == out_type, B2_ERR_LOGIC, "segmented_reduce min/max requires matching output type");
  else
    B2_EXPECTS(is_numeric(col.type_id) && is_numeric(out_type), B2_ERR_DATA_TYPE, "unsupported type for segmented_reduce");
  if (mean) B2_EXPECTS(is_float_id(out_type), B2_ERR_DATA_TYPE, "Unsupported output data type");

  const int64_t nseg = num_offsets - 1;
  auto out = make_column(out_type, (int32_t)nseg, true, stream);
  if (nseg == 0) { out->mask.reset(); return out; }
  out->pending = dbuf(sizeof(unsigned long long), stream);
  out->pending_stream = stream;
  out->pending_is_valid_count = true;
  out->null_count = -1;
  B2_CUDA_TRY(cudaMemsetAsync(out->pending.ptr, 0, sizeof(unsigned long long), stream));
  const int inc = null_handling == B2_NULL_INCLUDE;
  const int32_t sid = storage_type(col.type_id);
  const bool same = out_type == col.type_id && !mean;
#define SEG(T, A) dispatch_seg_op<T, A>(op, mean, col, offsets, nseg, out_type, inc, init, *out, stream)
  if (mean) {
    const bool f32 = out_type == B2_FLOAT32;
    switch (sid) {
      case B2_INT8: if (f32) SEG(int8_t, float); else SEG(int8_t, double); break;
      case B2_INT16: if (f32) SEG(int16_t, float); else SEG(int16_t, double); break;
      case B2_INT32: if (f32) SEG(int32_t, float); else SEG(int32_t, double); break;
      case B2_INT64: if (f32) SEG(int64_t, float); else SEG(int64_t, double); break;
      case B2_UINT8: case B2_BOOL8: if (f32) SEG(uint8_t, float); else SEG(uint8_t, double); break;
      case B2_UINT16: if (f32) SEG(uint16_t, float); else SEG(uint16_t, double); break;
      case B2_UINT32: if (f32) SEG(uint32_t, float); else SEG(uint32_t, double); break;
      case B2_UINT64: if (f32) SEG(uint64_t, float); else SEG(uint64_t, double); break;
      case B2_FLOAT32: if (f32) SEG(float, float); else SEG(float, double); break;
      case B2_FLOAT64: if (f32) SEG(double, float); else SEG(double, double); break;
      default: B2_FAIL(B2_ERR_DATA_TYPE, "unsupported type for segmented_reduce");
    }
  } else {
    // unsigned inputs: uint64 when the output is the input type (MIN / MAX order), else int64 like the signed ones
    // (segmented/simple.cuh reduce_numeric): a sum with bit 63 set then converts to a negative float, as in the reference
    switch (sid) {
      case B2_INT8: SEG(int8_t, int64_t); break;
      case B2_INT16: SEG(int16_t, int64_t); break;
      case B2_INT32: SEG(int32_t, int64_t); break;
      case B2_INT64: SEG(int64_t, int64_t); break;
      case B2_UINT8: case B2_BOOL8: if (same) SEG(uint8_t, uint64_t); else SEG(uint8_t, int64_t); break;
      case B2_UINT16: if (same) SEG(uint16_t, uint64_t); else SEG(uint16_t, int64_t); break;
      case B2_UINT32: if (same) SEG(uint32_t, uint64_t); else SEG(uint32_t, int64_t); break;
      case B2_UINT64: if (same) SEG(uint64_t, uint64_t); else SEG(uint64_t, int64_t); break;
      case B2_FLOAT32: if (same) SEG(float, float); else SEG(float, double); break;
      case B2_FLOAT64: SEG(double, double); break;
      default: B2_FAIL(B2_ERR_DATA_TYPE, "unsupported type for segmented_reduce");
    }
  }
#undef SEG
  return out;
}

}  // namespace b2

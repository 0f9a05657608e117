// unary.cuh — the streaming kernels of cudf::unary_operation, cast, is_nan / is_not_nan and is_null / is_valid (unary.cu),
// instantiated per family in unary_{math,bits,cast}.cu so that the three files compile in parallel.
//
// unary_kernel<F, C, In, Out> computes out[i] = Out(f(C(in[i]))) for one functor F and one compute type C. One pass writes the
// values and, when the output has a mask, the output's mask words (a copy of the input's, realigned to offset 0); the null count
// is the input's, so nothing is counted. In / Out are the element types, or `rt`: the type is a warp-uniform runtime parameter
// read and written through binop::load_as / store_as.
//  - generic path: a warp covers 32 consecutive rows per step, one row per lane; lane 0 writes the step's mask word;
//  - vector path (In and Out compile-time, input and output 16-byte aligned): a lane owns V = 16 / max(sizeof(In), sizeof(Out))
//    consecutive rows, the wider side moves 16 bytes per access, and lanes 0..V-1 write the step's V mask words.
// `fold` >= 0 makes the output non-nullable instead: a null row gets the value `fold` (is_nan: 0, is_not_nan: 1).
//
// validity_kernel writes is_null / is_valid: a thread expands one 32-bit mask word into 32 BOOL8 bytes.
#pragma once
#include "binaryop.cuh"

#include <cmath>
#include <type_traits>

namespace b2 {
namespace unary {

struct rt {};  // element type given at run time (args::in_type / out_type)

struct args {
  const void* in;         // row 0 of the view (offset applied)
  const uint32_t* mask;   // the input's mask; nullptr: every row valid
  int64_t bit;            // bit of row 0 in mask (the view's offset)
  int64_t last_word;      // last mask word holding a bit of the view
  int32_t in_type;        // storage type ids
  int32_t out_type;
  void* out;
  uint32_t* out_mask;     // nullptr: the output has no mask
  int64_t n;
  int64_t mul, div;       // chrono casts: out ticks = floor(in ticks * mul / div), one of the two is 1
  int32_t fold;           // -1, or the value of a null row in a non-nullable output
  bool fast;
};

// the family entry points (unary_*.cu); a type they have no kernel for is an internal error
void launch_math(int op, const args& a, cudaStream_t stream);
void launch_bits(int op, const args& a, cudaStream_t stream);
void launch_nan(bool want_nan, const args& a, cudaStream_t stream);
void launch_validity(bool want_valid, const args& a, cudaStream_t stream);
void launch_cast(const args& a, cudaStream_t stream);

template <typename T> constexpr int32_t type_of() {
  if constexpr (std::is_same_v<T, int8_t>) return B2_INT8;
  else if constexpr (std::is_same_v<T, int16_t>) return B2_INT16;
  else if constexpr (std::is_same_v<T, int32_t>) return B2_INT32;
  else if constexpr (std::is_same_v<T, int64_t>) return B2_INT64;
  else if constexpr (std::is_same_v<T, uint8_t>) return B2_UINT8;
  else if constexpr (std::is_same_v<T, uint16_t>) return B2_UINT16;
  else if constexpr (std::is_same_v<T, uint32_t>) return B2_UINT32;
  else if constexpr (std::is_same_v<T, uint64_t>) return B2_UINT64;
  else if constexpr (std::is_same_v<T, float>) return B2_FLOAT32;
  else return B2_FLOAT64;
}

// ---- functors: operator()(C x, const args&) ---------------------------------------------------------------------------
template <int OP>
struct math_fn {  // SIN .. ABS and RINT; C is float, double, or an integer type for ABS
  template <typename C>
  __device__ __forceinline__ C operator()(C x, const args&) const
  {
    if constexpr (OP == B2_UNARY_ABS) {
      if constexpr (std::is_floating_point_v<C>) return std::fabs(x);
      else if constexpr (std::is_signed_v<C>) return x < 0 ? binop::wrap_sub(C(0), x) : x;
      else return x;
    } else if constexpr (OP == B2_UNARY_SIN) return std::sin(x);
    else if constexpr (OP == B2_UNARY_COS) return std::cos(x);
    else if constexpr (OP == B2_UNARY_TAN) return std::tan(x);
    else if constexpr (OP == B2_UNARY_ARCSIN) return std::asin(x);
    else if constexpr (OP == B2_UNARY_ARCCOS) return std::acos(x);
    else if constexpr (OP == B2_UNARY_ARCTAN) return std::atan(x);
    else if constexpr (OP == B2_UNARY_SINH) return std::sinh(x);
    else if constexpr (OP == B2_UNARY_COSH) return std::cosh(x);
    else if constexpr (OP == B2_UNARY_TANH) return std::tanh(x);
    else if constexpr (OP == B2_UNARY_ARCSINH) return std::asinh(x);
    else if constexpr (OP == B2_UNARY_ARCCOSH) return std::acosh(x);
    else if constexpr (OP == B2_UNARY_ARCTANH) return std::atanh(x);
    else if constexpr (OP == B2_UNARY_EXP) return std::exp(x);
    else if constexpr (OP == B2_UNARY_LOG) return std::log(x);
    else if constexpr (OP == B2_UNARY_SQRT) return std::sqrt(x);
    else if constexpr (OP == B2_UNARY_CBRT) return std::cbrt(x);
    else if constexpr (OP == B2_UNARY_CEIL) return std::ceil(x);
    else if constexpr (OP == B2_UNARY_FLOOR) return std::floor(x);
    else return std::rint(x);  // RINT: the current rounding mode, to nearest even
  }
};

// BIT_COUNT (C: the unsigned type of the input's width), BIT_INVERT (C = uint64: ~x keeps its low bits on the narrowing store),
// NOT (C = double: x == 0 for every numeric x), NEGATE (C = uint64 for the integers, the two's-complement negation; or float /
// double)
template <int OP>
struct bits_fn {
  template <typename C>
  __device__ __forceinline__ auto operator()(C x, const args&) const
  {
    if constexpr (OP == B2_UNARY_BIT_COUNT) {
      if constexpr (sizeof(C) == 8) return (int32_t)__popcll((unsigned long long)x);
      else return (int32_t)__popc((unsigned)x);
    } else if constexpr (OP == B2_UNARY_BIT_INVERT) return static_cast<C>(~x);
    else if constexpr (OP == B2_UNARY_NOT) return x == C(0);
    else if constexpr (std::is_integral_v<C>) return binop::wrap_sub(C(0), x);  // NEGATE
    else return -x;
  }
};

template <bool WANT_NAN>
struct nan_fn {
  template <typename C>
  __device__ __forceinline__ bool operator()(C x, const args&) const { return std::isnan(x) == WANT_NAN; }
};

struct cast_fn {  // numeric casts: the conversion is the store's static_cast
  template <typename C>
  __device__ __forceinline__ C operator()(C x, const args&) const { return x; }
};

struct chrono_fn {  // C = int64: ticks of one unit to another, toward -inf
  __device__ __forceinline__ int64_t operator()(int64_t x, const args& a) const
  {
    if (a.div == 1) return binop::wrap_mul(x, a.mul);
    const int64_t q = x / a.div;
    return q - (int64_t)(x % a.div < 0);
  }
};

// ---- loads and stores -------------------------------------------------------------------------------------------------
template <typename C, typename In>
__device__ __forceinline__ C load_one(const args& a, int64_t i)
{
  if constexpr (std::is_same_v<In, rt>) return binop::load_as<C>(a.in, a.in_type, i);
  else return static_cast<C>(static_cast<const In*>(a.in)[i]);
}
template <typename Out, typename R>
__device__ __forceinline__ void store_one(const args& a, int64_t i, R v)
{
  if constexpr (std::is_same_v<Out, rt>) binop::store_as(a.out, a.out_type, i, v);
  else static_cast<Out*>(a.out)[i] = static_cast<Out>(v);
}

// V consecutive elements at p[row], row a multiple of V, p 16-byte aligned: one access of V * sizeof(T) <= 16 bytes
template <typename T, int V>
__device__ __forceinline__ void load_vec(const void* p, int64_t row, T (&v)[V])
{
  const T* s = static_cast<const T*>(p) + row;
  if constexpr (sizeof(v) == 16) {
    const int4 q = ld_nc_v4(s);
    memcpy(&v[0], &q, 16);
  } else if constexpr (sizeof(v) == 8) {
    const uint2 q = *reinterpret_cast<const uint2*>(s);
    memcpy(&v[0], &q, 8);
  } else if constexpr (sizeof(v) == 4) {
    const uint32_t q = *reinterpret_cast<const uint32_t*>(s);
    memcpy(&v[0], &q, 4);
  } else if constexpr (sizeof(v) == 2) {
    const uint16_t q = *reinterpret_cast<const uint16_t*>(s);
    memcpy(&v[0], &q, 2);
  } else {
    v[0] = s[0];
  }
}
template <typename T, int V>
__device__ __forceinline__ void store_vec(void* p, int64_t row, const T (&v)[V])
{
  T* d = static_cast<T*>(p) + row;
  if constexpr (sizeof(v) == 16) {
    int4 q;
    memcpy(&q, &v[0], 16);
    st_na_v4(d, q);
  } else if constexpr (sizeof(v) == 8) {
    uint2 q;
    memcpy(&q, &v[0], 8);
    *reinterpret_cast<uint2*>(d) = q;
  } else if constexpr (sizeof(v) == 4) {
    uint32_t q;
    memcpy(&q, &v[0], 4);
    *reinterpret_cast<uint32_t*>(d) = q;
  } else if constexpr (sizeof(v) == 2) {
    uint16_t q;
    memcpy(&q, &v[0], 2);
    *reinterpret_cast<uint16_t*>(d) = q;
  } else {
    d[0] = v[0];
  }
}

// the output mask word of rows [r0, r0 + 32): the input's bits, those past n cleared
__device__ __forceinline__ uint32_t out_word(const args& a, int64_t r0)
{
  uint32_t w     = load_mask_word_unaligned(a.mask, a.bit + r0, a.last_word);
  const int64_t rows = a.n - r0;
  if (rows < 32) w &= (1u << rows) - 1u;
  return w;
}

template <typename F, typename C, typename In, typename Out>
__global__ void __launch_bounds__(256) unary_kernel(args a)
{
  const int lane      = (int)lane_id();
  const int64_t warp  = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n     = a.n;
  const F f{};

  if constexpr (!std::is_same_v<In, rt> && !std::is_same_v<Out, rt>) {
    if (a.fast) {
      constexpr int V = 16 / (sizeof(In) > sizeof(Out) ? sizeof(In) : sizeof(Out));
      for (int64_t t = warp; t * 32 * V < n; t += warps) {
        const int64_t base = t * 32 * V, row0 = base + (int64_t)lane * V;
        const bool full = base + 32 * V <= n;
        In x[V];
        if (full) {
          load_vec<In, V>(a.in, row0, x);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) x[k] = row0 + k < n ? static_cast<const In*>(a.in)[row0 + k] : In(0);
        }
        Out r[V];
#pragma unroll
        for (int k = 0; k < V; ++k) r[k] = static_cast<Out>(f(static_cast<C>(x[k]), a));
        if (a.fold >= 0 && a.mask && row0 < n) {  // V divides 32: the lane's rows share one mask word
          const uint32_t w = load_mask_word_unaligned(a.mask, a.bit + (row0 & ~int64_t(31)), a.last_word) >> (row0 & 31);
#pragma unroll
          for (int k = 0; k < V; ++k)
            if (!((w >> k) & 1u)) r[k] = static_cast<Out>(a.fold);
        }
        if (full) {
          store_vec<Out, V>(a.out, row0, r);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k)
            if (row0 + k < n) static_cast<Out*>(a.out)[row0 + k] = r[k];
        }
        if (a.out_mask && lane < V && base + 32 * lane < n) {
          const int64_t r0 = base + 32 * lane;
          a.out_mask[r0 >> 5] = out_word(a, r0);
        }
      }
      return;
    }
  }

  for (int64_t g = warp; g * 32 < n; g += warps) {
    const int64_t r0 = g * 32, row = r0 + lane;
    if (row < n) {
      auto v = f(load_one<C, In>(a, row), a);
      if (a.fold >= 0 && a.mask && !((load_mask_word_unaligned(a.mask, a.bit + r0, a.last_word) >> lane) & 1u))
        v = static_cast<decltype(v)>(a.fold);
      store_one<Out>(a, row, v);
    }
    if (a.out_mask && lane == 0) a.out_mask[g] = out_word(a, r0);
  }
}

template <typename F, typename C, typename In, typename Out>
void launch(const args& a, cudaStream_t stream)
{
  int64_t rows_per_warp = 32;
  if constexpr (!std::is_same_v<In, rt> && !std::is_same_v<Out, rt>)
    if (a.fast) rows_per_warp = 32 * (16 / (int64_t)std::max(sizeof(In), sizeof(Out)));
  B2_LAUNCH((unary_kernel<F, C, In, Out>), binop::grid_for((a.n + rows_per_warp - 1) / rows_per_warp), 256, 0, stream, a);
}

}  // namespace unary
}  // namespace b2

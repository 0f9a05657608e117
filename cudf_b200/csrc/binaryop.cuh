// binaryop.cuh — the streaming kernel of cudf::binary_operation (binaryop.cu), instantiated per operator family in
// binaryop_{arith,math,bits,compare,logical}.cu so that the five files compile in parallel.
//
// binop_kernel<OP, C> computes out[i] = Out(op(C(lhs[i]), C(rhs[i]))) for one operator and one compute type C; the operand and
// output element types are warp-uniform runtime parameters (a switch on load and store). One pass writes the values, the output
// mask words and the null count:
//  - generic path: a warp covers 32 consecutive rows per step, one row per lane; the output mask word is one __ballot_sync of
//    the rows' validity (the AND of the operands' validity, or the null-aware operator's own rule);
//  - fast path (not null-aware, both operands of type C, output of type C or BOOL8 for a comparison / logical operator, column
//    operands 16-byte aligned): a lane owns 16 / sizeof(C) consecutive rows, read and written with vector accesses, and the
//    warp's mask words are the AND of the operands' mask words, one per lane.
// The null count accumulates into the column's `pending` counter (one atomic per warp), so the call stays stream-ordered.
//
// C is the host's choice (binaryop.cu: kernel_type): std::common_type of (out, lhs, rhs) with integer types narrower than 32
// bits replaced by int32, which is what C++ computes in after integral promotion. SHIFT_RIGHT_UNSIGNED alone keeps int8 /
// int16, because it converts to the unsigned type of C's own width before shifting.
#pragma once
#include "common.cuh"
#include "device_utils.cuh"

#include <cmath>
#include <limits>
#include <type_traits>

namespace b2 {
namespace binop {

struct operand {
  const void* data;       // row 0 of the view (offset applied), or the scalar's value
  const uint32_t* mask;   // nullptr: every row valid
  int64_t bit;            // bit of row 0 in mask (the view's offset)
  int64_t last_word;      // last mask word holding a bit of the view
  int32_t type;           // storage type id (chrono ids are mapped to their integers)
  bool scalar;
  bool valid;             // the scalar's validity
};
struct result {
  void* data;
  uint32_t* mask;             // nullptr: the output has no mask
  int32_t type;               // storage type id
  unsigned long long* nulls;  // the column's pending null count
};
struct args {
  operand a, b;
  result o;
  int64_t n;
  bool fast;
};

// the family entry points (binaryop_*.cu): launch binop_kernel<op, ctype>
void launch_arith(int op, int32_t ctype, const args& a, cudaStream_t stream);
void launch_math(int op, int32_t ctype, const args& a, cudaStream_t stream);
void launch_bits(int op, int32_t ctype, const args& a, cudaStream_t stream);
void launch_compare(int op, int32_t ctype, const args& a, cudaStream_t stream);
void launch_logical(int op, int32_t ctype, const args& a, cudaStream_t stream);

__host__ __device__ constexpr bool is_null_aware(int op)
{
  return op == B2_BINOP_NULL_EQUALS || op == B2_BINOP_NULL_NOT_EQUALS || op == B2_BINOP_NULL_MAX || op == B2_BINOP_NULL_MIN ||
         op == B2_BINOP_NULL_LOGICAL_AND || op == B2_BINOP_NULL_LOGICAL_OR;
}
// operators whose result is BOOL8 (the output type must be BOOL8)
__host__ __device__ constexpr bool is_bool_op(int op)
{
  return (op >= B2_BINOP_LOGICAL_AND && op <= B2_BINOP_NULL_NOT_EQUALS) || op == B2_BINOP_NULL_LOGICAL_AND ||
         op == B2_BINOP_NULL_LOGICAL_OR;
}
// operators defined on integers only (a float compute type has no result)
__host__ __device__ constexpr bool is_integer_op(int op)
{
  return op == B2_BINOP_INT_POW || (op >= B2_BINOP_SHIFT_LEFT && op <= B2_BINOP_BITWISE_XOR);
}

template <typename T>
__device__ __forceinline__ T load_as(const void* p, int32_t type, int64_t i)
{
  switch (type) {
    case B2_INT8: return static_cast<T>(static_cast<const int8_t*>(p)[i]);
    case B2_INT16: return static_cast<T>(static_cast<const int16_t*>(p)[i]);
    case B2_INT32: return static_cast<T>(static_cast<const int32_t*>(p)[i]);
    case B2_INT64: return static_cast<T>(static_cast<const int64_t*>(p)[i]);
    case B2_UINT8: return static_cast<T>(static_cast<const uint8_t*>(p)[i]);
    case B2_UINT16: return static_cast<T>(static_cast<const uint16_t*>(p)[i]);
    case B2_UINT32: return static_cast<T>(static_cast<const uint32_t*>(p)[i]);
    case B2_UINT64: return static_cast<T>(static_cast<const uint64_t*>(p)[i]);
    case B2_FLOAT32: return static_cast<T>(static_cast<const float*>(p)[i]);
    case B2_FLOAT64: return static_cast<T>(static_cast<const double*>(p)[i]);
    default: return static_cast<T>(static_cast<const uint8_t*>(p)[i] != 0);  // BOOL8
  }
}

template <typename R>
__device__ __forceinline__ void store_as(void* p, int32_t type, int64_t i, R v)
{
  switch (type) {
    case B2_INT8: static_cast<int8_t*>(p)[i] = static_cast<int8_t>(v); break;
    case B2_INT16: static_cast<int16_t*>(p)[i] = static_cast<int16_t>(v); break;
    case B2_INT32: static_cast<int32_t*>(p)[i] = static_cast<int32_t>(v); break;
    case B2_INT64: static_cast<int64_t*>(p)[i] = static_cast<int64_t>(v); break;
    case B2_UINT8: static_cast<uint8_t*>(p)[i] = static_cast<uint8_t>(v); break;
    case B2_UINT16: static_cast<uint16_t*>(p)[i] = static_cast<uint16_t>(v); break;
    case B2_UINT32: static_cast<uint32_t*>(p)[i] = static_cast<uint32_t>(v); break;
    case B2_UINT64: static_cast<uint64_t*>(p)[i] = static_cast<uint64_t>(v); break;
    case B2_FLOAT32: static_cast<float*>(p)[i] = static_cast<float>(v); break;
    case B2_FLOAT64: static_cast<double*>(p)[i] = static_cast<double>(v); break;
    default: static_cast<uint8_t*>(p)[i] = static_cast<bool>(v) ? 1 : 0; break;  // BOOL8
  }
}

// two's-complement wrap for signed integers (the reference relies on it; here it is defined behaviour)
template <typename C>
__device__ __forceinline__ C wrap_add(C x, C y)
{
  if constexpr (std::is_integral_v<C>) {
    using U = std::make_unsigned_t<C>;
    return static_cast<C>(static_cast<U>(static_cast<U>(x) + static_cast<U>(y)));
  } else {
    return x + y;
  }
}
template <typename C>
__device__ __forceinline__ C wrap_sub(C x, C y)
{
  if constexpr (std::is_integral_v<C>) {
    using U = std::make_unsigned_t<C>;
    return static_cast<C>(static_cast<U>(static_cast<U>(x) - static_cast<U>(y)));
  } else {
    return x - y;
  }
}
template <typename C>
__device__ __forceinline__ C wrap_mul(C x, C y)
{
  if constexpr (std::is_integral_v<C>) {
    using U = std::make_unsigned_t<C>;
    return static_cast<C>(static_cast<U>(static_cast<U>(x) * static_cast<U>(y)));
  } else {
    return x * y;
  }
}

// integer division by zero and INT_MIN / -1 have no defined value; dividing by 1 instead keeps them from trapping where
// integer division traps (a CPU build of the kernels)
template <typename C>
__device__ __forceinline__ C divisor(C x, C y)
{
  if constexpr (std::is_signed_v<C>) return (y == 0 || (y == C(-1) && x == std::numeric_limits<C>::min())) ? C(1) : y;
  else return y == 0 ? C(1) : y;
}

// op(x, y) of a value operator in C (the null-aware ones are in row_op); the result type is the C++ one
template <int OP, typename C>
__device__ __forceinline__ auto value_op(C x, C y)
{
  constexpr bool INT = std::is_integral_v<C>;
  if constexpr (INT && (OP == B2_BINOP_DIV || OP == B2_BINOP_FLOOR_DIV || OP == B2_BINOP_MOD || OP == B2_BINOP_PMOD ||
                        OP == B2_BINOP_PYMOD))
    y = divisor(x, y);
  if constexpr (OP == B2_BINOP_ADD) return wrap_add(x, y);
  else if constexpr (OP == B2_BINOP_SUB) return wrap_sub(x, y);
  else if constexpr (OP == B2_BINOP_MUL) return wrap_mul(x, y);
  else if constexpr (OP == B2_BINOP_DIV) return x / y;
  else if constexpr (OP == B2_BINOP_TRUE_DIV) return static_cast<double>(x) / static_cast<double>(y);
  else if constexpr (OP == B2_BINOP_FLOOR_DIV) {
    if constexpr (INT && std::is_signed_v<C>) {
      const C q = x / y;
      return static_cast<C>(q - static_cast<C>((x % y) != 0 && (x ^ y) < 0));
    } else if constexpr (INT) {
      return x / y;
    } else {
      return std::floor(x / y);  // floorf for float
    }
  } else if constexpr (OP == B2_BINOP_MOD) {
    if constexpr (INT) return x % y;
    else return std::fmod(x, y);
  } else if constexpr (OP == B2_BINOP_PMOD) {
    if constexpr (INT) {
      C r = x % y;
      if constexpr (std::is_signed_v<C>)
        if (r < 0) r = wrap_add(r, y) % y;
      return r;
    } else {
      C r = std::fmod(x, y);
      if (r < 0) r = std::fmod(r + y, y);
      return r;
    }
  } else if constexpr (OP == B2_BINOP_PYMOD) {
    if constexpr (INT) {
      return wrap_add(static_cast<C>(x % y), y) % y;
    } else {
      const double a = static_cast<double>(x), b = static_cast<double>(y);
      return fmod(fmod(a, b) + b, b);
    }
  } else if constexpr (OP == B2_BINOP_POW) return pow(static_cast<double>(x), static_cast<double>(y));
  else if constexpr (OP == B2_BINOP_INT_POW) {
    // exponentiation by squaring in C; a negative exponent gives 0
    using U = std::make_unsigned_t<C>;
    if constexpr (std::is_signed_v<C>)
      if (y < 0) return C(0);
    if (y == 0) return C(1);
    if (x == 0) return C(0);
    U b = static_cast<U>(x), e = static_cast<U>(y), extra = 1;
    while (e > 1) {
      if (e & 1) extra = static_cast<U>(extra * b);
      e >>= 1;
      b = static_cast<U>(b * b);
    }
    return static_cast<C>(static_cast<U>(b * extra));
  } else if constexpr (OP == B2_BINOP_LOG_BASE) return log(static_cast<double>(x)) / log(static_cast<double>(y));
  else if constexpr (OP == B2_BINOP_ATAN2) return atan2(static_cast<double>(x), static_cast<double>(y));
  else if constexpr (OP == B2_BINOP_SHIFT_LEFT) {
    using U = std::make_unsigned_t<C>;
    return static_cast<C>(static_cast<U>(static_cast<U>(x) << y));
  } else if constexpr (OP == B2_BINOP_SHIFT_RIGHT) return static_cast<C>(x >> y);
  else if constexpr (OP == B2_BINOP_SHIFT_RIGHT_UNSIGNED) return static_cast<std::make_unsigned_t<C>>(x) >> y;
  else if constexpr (OP == B2_BINOP_BITWISE_AND) return static_cast<C>(x & y);
  else if constexpr (OP == B2_BINOP_BITWISE_OR) return static_cast<C>(x | y);
  else if constexpr (OP == B2_BINOP_BITWISE_XOR) return static_cast<C>(x ^ y);
  else if constexpr (OP == B2_BINOP_LOGICAL_AND) return static_cast<bool>(x) && static_cast<bool>(y);
  else if constexpr (OP == B2_BINOP_LOGICAL_OR) return static_cast<bool>(x) || static_cast<bool>(y);
  else if constexpr (OP == B2_BINOP_EQUAL) return x == y;
  else if constexpr (OP == B2_BINOP_NOT_EQUAL) return x != y;
  else if constexpr (OP == B2_BINOP_LESS) return x < y;
  else if constexpr (OP == B2_BINOP_GREATER) return x > y;
  else if constexpr (OP == B2_BINOP_LESS_EQUAL) return x <= y;
  else return x >= y;  // GREATER_EQUAL
}

// one row: the value, and in `valid` the output validity given the operands' (operation.cuh's rules for the null-aware ops)
template <int OP, typename C>
__device__ __forceinline__ auto row_op(C x, C y, bool lv, bool rv, bool& valid)
{
  if constexpr (OP == B2_BINOP_NULL_EQUALS || OP == B2_BINOP_NULL_NOT_EQUALS) {
    valid = true;
    const bool eq = (lv && rv) ? (x == y) : (!lv && !rv);
    return OP == B2_BINOP_NULL_EQUALS ? eq : !eq;
  } else if constexpr (OP == B2_BINOP_NULL_MAX || OP == B2_BINOP_NULL_MIN) {
    valid = lv || rv;
    if (lv && rv) return OP == B2_BINOP_NULL_MAX ? (x > y ? x : y) : (x < y ? x : y);
    return lv ? x : y;
  } else if constexpr (OP == B2_BINOP_NULL_LOGICAL_AND) {
    const bool lf = lv && !x, rf = rv && !y;
    valid = lf || rf || (lv && rv);
    return lv && rv && !lf && !rf;
  } else if constexpr (OP == B2_BINOP_NULL_LOGICAL_OR) {
    const bool lt = lv && static_cast<bool>(x), rt = rv && static_cast<bool>(y);
    valid = lt || rt || (lv && rv);
    return lt || rt;
  } else {
    valid = lv && rv;
    return value_op<OP, C>(x, y);
  }
}

template <typename C>
__device__ __forceinline__ void load_vec(const void* p, int64_t row, C (&v)[16 / sizeof(C)])
{
  const int4 q = ld_nc_v4(static_cast<const C*>(p) + row);
  memcpy(&v[0], &q, 16);
}

template <int OP, typename C>
__global__ void __launch_bounds__(256) binop_kernel(operand a, operand b, result o, int64_t n, bool fast)
{
  const int lane      = (int)lane_id();
  const int64_t warp  = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const C xs = a.scalar ? load_as<C>(a.data, a.type, 0) : C(0);
  const C ys = b.scalar ? load_as<C>(b.data, b.type, 0) : C(0);
  unsigned long long nulls = 0;

  if constexpr (!is_null_aware(OP)) {
    if (fast) {
      constexpr int V = 16 / sizeof(C);
      using out_t = std::conditional_t<is_bool_op(OP), uint8_t, C>;
      for (int64_t t = warp; t * 32 * V < n; t += warps) {
        const int64_t base = t * 32 * V, row0 = base + (int64_t)lane * V;
        const bool full = base + 32 * V <= n;
        C x[V], y[V];
        if (full) {
          if (!a.scalar) load_vec<C>(a.data, row0, x);
          if (!b.scalar) load_vec<C>(b.data, row0, y);
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k) {
            x[k] = (!a.scalar && row0 + k < n) ? static_cast<const C*>(a.data)[row0 + k] : C(0);
            y[k] = (!b.scalar && row0 + k < n) ? static_cast<const C*>(b.data)[row0 + k] : C(0);
          }
        }
        out_t r[V];
#pragma unroll
        for (int k = 0; k < V; ++k)
          r[k] = static_cast<out_t>(value_op<OP, C>(a.scalar ? xs : x[k], b.scalar ? ys : y[k]));
        out_t* out = static_cast<out_t*>(o.data) + row0;
        if (full) {
          if constexpr (sizeof(r) == 16) {
            int4 q;
            memcpy(&q, r, 16);
            st_na_v4(out, q);
          } else if constexpr (sizeof(r) == 8) {
            uint2 q;
            memcpy(&q, r, 8);
            *reinterpret_cast<uint2*>(out) = q;
          } else if constexpr (sizeof(r) == 4) {
            uint32_t q;
            memcpy(&q, r, 4);
            *reinterpret_cast<uint32_t*>(out) = q;
          } else {
            uint16_t q;
            memcpy(&q, r, 2);
            *reinterpret_cast<uint16_t*>(out) = q;
          }
        } else {
#pragma unroll
          for (int k = 0; k < V; ++k)
            if (row0 + k < n) out[k] = r[k];
        }
        // the tile's V mask words: lane w writes word w
        if (o.mask && lane < V && base + 32 * lane < n) {
          const int64_t r0 = base + 32 * lane;
          uint32_t w = ~0u;
          if (a.mask) w &= load_mask_word_unaligned(a.mask, a.bit + r0, a.last_word);
          if (b.mask) w &= load_mask_word_unaligned(b.mask, b.bit + r0, b.last_word);
          const int rows = (int)min((int64_t)32, n - r0);
          if (rows < 32) w &= (1u << rows) - 1u;
          o.mask[r0 >> 5] = w;
          nulls += (unsigned long long)(rows - __popc(w));
        }
      }
      if (o.mask) {
        nulls = warp_sum(nulls);
        if (lane == 0 && nulls) atomicAdd(o.nulls, nulls);
      }
      return;
    }
  }

  for (int64_t g = warp; g * 32 < n; g += warps) {
    const int64_t r0 = g * 32, row = r0 + lane;
    const bool in = row < n;
    const C x = a.scalar ? xs : (in ? load_as<C>(a.data, a.type, row) : C(0));
    const C y = b.scalar ? ys : (in ? load_as<C>(b.data, b.type, row) : C(0));
    bool lv = a.scalar ? a.valid : true, rv = b.scalar ? b.valid : true;
    if (!a.scalar && a.mask) lv = (load_mask_word_unaligned(a.mask, a.bit + r0, a.last_word) >> lane) & 1u;
    if (!b.scalar && b.mask) rv = (load_mask_word_unaligned(b.mask, b.bit + r0, b.last_word) >> lane) & 1u;
    bool valid;
    const auto v = row_op<OP, C>(x, y, lv, rv, valid);
    if (in) store_as(o.data, o.type, row, v);
    if (o.mask) {
      const uint32_t w = __ballot_sync(0xffffffffu, in && valid);
      if (lane == 0) {
        o.mask[g] = w;
        nulls += (unsigned long long)(min((int64_t)32, n - r0) - __popc(w));
      }
    }
  }
  if (o.mask && lane == 0 && nulls) atomicAdd(o.nulls, nulls);
}

inline int grid_for(int64_t warps_of_work)
{
  return (int)std::max<int64_t>(1, std::min<int64_t>((warps_of_work + 7) / 8, (int64_t)num_sms() * 16));
}

template <int OP, typename C>
void launch(const args& a, cudaStream_t stream)
{
  const int64_t rows_per_warp = a.fast ? 32 * (16 / (int64_t)sizeof(C)) : 32;
  B2_LAUNCH((binop_kernel<OP, C>), grid_for((a.n + rows_per_warp - 1) / rows_per_warp), 256, 0, stream, a.a, a.b, a.o, a.n, a.fast);
}

// binop_kernel<OP, C> for a compute type id; an id the family does not instantiate is an internal error
template <int OP>
void launch_ctype(int32_t ctype, const args& a, cudaStream_t stream)
{
  if constexpr (OP == B2_BINOP_SHIFT_RIGHT_UNSIGNED) {
    if (ctype == B2_INT8) return launch<OP, int8_t>(a, stream);
    if (ctype == B2_INT16) return launch<OP, int16_t>(a, stream);
  }
  switch (ctype) {
    case B2_INT32: return launch<OP, int32_t>(a, stream);
    case B2_UINT32: return launch<OP, uint32_t>(a, stream);
    case B2_INT64: return launch<OP, int64_t>(a, stream);
    case B2_UINT64: return launch<OP, uint64_t>(a, stream);
    default: break;
  }
  if constexpr (!is_integer_op(OP)) {
    if (ctype == B2_FLOAT32) return launch<OP, float>(a, stream);
    if (ctype == B2_FLOAT64) return launch<OP, double>(a, stream);
  }
  B2_FAIL(B2_ERR_LOGIC, "binary_operation: no kernel for this compute type");
}

}  // namespace binop
}  // namespace b2

// replace.cuh — the kernels of cudf::replace_nulls, replace_nans, find_and_replace_all, clamp and normalize_nans_and_zeros
// (replace.cu).
//
// replace_kernel<M, T> is one streaming pass per call for every form but the preceding / following fill. It writes the values,
// the output mask words and, when asked, the null count (into the column's pending counter, one atomic per warp). T is the
// storage width's unsigned type where the form only selects bits (replace_nulls), and the element type where it compares
// (replace_nans, clamp, the lookup of find_and_replace_all, normalize_nans_and_zeros).
//  - generic path: a warp covers 32 consecutive rows per step, one row per lane; the mask word is one __ballot_sync;
//  - vector path (input, output and a replacement column 16-byte aligned): a lane owns V = 16 / sizeof(T) consecutive rows read
//    and written with 16-byte accesses; the V validity bits of 32 / V lanes are OR-ed into one mask word by shuffles.
// The lookup stages its sorted table (keys as unsigned bit patterns, each with its position in the old values) in shared
// memory when it fits, and otherwise searches it in global memory; a row takes the lower_bound of its key.
//
// fill_kernel<T, FOLLOW> is the preceding / following fill in one pass: a single-pass decoupled look-back (the 16-byte records
// of device_utils.cuh, tiles in ticket order as in compact.cuh) over the index of the last valid row before each tile (-1 for
// none; FOLLOWING: the first valid row after it, n for none, with ticket t on tile T-1-t). A tile publishes its aggregate as
// soon as it has read its mask words. Inside a warp a row's source is the nearest set bit of its mask word at or before
// (after) the row; words without one take the carried index.
#pragma once
#include "unary.cuh"

#include <cmath>
#include <limits>
#include <type_traits>

namespace b2 {
namespace repl {

enum mode : int { NULLS = 0, NANS = 1, CLAMP = 2, LOOKUP = 3, NORMALIZE = 4 };

struct side {
  const void* data;      // row 0 of the view (offset applied), or the scalar's value; nullptr: no such operand
  const uint32_t* mask;  // nullptr: every row valid
  int64_t bit;           // bit of row 0 in mask (the view's offset)
  int64_t last_word;     // last mask word holding a bit of the view
  const int32_t* scalar_valid;  // a scalar's validity flag on the device; nullptr: a column
};

struct args {
  side in;
  side repl;                   // NULLS / NANS: the replacement; LOOKUP: the new values (indexed by position)
  const void* lo;              // CLAMP: the scalars' values; lo / hi nullptr when that bound is null
  const void* lo_r;
  const void* hi;
  const void* hi_r;
  const void* keys;            // LOOKUP: k sorted keys and their positions
  const int32_t* pos;
  int32_t k;
  bool staged;                 // LOOKUP: the table is copied to shared memory first
  void* out;
  uint32_t* out_mask;          // nullptr: the output has no mask
  unsigned long long* nulls;   // nullptr: the null count is known without counting
  int64_t n;
  bool fast;
};

// the shared-memory budget of a staged lookup table (no opt-in attribute needed)
constexpr size_t LOOKUP_SMEM = 48 * 1024;
inline size_t lookup_smem_bytes(int32_t k, int width) { return ((size_t)k * 4 + 15) / 16 * 16 + (size_t)k * width; }

template <typename T> using bits_t = typename key_bits<sizeof(T)>::type;

// the key of a value: its bit pattern, with -0.0 as +0.0 (a NaN key is kept; no non-NaN row has its pattern)
template <typename T>
__host__ __device__ __forceinline__ bits_t<T> key_of(T x)
{
  if constexpr (std::is_floating_point_v<T>)
    if (x == T(0)) x = T(0);
  bits_t<T> u;
  memcpy(&u, &x, sizeof(T));
  return u;
}

__device__ __forceinline__ bool side_valid(const side& s, int64_t i)
{
  return s.mask == nullptr || ((s.mask[(s.bit + i) >> 5] >> ((s.bit + i) & 31)) & 1u);
}

// validity bits of rows [r, r + 32) of a column operand (bits past the view are undefined)
__device__ __forceinline__ uint32_t side_bits(const side& s, int64_t r)
{
  return s.mask ? load_mask_word_unaligned(s.mask, s.bit + r, s.last_word) : ~0u;
}

template <typename T>
struct consts {
  T y;      // a scalar replacement
  bool yv;
  T lo, lo_r, hi, hi_r;
  bool has_lo, has_hi;
};

template <typename T>
__device__ __forceinline__ T load_scalar(const void* p)
{
  return p ? *static_cast<const T*>(p) : T(0);
}

// one row: x with validity xv, the replacement y with validity yv (NULLS / NANS); the output value and, in ov, its validity
template <int M, typename T>
__device__ __forceinline__ T apply(const args& a, const consts<T>& c, const bits_t<T>* keys, const int32_t* pos, T x, bool xv, T y,
                                   bool yv, bool& ov)
{
  if constexpr (M == NULLS) {
    ov = xv || yv;
    return xv ? x : y;
  } else if constexpr (M == NANS) {
    const bool nan = xv && std::isnan(x);
    ov = nan ? yv : xv;
    return nan ? y : x;
  } else if constexpr (M == CLAMP) {
    ov = xv;
    if (c.has_lo && x < c.lo) return c.lo_r;
    if (c.has_hi && x > c.hi) return c.hi_r;
    return x;
  } else if constexpr (M == LOOKUP) {
    ov = xv;
    if constexpr (std::is_floating_point_v<T>)
      if (std::isnan(x)) return x;
    if (!xv) return x;
    const bits_t<T> key = key_of(x);
    int32_t lo = 0, hi = a.k;
    while (lo < hi) {
      const int32_t mid = (lo + hi) >> 1;
      if (keys[mid] < key) lo = mid + 1;
      else hi = mid;
    }
    if (lo < a.k && keys[lo] == key) {
      const int32_t p = pos[lo];
      ov = side_valid(a.repl, p);
      return static_cast<const T*>(a.repl.data)[p];
    }
    return x;
  } else {  // NORMALIZE
    ov = xv;
    if (std::isnan(x)) return std::numeric_limits<T>::quiet_NaN();
    return x == T(0) ? T(0) : x;
  }
}

template <int M, typename T>
__global__ void __launch_bounds__(256) replace_kernel(args a)
{
  using U = bits_t<T>;
  const U* keys      = static_cast<const U*>(a.keys);
  const int32_t* pos = a.pos;
  if constexpr (M == LOOKUP) {
    if (a.staged) {
      B2_DYNAMIC_SMEM(smem);
      int32_t* sp = reinterpret_cast<int32_t*>(smem);
      U* sk       = reinterpret_cast<U*>(smem + ((size_t)a.k * 4 + 15) / 16 * 16);
      for (int i = threadIdx.x; i < a.k; i += blockDim.x) {
        sp[i] = a.pos[i];
        sk[i] = keys[i];
      }
      __syncthreads();
      keys = sk;
      pos  = sp;
    }
  }
  consts<T> c;
  const bool repl_col = (M == NULLS || M == NANS) && a.repl.scalar_valid == nullptr;
  c.y    = repl_col ? T(0) : load_scalar<T>(a.repl.data);
  c.yv   = repl_col ? false : (a.repl.scalar_valid && *a.repl.scalar_valid != 0);
  c.lo   = load_scalar<T>(a.lo);
  c.lo_r = load_scalar<T>(a.lo_r);
  c.hi   = load_scalar<T>(a.hi);
  c.hi_r = load_scalar<T>(a.hi_r);
  c.has_lo = a.lo != nullptr;
  c.has_hi = a.hi != nullptr;

  const int lane      = (int)lane_id();
  const int64_t warp  = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n     = a.n;
  const T* in         = static_cast<const T*>(a.in.data);
  const T* rp         = static_cast<const T*>(a.repl.data);
  T* out              = static_cast<T*>(a.out);
  unsigned long long nulls = 0;

  if (a.fast) {
    constexpr int V = 16 / sizeof(T), G = 32 / V;
    for (int64_t t = warp; t * 32 * V < n; t += warps) {
      const int64_t base = t * 32 * V, row0 = base + (int64_t)lane * V;
      const bool full = base + 32 * V <= n;
      T x[V], y[V];
      if (full) {
        unary::load_vec<T, V>(in, row0, x);
        if (repl_col) unary::load_vec<T, V>(rp, row0, y);
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k) {
          x[k] = row0 + k < n ? in[row0 + k] : T(0);
          y[k] = (repl_col && row0 + k < n) ? rp[row0 + k] : T(0);
        }
      }
      // V divides 32: the lane's rows share one mask word
      uint32_t xb = 0, yb = c.yv ? ~0u : 0u;
      if (row0 < n) {
        xb = side_bits(a.in, row0 & ~int64_t(31)) >> (row0 & 31);
        if (repl_col) yb = side_bits(a.repl, row0 & ~int64_t(31)) >> (row0 & 31);
      }
      T r[V];
      uint32_t ob = 0;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        bool ov;
        r[k] = apply<M, T>(a, c, keys, pos, x[k], (xb >> k) & 1u, repl_col ? y[k] : c.y, (yb >> k) & 1u, ov);
        ob |= (uint32_t)(ov && row0 + k < n) << k;
      }
      if (full) {
        unary::store_vec<T, V>(out, row0, r);
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k)
          if (row0 + k < n) out[row0 + k] = r[k];
      }
      if (a.out_mask) {
        uint32_t w = ob << ((lane % G) * V);
#pragma unroll
        for (int o = 1; o < G; o <<= 1) w |= __shfl_xor_sync(0xffffffffu, w, o);
        const int64_t r0 = base + 32 * (lane / G);
        if (lane % G == 0 && r0 < n) {
          a.out_mask[r0 >> 5] = w;
          nulls += (unsigned long long)(min((int64_t)32, n - r0) - __popc(w));
        }
      }
    }
  } else {
    for (int64_t g = warp; g * 32 < n; g += warps) {
      const int64_t r0 = g * 32, row = r0 + lane;
      const bool inside = row < n;
      const T x     = inside ? in[row] : T(0);
      const bool xv = inside && side_valid(a.in, row);
      const T y     = (repl_col && inside) ? rp[row] : c.y;
      const bool yv = repl_col ? (inside && side_valid(a.repl, row)) : c.yv;
      bool ov;
      const T r = apply<M, T>(a, c, keys, pos, x, xv, y, yv, ov);
      if (inside) out[row] = r;
      if (a.out_mask) {
        const uint32_t w = __ballot_sync(0xffffffffu, inside && ov);
        if (lane == 0) {
          a.out_mask[g] = w;
          nulls += (unsigned long long)(min((int64_t)32, n - r0) - __popc(w));
        }
      }
    }
  }
  if (a.nulls) {
    nulls = warp_sum(nulls);
    if (lane == 0 && nulls) atomicAdd(a.nulls, nulls);
  }
}

template <int M, typename T>
void launch(const args& a, size_t smem, cudaStream_t stream)
{
  const int64_t rows_per_warp = a.fast ? 32 * (16 / (int64_t)sizeof(T)) : 32;
  B2_LAUNCH((replace_kernel<M, T>), binop::grid_for((a.n + rows_per_warp - 1) / rows_per_warp), 256, smem, stream, a);
}

// ---- find_and_replace_all: the lookup table --------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) lookup_keys_kernel(const T* old, int32_t k, bits_t<T>* keys)
{
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) keys[i] = key_of(old[i]);
}
template <typename U>
__global__ void __launch_bounds__(256) lookup_table_kernel(const U* keys, const int32_t* order, int32_t k, U* sorted, int32_t* pos)
{
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) {
    const int32_t p = order[i];
    sorted[i] = keys[p];
    pos[i]    = p;
  }
}

// ---- preceding / following fill ---------------------------------------------------------------------------------------
constexpr int FL_THREADS  = 256;
constexpr int FL_NW       = FL_THREADS / 32;
constexpr int64_t FL_TILE = (int64_t)FL_NW * 32 * 32;  // a warp covers 32 mask words: 8192 rows per tile

struct fill_args {
  const void* in;        // row 0 of the view
  const uint32_t* mask;  // the input's mask (the input has nulls)
  int64_t bit, last_word;
  void* out;
  uint32_t* out_mask;
  unsigned long long* nulls;
  int64_t n;
};

template <typename T, bool FOLLOW>
__global__ void __launch_bounds__(FL_THREADS) fill_kernel(fill_args a, scan_state st, int64_t ntiles)
{
  __shared__ int64_t s_wagg[FL_NW];
  __shared__ int64_t s_carry;
  __shared__ uint32_t s_ticket;
  if (threadIdx.x == 0) s_ticket = atomicAdd(st.ticket, 1u);  // tiles start in ticket order: the look-back cannot wait on a
  __syncthreads();                                              // tile that has not been scheduled
  const int64_t t    = s_ticket;
  const int64_t tile = FOLLOW ? ntiles - 1 - t : t;
  const int64_t n    = a.n;
  const int64_t NONE = FOLLOW ? n : -1;
  auto comb = [](int64_t x, int64_t y) { return FOLLOW ? (x < y ? x : y) : (x > y ? x : y); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wbase = tile * FL_TILE + (int64_t)warp * 32 * 32;

  // lane j: the warp's mask word j, rows past n invalid; its last (first) valid row; the scan over words in fill order
  uint32_t word = 0;
  {
    const int64_t r0 = wbase + 32 * lane;
    if (r0 < n) {
      word = load_mask_word_unaligned(a.mask, a.bit + r0, a.last_word);
      if (n - r0 < 32) word &= (1u << (n - r0)) - 1u;
    }
  }
  int64_t inc = NONE;
  if (word) inc = wbase + 32 * lane + (FOLLOW ? __ffs((int)word) - 1 : 31 - __clz((int)word));
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int src = FOLLOW ? lane + o : lane - o;
    const int64_t v = __shfl_sync(0xffffffffu, inc, src & 31);
    if (src >= 0 && src < 32) inc = comb(inc, v);
  }
  int64_t excl;  // the nearest valid row of the warp's earlier words (in fill order)
  {
    const int src = FOLLOW ? lane + 1 : lane - 1;
    const int64_t v = __shfl_sync(0xffffffffu, inc, src & 31);
    excl = (src >= 0 && src < 32) ? v : NONE;
  }
  const int64_t wagg = __shfl_sync(0xffffffffu, inc, FOLLOW ? 0 : 31);
  if (lane == 0) s_wagg[warp] = wagg;
  __syncthreads();

  if (warp == 0) {
    int64_t tagg = NONE;
#pragma unroll
    for (int w = 0; w < FL_NW; ++w) tagg = comb(tagg, s_wagg[w]);
    int64_t carry = NONE;
    if (t == 0) {
      if (lane == 0) publish_rec<int64_t>(st.rec, 2u, tagg);
    } else {
      if (lane == 0) publish_rec<int64_t>(st.rec + t, 1u, tagg);
      int64_t base = t - 1;
      while (true) {
        // lane l reads the record at distance l; tickets before the first act as an inclusive NONE. A record settles the carry
        // when it is inclusive, or an aggregate that holds a valid row: row indices are monotone in ticket order, so the nearest
        // such record dominates every earlier one.
        const int64_t idx = base - lane;
        int64_t v = NONE;
        const uint32_t f = idx >= 0 ? read_rec<int64_t>(st.rec + idx, v) : 2u;
        const unsigned done = __ballot_sync(0xffffffffu, f == 2u || (f == 1u && v != NONE));
        const unsigned wait = __ballot_sync(0xffffffffu, f == 0u);
        const int first_done = done ? __ffs((int)done) - 1 : 32;
        const int first_wait = wait ? __ffs((int)wait) - 1 : 32;
        if (first_wait < first_done) continue;  // a needed record is not published yet: poll again (volatile loads)
        if (done) {
          carry = __shfl_sync(0xffffffffu, v, first_done);
          break;
        }
        base -= 32;
      }
      if (lane == 0) publish_rec<int64_t>(st.rec + t, 2u, comb(carry, tagg));
    }
    if (lane == 0) s_carry = carry;
  }
  __syncthreads();

  int64_t carry = s_carry;
  for (int w = 0; w < FL_NW; ++w)
    if (FOLLOW ? w > warp : w < warp) carry = comb(carry, s_wagg[w]);
  excl = comb(excl, carry);

  const T* in = static_cast<const T*>(a.in);
  T* out      = static_cast<T*>(a.out);
  const uint32_t le = lanemask_lt() | (1u << lane);
  unsigned long long nulls = 0;
#pragma unroll 4
  for (int j = 0; j < 32; ++j) {
    const int64_t r0 = wbase + 32 * j;
    if (r0 >= n) break;
    const uint32_t w     = __shfl_sync(0xffffffffu, word, j);
    const int64_t before = __shfl_sync(0xffffffffu, excl, j);
    const uint32_t m     = FOLLOW ? w & ~lanemask_lt() : w & le;
    const int64_t src    = m ? r0 + (FOLLOW ? __ffs((int)m) - 1 : 31 - __clz((int)m)) : before;
    const int64_t row    = r0 + lane;
    const bool ok        = src != NONE;
    if (row < n) out[row] = ok ? in[src] : T(0);
    const uint32_t vb = __ballot_sync(0xffffffffu, row < n && ok);
    if (lane == 0) {
      a.out_mask[r0 >> 5] = vb;
      nulls += (unsigned long long)(min((int64_t)32, n - r0) - __popc(vb));
    }
  }
  if (lane == 0 && nulls) atomicAdd(a.nulls, nulls);
}

}  // namespace repl
}  // namespace b2

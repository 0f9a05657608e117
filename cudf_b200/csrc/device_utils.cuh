// device_utils.cuh — sm_90a device helpers: cache-hinted vector loads/stores, warp primitives,
// order-preserving key twiddles, bit access (cpp/include/cudf/utilities/bit.hpp semantics).
#pragma once
#include <atomic>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

namespace b2 {

constexpr int WARP = 32;
// SMs of the current device: grid caps of the grid-stride kernels and the CTA count of the persistent ones. Queried once
// per device ordinal; 132 (H100 SXM) only if the query itself fails, in which case no kernel can launch either.
inline int num_sms()
{
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  std::atomic<int>& slot = cache[dev & 63];
  int v = slot.load(std::memory_order_relaxed);
  if (v == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    slot.store(v, std::memory_order_relaxed);
  }
  return v;
}

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ unsigned lanemask_lt()
{
#ifdef B2_EMU  // tests/emu: CPU emulation of the kernels (test infrastructure)
  return (1u << lane_id()) - 1u;
#else
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
#endif
}

// ---- bit.hpp semantics: bit i of word i/32, LSB first -----------------------------------------
__device__ __forceinline__ bool bit_is_set(const uint32_t* mask, int64_t i)
{
  return (mask[i >> 5] >> (i & 31)) & 1u;
}
__device__ __forceinline__ bool row_valid(const uint32_t* mask, int64_t i)
{
  return mask == nullptr || bit_is_set(mask, i);
}
// 32 validity bits starting at absolute bit `bit` (funnel shift of two words); bits past `end_bit`
// are undefined — callers mask them.
__device__ __forceinline__ uint32_t load_mask_word_unaligned(const uint32_t* mask, int64_t bit, int64_t last_word)
{
  int64_t w  = bit >> 5;
  int sh     = bit & 31;
  uint32_t lo = mask[w];
  if (sh == 0) return lo;
  uint32_t hi = (w + 1 <= last_word) ? mask[w + 1] : 0u;
  return __funnelshift_r(lo, hi, sh);
}

// ---- streaming global memory access (read-once data: bypass L1 allocation) --------------------
template <typename T> __device__ __forceinline__ T ld_stream(const T* p) { return __ldcs(p); }
template <typename T> __device__ __forceinline__ void st_stream(T* p, T v) { __stcs(p, v); }

__device__ __forceinline__ int4 ld_nc_v4(const void* p)
{
#ifdef B2_EMU
  return *static_cast<const int4*>(p);
#else
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
#endif
}
__device__ __forceinline__ void st_na_v4(void* p, const int4& v)
{
#ifdef B2_EMU
  *static_cast<int4*>(p) = v;
#else
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
#endif
}

// ---- warp scans / reductions ----------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T warp_inclusive_sum(T v)
{
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    T n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane_id() >= (unsigned)o) v += n;
  }
  return v;
}
template <typename T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- decoupled look-back records (scan_kernel, compact_kernel) ------------------------------------
// One 16-byte record per tile: {flag (0 nothing, 1 aggregate, 2 inclusive), pad, 8-byte value}. A 16-byte
// aligned store is observed all-or-nothing by a 16-byte load, so the look-back needs no fences.
struct scan_state {
  uint4* rec;
  uint32_t* ticket;
};
template <typename T>
__device__ __forceinline__ void publish_rec(uint4* p, uint32_t flag, T v)
{
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
#ifdef B2_EMU
  *p = make_uint4(flag, 0u, (uint32_t)bits, (uint32_t)(bits >> 32));
#else
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(flag), "r"(0u), "r"((uint32_t)bits),
               "r"((uint32_t)(bits >> 32))
               : "memory");
#endif
}
template <typename T>
__device__ __forceinline__ uint32_t read_rec(const uint4* p, T& v)
{
#ifdef B2_EMU
  const uint4 r = *p;
#else
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
#endif
  unsigned long long bits = (unsigned long long)r.z | ((unsigned long long)r.w << 32);
  memcpy(&v, &bits, sizeof(T));
  return r.x;
}

// ---- splitmix64 (SURVEY §8d generator) --------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x)
{
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// cheap 64-bit finalizer used for hash tables / hash partitioning (murmur3 fmix64)
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t k)
{
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

// inverse of mix64 (each xor-shift by 33 is an involution; the multipliers are odd): lets a kernel carry mix64(key)
// through a partition pass and recover the key afterwards
__host__ __device__ __forceinline__ uint64_t unmix64(uint64_t k)
{
  k ^= k >> 33; k *= 0x9cb4b2f8129337dbull;
  k ^= k >> 33; k *= 0x4f74430c22a54005ull;
  k ^= k >> 33;
  return k;
}

// ---- order-preserving twiddles: value -> unsigned radix key ---------------------------------------
// Integers: flip the sign bit.  Floats (sorted_order_radix.cu:41-50 + cub float ordering): -0 == +0,
// every NaN (either sign) maps to the all-ones key so NaNs sort last and tie (stable => input order).
template <typename U> struct uint_of;
template <> struct uint_of<uint8_t> { using type = uint8_t; };

template <int BYTES> struct key_bits;
template <> struct key_bits<1> { using type = uint8_t; };
template <> struct key_bits<2> { using type = uint16_t; };
template <> struct key_bits<4> { using type = uint32_t; };
template <> struct key_bits<8> { using type = uint64_t; };

enum class key_kind : int { UNSIGNED = 0, SIGNED = 1, FLOAT = 2 };

template <typename UK, key_kind K>
__device__ __forceinline__ UK twiddle_in(UK bits)
{
  constexpr UK SIGN = UK(1) << (sizeof(UK) * 8 - 1);
  if constexpr (K == key_kind::UNSIGNED) {
    return bits;
  } else if constexpr (K == key_kind::SIGNED) {
    return bits ^ SIGN;
  } else {
    // float32 / float64 bit patterns
    constexpr UK EXP = sizeof(UK) == 4 ? UK(0x7F800000u) : UK(0x7FF0000000000000ull);
    UK mag = bits & ~SIGN;
    if (mag > EXP) return ~UK(0);          // NaN
    if (mag == 0) return SIGN;             // +0 / -0 -> key of +0
    return (bits & SIGN) ? ~bits : (bits | SIGN);
  }
}

}  // namespace b2

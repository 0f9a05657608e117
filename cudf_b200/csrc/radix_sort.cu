// radix_sort.cu — LSD one-sweep radix sort for sm_90a (no thrust / cub).
//
// Replaces the cub::DeviceRadixSort / DeviceMergeSort call sites of the reference:
//   cpp/src/sort/sorted_order_radix.cu:57-180  (SortPairs over (key, row index))
//   cpp/src/sort/sort_radix.cu:59-161          (SortKeys fast path of cudf::sort)
//   cpp/src/sort/sort_column_impl.cuh:35-97    (nullable single column; comparator semantics)
//   cpp/src/sort/sort_impl.cuh:31-96           (table dispatch, defaults, multi-column lexicographic)
//
// Design (one GPU, N rows, key type of W bytes => W passes of 8 bits):
//   1. histogram kernel: one streaming read of the keys, W x 256 digit counts (smem atomics with a
//      warp match_all shortcut for constant digits).
//   2. plan kernel (1 CTA): exclusive scan of each histogram -> global digit bases; passes whose
//      digit is constant over all keys are marked trivial and skipped on the device (no host sync);
//      ping-pong buffer roles are chosen so that the last executed pass writes the output buffer.
//   3. one-sweep pass kernel per digit: dynamic tile ids, warp-level MATCH.ANY ranking (stable),
//      per-digit decoupled look-back over 32-bit {flag,count} words, keys and row indices staged
//      through shared memory in tile-sorted order and written as coalesced per-digit runs.
//      Pass 1 generates row indices on the fly; the last pass of sorted_order writes indices only.
//   4. nullable column: warp-ballot/popc compaction splits valid rows (twiddled key, row index) from
//      null rows (row index in input order), then 3. runs on the valid part only.
// Keys are twiddled to unsigned order-preserving bits on first load (device_utils.cuh) and inverted
// for descending order, which keeps the sort stable like cub's Descending variants.
#include "common.cuh"
#include "device_utils.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <type_traits>

namespace b2 {
namespace {

constexpr int RADIX_BITS = 8;
constexpr int RADIX      = 256;
constexpr uint32_t FLAG_AGG  = 1u << 30;
constexpr uint32_t FLAG_INCL = 2u << 30;
constexpr uint32_t VAL_MASK  = (1u << 30) - 1;

struct pass_plan {
  int32_t trivial;  // 1: every key has the same digit -> pass skipped
  int32_t key_src;  // 0 raw input, 1 buffer A, 2 buffer B
  int32_t key_dst;  // 1 / 2 (unused when last && pairs)
  int32_t idx_src;  // -1 implicit iota, 0 buffer X (output), 1 buffer Y (temp)
  int32_t idx_dst;  // 0 / 1
  int32_t last;     // 1: last executed pass
  int32_t hybrid;   // 1: partial LSD (top digits only) + segment fix-up follows; this pass keeps its keys and does not untwiddle
  int32_t pad;
};

struct sort_ctl {
  pass_plan plan[8];
  uint32_t base[2][8][RADIX];  // [portion parity][pass][digit] global start offset of digit
  int32_t any_pass;            // number of executed passes
  uint32_t nan_count;          // FLOAT keys only
  // hybrid sort (see segment_fix_kernel): the executed passes cover only the digits >= fix_shift / 8; rows whose keys agree
  // on those bits form short segments that the fix-up orders by the remaining low bits
  int32_t hybrid;              // decided by the plan kernel
  int32_t fix_shift;           // segment prefix = key >> fix_shift
  int32_t fix_key_buf;         // key buffer (1 / 2) written by the last executed pass
  int32_t fix_idx_buf;         // payload / row-id buffer (0 / 1 / 2) written by the last executed pass
  uint32_t overflow;           // set by the fix-up when a segment is too long for it: the host reruns the full LSD sort
  // two-phase histogram of the hybrid plan: phase 1 counts the top four digits only; the low digits are counted (phase 2) only
  // when the plan cannot stop above them
  int32_t need_low;            // 1: phase 1 could not decide, the low digits' histograms are required
  int32_t fix_fast;            // hybrid plan: which segment_fix_kernel instantiation runs (0: plain walks, 1: branch-free first neighbours)
  unsigned long long vary;     // OR of (key ^ first key) over the input
  // range tier of the hybrid plan (see range_sort_kernel): the executed passes sort only the range id = (key >> range_shift) &
  // (2^range_bits - 1); each range is then sorted in shared memory by the bits below range_shift
  int32_t range;
  int32_t range_shift;
  int32_t range_bits;
};

template <typename UK>
__device__ __forceinline__ UK twiddle_rt(UK bits, int kind, UK desc_mask)
{
  UK k;
  if (kind == (int)key_kind::SIGNED) k = twiddle_in<UK, key_kind::SIGNED>(bits);
  else if (kind == (int)key_kind::FLOAT) {
    if constexpr (sizeof(UK) >= 4) k = twiddle_in<UK, key_kind::FLOAT>(bits);
    else k = bits;
  } else k = bits;
  return k ^ desc_mask;
}
// inverse for integer kinds (float keys never take the keys-only path)
template <typename UK>
__device__ __forceinline__ UK untwiddle_rt(UK k, int kind, UK desc_mask)
{
  k ^= desc_mask;
  if (kind == (int)key_kind::SIGNED) k ^= (UK(1) << (sizeof(UK) * 8 - 1));
  return k;
}

// ------------------------------------------------------------------------------------------------
// 1. histogram
// ------------------------------------------------------------------------------------------------
// MIX (64-bit keys, join partitioning): keys are mix64(raw) and only the digits of passes 6 and 7 are counted.
// pass_mask: bit p set = count digit p (the hybrid plan first looks at the top digits only; a partition pass needs one).
// gate: when not null the kernel returns at once unless *gate != 0 (second-phase histogram of the low digits).
// vary_out: when not null receives the OR over all keys of (key ^ first key): a digit is constant over the input iff its
// byte of that word is zero (lets the plan know which uncounted digits are trivial).
template <typename UK, bool MIX = false>
__global__ void __launch_bounds__(512) histogram_kernel(const UK* __restrict__ keys, int64_t n, int raw, int kind,
                                                       UK desc_mask, uint32_t* __restrict__ ghist,
                                                       uint32_t* __restrict__ nan_count, uint32_t pass_mask = 0xffu,
                                                       const int32_t* __restrict__ gate = nullptr,
                                                       unsigned long long* __restrict__ vary_out = nullptr)
{
  constexpr int NP = sizeof(UK);
  if (gate != nullptr && *gate == 0) return;
  __shared__ uint32_t sh[NP][RADIX];
  for (int i = threadIdx.x; i < NP * RADIX; i += blockDim.x) (&sh[0][0])[i] = 0;
  __syncthreads();
  uint32_t nans = 0;
  constexpr int VEC = 16 / sizeof(UK);
  // head (unaligned prefix), vector body, tail
  const uintptr_t addr = reinterpret_cast<uintptr_t>(keys);
  int64_t head = ((16 - (addr & 15)) & 15) / sizeof(UK);
  if (head > n) head = n;
  const int64_t nvec = (n - head) / VEC;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;

  // reference key for the vary word: the (transformed) first key of the column
  UK k_first;
  {
    const UK r0 = keys[0];
    if constexpr (MIX) k_first = (UK)mix64((uint64_t)r0);
    else k_first = raw ? twiddle_rt<UK>(r0, kind, desc_mask) : r0;
  }
  uint64_t vary_acc = 0;
  auto account = [&](UK rawbits, bool active) {
    UK k;
    if constexpr (MIX) k = (UK)mix64((uint64_t)rawbits);
    else k = raw ? twiddle_rt<UK>(rawbits, kind, desc_mask) : rawbits;
    if (active && raw && kind == (int)key_kind::FLOAT && (UK)(k ^ desc_mask) == (UK)~UK(0)) nans++;
    if (active) vary_acc |= (uint64_t)(k ^ k_first);
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      if (!((pass_mask >> p) & 1u)) continue;
      unsigned d = (unsigned)(k >> (p * 8)) & 255u;
      unsigned amask = __ballot_sync(0xffffffffu, active);
      if (amask == 0) continue;
      int pred = 0;
      // constant-digit shortcut: one add per warp instead of 32 same-address atomics
      if (amask == 0xffffffffu) __match_all_sync(0xffffffffu, d, &pred);
      if (pred) {
        if (lane_id() == 0) atomicAdd(&sh[p][d], 32u);
      } else if (active) {
        atomicAdd(&sh[p][d], 1u);
      }
    }
  };

  // fast path: whole warps of full 16-byte vectors. Digits that are constant across the warp (the
  // common case for the high bytes of real data) are detected with two REDUX ops on key ^ key(lane 0)
  // and counted by one lane, so that skewed inputs do not serialise on same-address atomics.
  auto account_fast = [&](UK rawbits) {
    UK k;
    if constexpr (MIX) k = (UK)mix64((uint64_t)rawbits);
    else k = raw ? twiddle_rt<UK>(rawbits, kind, desc_mask) : rawbits;
    if (raw && kind == (int)key_kind::FLOAT && (UK)(k ^ desc_mask) == (UK)~UK(0)) nans++;
    // bits in which some lane differs from the column's first key: a digit whose byte is zero here is the same in all 32
    // lanes (counted once per warp), and the OR over all warps tells which digits are constant over the whole input
    const uint64_t d64 = (uint64_t)(k ^ k_first);
    uint32_t vary_lo = __reduce_or_sync(0xffffffffu, (uint32_t)d64);
    uint32_t vary_hi = sizeof(UK) > 4 ? __reduce_or_sync(0xffffffffu, (uint32_t)(d64 >> 32)) : 0u;
    const uint64_t vary = ((uint64_t)vary_hi << 32) | vary_lo;
    vary_acc |= vary;
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      if (!((pass_mask >> p) & 1u)) continue;
      const unsigned d = (unsigned)(k >> (p * 8)) & 255u;
      if (((vary >> (p * 8)) & 255u) == 0) {
        if (lane_id() == 0) atomicAdd(&sh[p][d], 32u);
      } else {
        atomicAdd(&sh[p][d], 1u);
      }
    }
  };
  const int4* vkeys = reinterpret_cast<const int4*>(keys + head);
  int64_t v = tid;
  for (; (v | 31) < nvec; v += nthreads) {
    int4 q = ld_nc_v4(vkeys + v);
    UK tmp[VEC];
    memcpy(tmp, &q, 16);
#pragma unroll
    for (int j = 0; j < VEC; ++j) account_fast(tmp[j]);
  }
  // remaining (< 32) vectors of the last partial warp-row, plus head / tail scalars: block 0, warp 0
  if (blockIdx.x == 0 && threadIdx.x < 32) {
    const int64_t vrem0 = nvec / 32 * 32;
    {
      const int64_t vv = vrem0 + threadIdx.x;
      const bool act = vv < nvec;
      int4 q = act ? ld_nc_v4(vkeys + vv) : make_int4(0, 0, 0, 0);
      UK tmp[VEC];
      memcpy(tmp, &q, 16);
#pragma unroll
      for (int j = 0; j < VEC; ++j) account(tmp[j], act);
    }
    int64_t tail_start = head + nvec * VEC;
    int64_t nscalar = head + (n - tail_start);
    for (int64_t b = 0; b < nscalar; b += 32) {
      int64_t j = b + threadIdx.x;
      bool act = j < nscalar;
      int64_t e = j < head ? j : tail_start + (j - head);
      UK rb = act ? keys[e] : UK(0);
      account(rb, act);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NP * RADIX; i += blockDim.x) {
    uint32_t c = (&sh[0][0])[i];
    if (c) atomicAdd(&ghist[i], c);
  }
  if (nan_count) {
    nans = warp_sum(nans);
    if (lane_id() == 0 && nans) atomicAdd(nan_count, nans);
  }
  if (vary_out) {
    const uint32_t lo = __reduce_or_sync(0xffffffffu, (uint32_t)vary_acc);
    const uint32_t hi = __reduce_or_sync(0xffffffffu, (uint32_t)(vary_acc >> 32));
    if (lane_id() == 0 && (lo | hi)) atomicOr(vary_out, ((unsigned long long)hi << 32) | lo);
  }
}

// ------------------------------------------------------------------------------------------------
// 2. plan
// ------------------------------------------------------------------------------------------------
// mode_pairs: 1 sorted_order (indices), 0 keys-only.  raw: 1 keys come from the user's column
// (implicit indices), 0 keys already twiddled in buffer A with explicit indices in idx buffer
// `pre_idx_buf`.
// hyb_allowed: the caller can run the segment fix-up (and rerun without it on overflow), so the plan may stop the LSD
// passes early. The number of top digits that has to be sorted is chosen from the digit histograms: if the digits
// were independent, rows would share a given combination of the chosen digits with probability prod_p sum_d (c_pd / n)^2,
// i.e. a segment would hold about n * prod rows. The estimate only selects the plan; the fix-up verifies it.
constexpr double HYB_MAX_EXPECTED_SEGMENT = 4.0;
constexpr int HYB_MIN_SAVED_PASSES = 2;

// phase 0: every digit was counted. phase 1 (64-bit keys, hybrid allowed): only digits 4..7 were counted; the low digits are
// known to be constant or not from ctl->vary; if the hybrid plan can stop within the top digits it is final, otherwise
// ctl->need_low is raised, the gated second histogram counts digits 0..3 and phase 2 plans with everything (phase 2 returns
// at once when phase 1 was final).
// range_allowed (hybrid plan only): the caller can run range_sort_kernel. The plan then stops the passes at the top one or two
// adjacent non-trivial digits once the expected range, n * prod coll, stays below RANGE_CAP by five standard deviations of a
// uniform spread (1e9 uniform keys: 15 259 + 5 * 124 rows against 16 384), and at least one digit is left to sort inside the ranges.
constexpr int RANGE_CAP = 16384;  // rows of one range: range_sort_kernel holds its keys in 128 KB of shared memory
__global__ void plan_kernel(const uint32_t* __restrict__ ghist, int npass, uint32_t n, int raw, int pre_idx_buf,
                            sort_ctl* ctl, int first_pass, int last_pass, int hyb_allowed, int phase = 0, int range_allowed = 0)
{
  __shared__ uint32_t warp_tot[8];
  __shared__ int triv[8];
  __shared__ double sq[RADIX];
  __shared__ double coll[8];  // sum_d (c_d / n)^2 of each pass
  const int d = threadIdx.x;  // 256 threads
  if (phase == 2 && ctl->need_low == 0) return;
  const int counted_from = phase == 1 ? 4 : 0;  // digits below were not counted
  const unsigned long long vary = ctl->vary;
  for (int p = 0; p < npass; ++p) {
    uint32_t c = ghist[p * RADIX + d];
    if (p < counted_from) c = ((vary >> (8 * p)) & 0xffull) == 0 ? (d == 0 ? n : 0u) : 0u;  // all-or-nothing stand-in: constant digit or unknown
    if (d == 0) triv[p] = 0;
    {
      const double f = (double)c / (double)n;
      sq[d] = f * f;
    }
    __syncthreads();
    if (d == 0) {
      double t = 0;
      for (int j = 0; j < RADIX; ++j) t += sq[j];
      coll[p] = t;
    }
    if (c == n || p < first_pass || p > last_pass) triv[p] = 1;  // passes outside [first,last] are skipped
    uint32_t inc = warp_inclusive_sum(c);
    if ((d & 31) == 31) warp_tot[d >> 5] = inc;
    __syncthreads();
    uint32_t woff = 0;
    for (int w = 0; w < (d >> 5); ++w) woff += warp_tot[w];
    ctl->base[0][p][d] = woff + inc - c;
    __syncthreads();
  }
  if (d == 0) {
    int nexec = 0;
    for (int p = 0; p < npass; ++p) nexec += triv[p] ? 0 : 1;
    int hybrid = 0, low = 0;
    double seg_est = 0.0;    // hybrid plan: expected rows per segment
    bool undecided = false;  // phase 1: the decision would need an uncounted digit
    if (hyb_allowed && nexec > HYB_MIN_SAVED_PASSES) {
      double e = (double)n;
      int k = 0;
      low = npass;
      for (int p = npass - 1; p >= 0 && (k == 0 || e > HYB_MAX_EXPECTED_SEGMENT); --p) {  // at least one pass
        if (triv[p]) continue;
        if (p < counted_from) { undecided = true; break; }
        e *= coll[p];
        ++k;
        low = p;
      }
      if (!undecided && e <= HYB_MAX_EXPECTED_SEGMENT && nexec - k >= HYB_MIN_SAVED_PASSES) {
        hybrid = 1;
        seg_est = e;
        for (int p = 0; p < low; ++p) triv[p] = 1;
        nexec = k;
      }
    }
    if (phase == 1) {
      // final only when the hybrid plan stops within the counted digits, or when no uncounted digit has to be sorted at all
      bool low_needed = false;
      for (int p = 0; p < counted_from; ++p) low_needed = low_needed || !triv[p];
      if (!hybrid && low_needed) {
        ctl->need_low = 1;
        return;
      }
      ctl->need_low = 0;
    }
    int range = 0, range_low = 0, range_bits = 0;
    if (hybrid && range_allowed) {
      double e = (double)n;
      for (int p = npass - 1; p > low && range_bits < 16; --p) {
        if (triv[p]) {
          if (range_bits == 0) continue;
          break;  // the range id is one run of adjacent digits
        }
        e *= coll[p];
        range_bits += RADIX_BITS;
        if (e + 5.0 * sqrt(e) <= (double)RANGE_CAP) {
          for (int q = low; q < p; ++q) range = range || !triv[q];  // at least one digit left to sort inside the ranges
          range_low = p;
          break;
        }
      }
      if (range) {
        for (int q = 0; q < range_low; ++q) triv[q] = 1;
        nexec = 0;
        for (int q = 0; q < npass; ++q) nexec += triv[q] ? 0 : 1;
      }
    }
    ctl->range        = range;
    ctl->range_shift  = range_low * RADIX_BITS;
    ctl->range_bits   = range ? range_bits : 0;
    ctl->hybrid    = hybrid;
    // expected rows per segment decides the fix-up flavour: mostly single-row segments (1e9 uniform keys: 0.23) take the
    // plain walks, ~2-row segments (a rank's shard of the sharded sort: 1.9) the branch-free form
    ctl->fix_fast  = (hybrid && seg_est > 0.75) ? 1 : 0;
    ctl->fix_shift = low * RADIX_BITS;
    ctl->overflow  = 0;
    // idx buffers: 0 = output, 1 = temp. the last executed pass must write 0.
    // key buffers: 1 = A, 2 = B (keys-only: 1 = output, 2 = temp; last executed pass must write 1)
    int k = 0;
    int key_cur = raw ? 0 : 1;
    int idx_cur = raw ? -1 : pre_idx_buf;
    for (int p = 0; p < npass; ++p) {
      pass_plan pl{};
      pl.trivial = triv[p];
      if (!triv[p]) {
        int remaining_after = nexec - 1 - k;  // passes after this one
        pl.key_src = key_cur;
        pl.idx_src = idx_cur;
        // A pass never writes the buffer it reads. Raw input: ping-pong so that the final pass lands in
        // key buffer 1 (the keys-only output) / idx buffer 0 (the output column). Pre-compacted input
        // (keys in A, row ids in idx buffer 1): keys alternate A/B (their final home is irrelevant,
        // pairs mode never returns keys); row ids go to 0 whenever an even number of passes remains,
        // else to a non-zero buffer other than the source (third buffer only for the first pass).
        // Hybrid (raw input only): the last pass must land in the TEMP buffers (key 2 / idx 1), because the fix-up writes
        // the output buffers (key 1 / idx 0) from them.
        const int par = (remaining_after + hybrid) % 2;
        pl.key_dst = raw ? (par == 0 ? 1 : 2) : (key_cur == 1 ? 2 : 1);
        pl.idx_dst = par == 0 ? 0 : (idx_cur == 1 ? 2 : 1);
        pl.last    = remaining_after == 0;
        pl.hybrid  = hybrid;
        if (pl.last) {
          ctl->fix_key_buf = pl.key_dst;
          ctl->fix_idx_buf = pl.idx_dst;
        }
        key_cur = pl.key_dst;
        idx_cur = pl.idx_dst;
        ++k;
      }
      ctl->plan[p] = pl;
    }
    ctl->any_pass = nexec;
  }
}

__global__ void set_fix_fast_kernel(sort_ctl* ctl, int v) { ctl->fix_fast = v; }

// ------------------------------------------------------------------------------------------------
// 3. one-sweep pass
// ------------------------------------------------------------------------------------------------
struct pass_args {
  const void* key_bufs[3];  // [0] raw input column data (already offset), [1], [2]
  int32_t* idx_bufs[3];
  sort_ctl* ctl;
  uint32_t* status;         // [tiles][256] flagged count / prefix rows for this (pass, portion)
  uint32_t* tile_counter;   // for this (pass, portion)
  int64_t portion_start;    // element offset of this portion
  uint32_t portion_n;       // elements in this portion
  int32_t pass;
  int32_t portion_parity;   // which base[] copy to read; the other is written for the next portion
  int32_t has_next_portion;
  int32_t kind;             // key_kind for raw loads / keys-only untwiddle
  int32_t pairs;            // 1: (key, idx) ; 0: keys only
  uint64_t desc_mask;
  int32_t keep_keys;        // pairs mode: also write the keys in the last executed pass (partial sorts)
  const void* val_in;       // CARRY kernels: the caller's payload column (first pass source); last member on purpose
  // RANGE kernels (sharded sort: the range partition IS the exchange): digit = number of splitters <= key; the rows of digit d
  // are written to range_key_dst[d] / range_val_dst[d] (local or PEER memory) at their rank inside this GPU's digit-d run
  // EST kernels share the slot (the parameter block keeps its size): tile table of the estimated-base second pass (run_est_range):
  // tile t reads rows [x, x + (y & 0x7fffffff)) of its source (one window of the first pass), y >> 31 marks the last tile, y == 0
  // lies past the last tile
  union {
    const void* range_splitters;     // device array of (range_parts - 1) twiddled keys, ascending
    const uint2* est_tiles;
  };
  void* const* range_key_dst;        // device array of range_parts pointers
  void* const* range_val_dst;        // same for the carried payload (CARRY) or null
  int32_t range_parts;
  int32_t range_hash;                // 1: no splitters, bucket = range_hash_bucket(key) (hash partition: the sharded join's shuffle)
  // MIX kernels, estimated bases (radix_partition_mix_carry_est): no histogram ran; digit d owns rows [d * est_cap, (d + 1) * est_cap) of the
  // output, rows beyond that range are dropped and ctl->overflow is raised; the last tile leaves every digit's end offset in
  // ctl->base[portion_parity ^ 1][pass]
  uint32_t est_cap;
};

// Hash bucket of the fused partition pass. The additive constant decorrelates it from the local radix join, which partitions
// by the top bits of mix64(key) itself: rows that share an exchange bucket still spread over all of the join's partitions.
__host__ __device__ __forceinline__ unsigned range_hash_bucket(uint64_t twiddled_key, int parts)
{
  const uint64_t h = mix64(twiddled_key + 0x9E3779B97F4A7C15ull);
  return (unsigned)(((h >> 32) * (uint64_t)parts) >> 32);
}

// Block-wide barrier of a warp-specialised kernel: the ranking warps and the look-back warps reach it from different branches, which
// `__syncthreads()` only tolerates in practice; a named barrier with the explicit thread count (`bar.sync 2, n`) is the
// PTX-conformant form for sm_70+ (barrier 0 is what `__syncthreads()` lowers to, and compute-sanitizer synccheck holds it to the
// C++ rule that every thread reaches the same call site).
__device__ __forceinline__ void cta_barrier(int nthreads)
{
#ifdef B2_EMU
  (void)nthreads;
  __syncthreads();
#else
  asm volatile("bar.sync 2, %0;" ::"r"(nthreads) : "memory");
#endif
}
__device__ __forceinline__ void ranker_barrier(int nthreads)
{
#ifdef B2_EMU
  ::emu::named_barrier(1, nthreads);
#else
  asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
#endif
}
__device__ __forceinline__ uint4 ld_volatile_v4(const uint32_t* p)
{
#ifdef B2_EMU
  uint4 v;
  memcpy(&v, p, sizeof(v));
  return v;
#else
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
#endif
}

// One CTA = THREADS ranking threads (NWARPS warps holding IPT keys per thread) + LBW look-back warps.
// Decoupled look-back without fences: a tile's digit counts (later: inclusive prefixes) are published
// as rows of 256 words written in 16-byte groups, ONE lane per group, with a 2-bit state in the top
// bits of the group's first word (0 nothing, 1 aggregate, 2 inclusive; the other three words carry
// plain 32-bit values).  A 16-byte aligned store is observed all-or-nothing by a 16-byte load, so a
// reader lane checks one flag per group and needs no memory fence (a release/acquire variant with a
// separate state word, and polling 256 individually flagged words, were both slower).  Each look-back lane owns one group
// (DPL = 4 digits), fetches LBT predecessor rows per round with independent 128-bit loads and folds
// them with warp-uniform decisions (REDUX and/or over the ready / inclusive bits).
constexpr int LBW = 2;   // look-back warps per CTA
constexpr int DPL = 4;   // digits per look-back lane (one 128-bit load per predecessor tile)
constexpr int LBT = 8;   // predecessor tiles fetched per round

// VT = uint32_t: payload = 32-bit row ids (generated in the first pass) — the shipped path.
// VT = uint64_t / CARRY: payload = the caller's 8-byte (or 4-byte with VT = uint32_t) values column, loaded coalesced in
// the first pass and carried through every pass, so that sort_by_key needs neither row ids nor a gather
// (EXPERIMENTAL in round 1: opt-in with B2_SORT_CARRY=1, not yet run on hardware; DESIGN.md §7.1).
// MIX: raw 64-bit keys are replaced by mix64(key) on load (hash-join partitioning: the first executed pass reads the
// packed key column itself, so the mixed keys are never materialised unsorted).
#ifdef B2_EMU
constexpr bool EMU_BUILD = true;
#else
constexpr bool EMU_BUILD = false;
#endif
// Warp-private digit histogram of the first `nit` of a thread's IPT items (shared-memory atomics, no dependency chain);
// returns the number of distinct digits among the warp's items, which picks the ranking flavour of warp_rank.
template <int IPT, typename DigitAt>
__device__ __forceinline__ int warp_digit_counts(const DigitAt& digit_at, int nit, int lane, uint32_t* my_hist)
{
#pragma unroll
  for (int i = 0; i < IPT; ++i)
    if (i < nit) atomicAdd(&my_hist[digit_at(i)], 1u);
  __syncwarp();
  int distinct = 0;
#pragma unroll
  for (int j = 0; j < RADIX / 32; ++j) distinct += my_hist[j * 32 + lane] != 0u;
  return __reduce_add_sync(0xffffffffu, distinct);
}

// Stable rank of a thread's first `nit` items (item i of lane l comes after item i of lanes < l and after every item < i):
// pos[i] = my_hist[digit] + rank among the warp's earlier items of that digit; my_hist[d] advances past the warp's digit-d items.
// my_hist must hold the warp's starting offset of every digit, and my_bm must be zero (it is left zero).
// Peer masks (lanes of the warp holding the same digit; scripts/ubench/rank_probe.cu compares the strategies):
// MATCH.ANY is cheap only when the warp holds few distinct digits, the shared-memory atomicOr bitmap costs
// about the same at any digit mix.  Hence: bitmap for the general case, MATCH.ANY when the warp holds only a handful of distinct digits.
// All MATCH ops are issued first (independent, pipelined); only the counter chain is serial.
// In the bitmap flavour a __syncwarp separates the followers' read of the peer bitmap from the leader's clear (race-free
// under independent thread scheduling), and the leader advances the warp's running digit offset with one ATOMS.ADD
// (returning the old value) instead of LDS + STS — one shared-memory operation less per key in a kernel bound by
// shared-memory wavefronts.
template <int IPT, typename DigitAt>
__device__ __forceinline__ void warp_rank(const DigitAt& digit_at, int nit, int distinct, int lane, uint32_t* my_hist, uint32_t* my_bm,
                                          uint32_t (&pos)[IPT])
{
  if (distinct > 4) {
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
      if (i >= nit) break;
      const unsigned d = digit_at(i);
      atomicOr(&my_bm[d], 1u << lane);
      __syncwarp();
      const unsigned peers = my_bm[d];
      const unsigned lt = __popc(peers & lanemask_lt());
      uint32_t prev = 0;
      __syncwarp();
      if (lt == 0) {
        prev = atomicAdd(&my_hist[d], (uint32_t)__popc(peers));
        my_bm[d] = 0;
      }
      __syncwarp();
      prev = __shfl_sync(0xffffffffu, prev, __ffs(peers) - 1);
      pos[i] = prev + lt;
    }
  } else {
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
      if (i >= nit) break;
      const unsigned d = digit_at(i);
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      const unsigned lt = __popc(peers & lanemask_lt());
      uint32_t prev = 0;
      if (lt == 0) {
        prev = my_hist[d];
        my_hist[d] = prev + __popc(peers);
      }
      __syncwarp();
      prev = __shfl_sync(0xffffffffu, prev, __ffs(peers) - 1);
      pos[i] = prev + lt;
    }
  }
}

// One bulk async copy (cp.async.bulk, the 1-D TMA path: UBLKCP in SASS) of `bytes` (a multiple of 16, both addresses 16-byte
// aligned) into shared memory, completing on the mbarrier at shared address `mbar` (initialised with one arrival), and the
// wait for it (phase 0). Not in the emulator build, which replays the data movement with ordinary loads.
__device__ __forceinline__ void mbar_init_one(uint32_t mbar)
{
#ifndef B2_EMU
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#else
  (void)mbar;
#endif
}
__device__ __forceinline__ void bulk_copy_to_smem(void* sdst, const void* gsrc, uint32_t bytes, uint32_t mbar)
{
#ifndef B2_EMU
  const uint32_t dst = (uint32_t)__cvta_generic_to_shared(sdst);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(gsrc), "r"(bytes),
               "r"(mbar)
               : "memory");
#else
  (void)sdst; (void)gsrc; (void)bytes; (void)mbar;
#endif
}
__device__ __forceinline__ void mbar_wait_phase0(uint32_t mbar)
{
#ifndef B2_EMU
  asm volatile("{\n .reg .pred p;\n BULK_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n @p bra BULK_DONE;\n bra BULK_WAIT;\n BULK_DONE:\n}" ::"r"(mbar)
               : "memory");
#else
  (void)mbar;
#endif
}

// Tile shape of a one-sweep pass: `threads` ranking threads holding `ipt` keys each, `min_blocks` CTAs per SM.
// `bulk`: full, 16-byte aligned key tiles arrive in shared memory through ONE bulk async copy (cp.async.bulk, the 1-D TMA
// path: UBLKCP in SASS) signalled by an mbarrier, and the ranking warps pick their keys up from there instead of issuing
// `ipt` global loads each (other tiles take the ordinary loads). H100 timings of these and other shapes: DESIGN.md §4.1.
template <int THREADS, int IPT, int MIN_BLOCKS, bool BULK = false>
struct tile_shape {
  static constexpr int threads = THREADS, ipt = IPT, min_blocks = MIN_BLOCKS, tile = THREADS * IPT;
  static constexpr bool bulk = BULK;
};
using tile_384x16      = tile_shape<384, 16, 2>;        // 8-byte keys: row ids, 4-byte payloads, partition passes
using tile_512x16      = tile_shape<512, 16, 1>;        // 1-, 2- and 4-byte keys
using tile_512x20_bulk = tile_shape<512, 20, 1, true>;  // 8-byte keys carrying 8-byte payloads

// BULK passes run one CTA per SM with nothing beside it, so a tile's 80 KB key copy would otherwise wait on HBM with the SM idle
// (a third of the tile: DESIGN.md §4.1). Each tile's first look-back lane, idle until S2, bulk-prefetches into L2 the keys of
// the tile KEY_PREFETCH_TILES ids ahead. Tiles are claimed in order at ~8 per µs over 132 SMs, so that tile starts ~3 µs
// later, about the time its copy takes from HBM: its copy then reads L2. Measured on the H100 at 8 / 16 / 24 / 32 / 48 / 132
// tiles ahead: 24 is the fastest, 16 and 32 are within 0.06 ms per pass of it; 132 tiles (10.5 MB in flight) is slower than
// no prefetch, since the lines are evicted by the running tiles' scattered writes before they are read. Prefetching the
// payload as well is slower too.
constexpr uint32_t KEY_PREFETCH_TILES = 24;

// Phase probe of onesweep_kernel (scripts/onesweep_probe.py), compiled only with -DB2_ONESWEEP_PROBE: ranking thread 0 (and
// the first look-back lane for the look-back stamp) of the CTA that runs tile t writes clock64() at each phase boundary to
// g_onesweep_probe[slot][phase][t], slot 0 for the pass that reads the raw keys and 1 for the others, and its SM id behind the
// stamps. ONESWEEP_PROBE(...) expands to its argument only in that build: the shipped SASS is the same with and without it.
#ifdef B2_ONESWEEP_PROBE
constexpr int ONESWEEP_PROBE_TILES  = 1 << 17;
// entry, tile id known, keys landed, S1, S1b, S2, ranked and staged, S4, look-back done, keys written, payload landed,
// payload written
constexpr int ONESWEEP_PROBE_STAMPS = 12;
__device__ long long g_onesweep_probe[2][ONESWEEP_PROBE_STAMPS + 1][ONESWEEP_PROBE_TILES];
void* g_onesweep_probe_ptr()
{
  void* p = nullptr;
  cudaGetSymbolAddress(&p, g_onesweep_probe);
  return p;
}
__device__ __forceinline__ long long onesweep_probe_clock()
{
  long long v;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(v)::"memory");  // not moved across the phase's memory operations
  return v;
}
__device__ __forceinline__ void onesweep_probe_put(int slot, int i, uint32_t tile, long long v)
{
  if (tile < (uint32_t)ONESWEEP_PROBE_TILES) g_onesweep_probe[slot][i][tile] = v;
}
__device__ __forceinline__ long long onesweep_probe_smid()
{
  uint32_t s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}
#define ONESWEEP_PROBE(...) __VA_ARGS__
#else
#define ONESWEEP_PROBE(...)
#endif
// one stamp by the thread `who` of the current tile
#define ONESWEEP_STAMP_BY(who, i) ONESWEEP_PROBE(if (tid == (who)) onesweep_probe_put(pl.key_src != 0, i, tile, onesweep_probe_clock());)
#define ONESWEEP_STAMP(i) ONESWEEP_STAMP_BY(0, i)

// EST (64-bit raw keys, range sort with estimated bases): digit d owns rows [d * est_cap, (d + 1) * est_cap) of the output (overflow
// check as MIX), the last tile publishes every digit's end, and the first pass ORs (key ^ first key) into ctl->vary; with est_tiles
// the tiles come from that table (the windows of the first pass) instead of one contiguous portion.
template <typename UK, typename Shape, typename VT, bool CARRY, bool MIX, bool RANGE, bool EST = false>
__global__ void __launch_bounds__(Shape::threads + 32 * LBW, Shape::min_blocks) onesweep_kernel(pass_args a)
{
  constexpr int THREADS = Shape::threads;
  constexpr int IPT     = Shape::ipt;
  constexpr bool BULK   = Shape::bulk;
  constexpr int TILE    = THREADS * IPT;
  constexpr int NWARPS = THREADS / 32;
  static_assert(THREADS >= RADIX, "need one ranking thread per digit");
  static_assert(!RANGE || (!MIX && !BULK), "the range-partition pass uses the plain key load");

  const pass_plan pl = a.ctl->plan[a.pass];
  if (pl.trivial) return;
  ONESWEEP_PROBE(const long long probe_entry = onesweep_probe_clock();)

  B2_DYNAMIC_SMEM(smem_raw);
  constexpr int STAGE_W = sizeof(UK) > sizeof(VT) ? sizeof(UK) : sizeof(VT);  // staging holds keys, then the payload
  UK* s_keys          = reinterpret_cast<UK*>(smem_raw);
  VT* s_vals          = reinterpret_cast<VT*>(smem_raw);
  uint32_t* s_whist   = reinterpret_cast<uint32_t*>(smem_raw + (size_t)STAGE_W * TILE);  // [NWARPS][256]
  uint32_t* s_bm      = s_whist + NWARPS * RADIX;  // [NWARPS][256] per-warp digit -> lane bitmaps (ranking)
  uint32_t* s_off     = s_bm + NWARPS * RADIX;     // [256] global offset of digit - tile-local start
  uint32_t* s_cnt     = s_off + RADIX;             // [256] {tile count of digit, tile-local start} pairs
  uint32_t* s_misc    = s_cnt + 2 * RADIX;         // [16]
  // RANGE only: splitters, per-digit destination pointers, digit of every staged item
  UK* s_split         = reinterpret_cast<UK*>(s_misc + 16);                  // [256]
  void** s_kdst       = reinterpret_cast<void**>(s_split + RADIX);           // [256]
  void** s_vdst       = s_kdst + RADIX;                                      // [256]
  uint8_t* s_dig      = reinterpret_cast<uint8_t*>(s_vdst + RADIX);          // [TILE]

  const int tid  = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const bool ranker = warp < NWARPS;

  if (tid == 0) {
    const uint32_t t = atomicAdd(a.tile_counter, 1u);
    s_misc[0] = t;
    if constexpr (EST) {
      s_misc[10] = 0;  // the tile's vary word
      s_misc[11] = 0;
      if (a.est_tiles != nullptr) {
        const uint2 e = a.est_tiles[t];
        s_misc[9]  = e.x;
        s_misc[14] = e.y;
      }
    }
  }
  if constexpr (BULK && !EMU_BUILD) {
    if (tid == 0) mbar_init_one((uint32_t)__cvta_generic_to_shared(s_misc + 12));  // 8-byte aligned slot behind the scan scratch (s_misc[1..8])
  }
  if (ranker) {
#pragma unroll
    for (int j = 0; j < RADIX / 32; ++j) {
      s_whist[warp * RADIX + j * 32 + lane] = 0;
      s_bm[warp * RADIX + j * 32 + lane]    = 0;
    }
  }
  if constexpr (RANGE) {
    for (int i = tid; i < RADIX; i += THREADS + 32 * LBW) {
      s_split[i] = (!a.range_hash && i < a.range_parts - 1) ? static_cast<const UK*>(a.range_splitters)[i] : ~UK(0);
      s_kdst[i]  = i < a.range_parts ? a.range_key_dst[i] : nullptr;
      s_vdst[i]  = (CARRY && i < a.range_parts) ? a.range_val_dst[i] : nullptr;
    }
  }
  __syncthreads();
  const uint32_t tile = s_misc[0];
  uint32_t tile_base = tile * (uint32_t)TILE;  // within portion (EST table: first source row of the tile)
  uint32_t tile_n = min((uint32_t)TILE, a.portion_n - tile_base);
  uint32_t nlim = a.portion_n;                 // source rows below nlim exist
  if constexpr (EST) {
    if (a.est_tiles != nullptr) {
      if (s_misc[14] == 0) return;  // past the last tile: the whole CTA leaves before the named barriers
      tile_base = s_misc[9];
      tile_n    = s_misc[14] & 0x7fffffffu;
      nlim      = tile_base + tile_n;
    }
  }
  ONESWEEP_PROBE(if (tid == 0) {
    onesweep_probe_put(pl.key_src != 0, 0, tile, probe_entry);
    onesweep_probe_put(pl.key_src != 0, ONESWEEP_PROBE_STAMPS, tile, onesweep_probe_smid());
  })
  ONESWEEP_STAMP(1);
  const bool full = tile_n == (uint32_t)TILE;
  const uint32_t pad = (uint32_t)TILE - tile_n;      // padding items sit at the end of digit 255
  const int shift = a.pass * RADIX_BITS;
  const UK desc = (UK)a.desc_mask;

  if (!ranker) {
    // ================================ look-back warp ==============================================
    if constexpr (BULK && !EMU_BUILD) {
      if (tid == THREADS) {  // keys of a later tile into L2 (KEY_PREFETCH_TILES): only full, 16-byte aligned tiles take bulk copies
        const uint32_t tp = tile + KEY_PREFETCH_TILES, ntiles = (a.portion_n + TILE - 1) / TILE;
        uint32_t base = tp * (uint32_t)TILE, rows = 0;
        if (EST && a.est_tiles != nullptr) {
          if (tp < ntiles + RADIX) {  // the tile table's size (run_est_range)
            const uint2 e = a.est_tiles[tp];
            base = e.x;
            rows = e.y & 0x7fffffffu;
          }
        } else if (tp < ntiles) {
          rows = min((uint32_t)TILE, a.portion_n - base);
        }
        const UK* ks = static_cast<const UK*>(pl.key_src == 0 ? a.key_bufs[0] : (pl.key_src == 1 ? a.key_bufs[1] : a.key_bufs[2])) +
                       a.portion_start + base;
        if (rows == (uint32_t)TILE && (reinterpret_cast<uintptr_t>(ks) & 15) == 0)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(ks), "r"((uint32_t)(sizeof(UK) * TILE)) : "memory");
      }
    }
    cta_barrier(THREADS + 32 * LBW);  // (S2) agg[tile][*] written by the rankers; s_cnt = {count, tile-local start}
    const int d0 = ((warp - NWARPS) * 32 + lane) * DPL;
    uint32_t cnt[DPL], loc[DPL], excl[DPL];
#pragma unroll
    for (int j = 0; j < DPL; j += 2) {
      const uint4 cs = *reinterpret_cast<const uint4*>(s_cnt + 2 * (d0 + j));  // {cnt, start, cnt, start}
      cnt[j] = cs.x; loc[j] = cs.y; cnt[j + 1] = cs.z; loc[j + 1] = cs.w;
      excl[j] = 0; excl[j + 1] = 0;
    }
    uint32_t* const my_row = a.status + (size_t)tile * RADIX + d0;
    auto publish = [&](uint32_t flag, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
#ifdef B2_EMU
      my_row[0] = flag | w0; my_row[1] = w1; my_row[2] = w2; my_row[3] = w3;
#else
      asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(my_row), "r"(flag | w0), "r"(w1), "r"(w2), "r"(w3) : "memory");
#endif
    };
    if (tile == 0) {
      publish(FLAG_INCL, cnt[0], cnt[1], cnt[2], cnt[3]);  // first tile of the portion: counts are inclusive
    } else {
      publish(FLAG_AGG, cnt[0], cnt[1], cnt[2], cnt[3]);
      int64_t t = (int64_t)tile - 1;  // nearest predecessor not folded yet
      bool done = false;
      while (!done) {
        uint4 v[LBT];
#pragma unroll
        for (int r = 0; r < LBT; ++r) {
          const int64_t tt = t - r;
          v[r] = make_uint4(FLAG_INCL, 0, 0, 0);  // tiles before the first one: inclusive zero
          if (tt >= 0) v[r] = ld_volatile_v4(a.status + (size_t)tt * RADIX + d0);
        }
        uint32_t rdy = 0, inc = 0;
#pragma unroll
        for (int r = 0; r < LBT; ++r) {
          rdy |= ((v[r].x >> 30) != 0u ? 1u : 0u) << r;
          inc |= (v[r].x >> 31) << r;
        }
        const uint32_t rdy_all = __reduce_and_sync(0xffffffffu, rdy);
        const uint32_t inc_all = __reduce_and_sync(0xffffffffu, inc);
        const uint32_t inc_any = __reduce_or_sync(0xffffffffu, inc);
        const uint32_t usable  = rdy_all & ~(inc_any & ~inc_all);      // rows every lane sees in the same state
        const int n_ready   = __ffs(~usable) - 1;                       // leading usable rows (LBT if all)
        const int first_inc = (inc_all & usable) ? (__ffs(inc_all & usable) - 1) : LBT;
        const int take = min(n_ready, first_inc + 1);
        if (take == 0) { __nanosleep(40); continue; }
#pragma unroll
        for (int r = 0; r < LBT; ++r) {
          if (r < take) { excl[0] += v[r].x & VAL_MASK; excl[1] += v[r].y; excl[2] += v[r].z; excl[3] += v[r].w; }
        }
        done = first_inc < n_ready;
        t -= take;
      }
      publish(FLAG_INCL, excl[0] + cnt[0], excl[1] + cnt[1], excl[2] + cnt[2], excl[3] + cnt[3]);
    }
    const uint32_t* gb = &a.ctl->base[a.portion_parity][a.pass][d0];
    bool wants_end = a.has_next_portion != 0;
    if constexpr (MIX || EST) wants_end = wants_end || a.est_cap != 0u;
    bool last_tile = tile_base + tile_n == a.portion_n;
    if constexpr (EST) {
      if (a.est_tiles != nullptr) last_tile = (s_misc[14] >> 31) != 0u;
    }
    const bool last_of_portion = wants_end && last_tile;
#pragma unroll
    for (int j = 0; j < DPL; ++j) {
      const uint32_t g = gb[j];
      s_off[d0 + j] = g + excl[j] - loc[j];
      if (last_of_portion) a.ctl->base[a.portion_parity ^ 1][a.pass][d0 + j] = g + excl[j] + cnt[j];
    }
    ONESWEEP_STAMP_BY(THREADS, 8);
    cta_barrier(THREADS + 32 * LBW);  // (S4) offsets ready
    return;
  }

  // ================================== ranking warps ================================================
  // ---- load (warp-striped: item i of lane l in warp w = w*32*IPT + i*32 + l) -------------------
  UK key[IPT];
  const uint32_t wbase = tile_base + warp * (32 * IPT) + lane;
  {
    const UK* src = static_cast<const UK*>(pl.key_src == 0 ? a.key_bufs[0] : (pl.key_src == 1 ? a.key_bufs[1] : a.key_bufs[2])) + a.portion_start;
    bool via_smem = false;
    if constexpr (BULK) via_smem = full && (reinterpret_cast<uintptr_t>(src + tile_base) & 15) == 0;  // uniform over the CTA
    if (via_smem) {
      if constexpr (BULK) {
        constexpr uint32_t BYTES = (uint32_t)(sizeof(UK) * TILE);
        static_assert(!BULK || BYTES % 16 == 0, "bulk copies move multiples of 16 bytes");
        if constexpr (EMU_BUILD) {  // emulator: the same data movement with ordinary loads
          for (int q = tid; q < TILE; q += THREADS) s_keys[q] = src[tile_base + q];
          ranker_barrier(THREADS);
        } else {
          const uint32_t mbar = (uint32_t)__cvta_generic_to_shared(s_misc + 12);
          if (tid == 0) bulk_copy_to_smem(s_keys, src + tile_base, BYTES, mbar);
          mbar_wait_phase0(mbar);
        }
#pragma unroll
        for (int i = 0; i < IPT; ++i) key[i] = s_keys[warp * (32 * IPT) + i * 32 + lane];
      }
    } else if (full) {
#pragma unroll
      for (int i = 0; i < IPT; ++i) key[i] = ld_stream(src + wbase + i * 32);
    } else {
#pragma unroll
      for (int i = 0; i < IPT; ++i) {
        uint32_t e = wbase + i * 32;
        key[i] = e < nlim ? ld_stream(src + e) : UK(0);
      }
    }
    if (pl.key_src == 0) {
#pragma unroll
      for (int i = 0; i < IPT; ++i) {
        if constexpr (MIX) key[i] = (UK)mix64((uint64_t)key[i]);
        else key[i] = twiddle_rt<UK>(key[i], a.kind, desc);
      }
    }
    if (!full) {
      // padding items take the maximum key so that they rank last in the tile
#pragma unroll
      for (int i = 0; i < IPT; ++i)
        if (wbase + i * 32 >= nlim) key[i] = ~UK(0);
    }
    if constexpr (EST) {
      if (pl.key_src == 0) {  // first pass: OR of (key ^ first key of the column), the range sort's bucket bits need it exact
        const UK k0 = twiddle_rt<UK>(static_cast<const UK*>(a.key_bufs[0])[0], a.kind, desc);
        uint64_t v = 0;
#pragma unroll
        for (int i = 0; i < IPT; ++i)
          if (wbase + i * 32 < nlim) v |= (uint64_t)(key[i] ^ k0);
        const uint32_t lo = __reduce_or_sync(0xffffffffu, (uint32_t)v);
        const uint32_t hi = __reduce_or_sync(0xffffffffu, (uint32_t)(v >> 32));
        if (lane == 0 && (lo | hi)) {
          atomicOr(&s_misc[10], lo);
          atomicOr(&s_misc[11], hi);
        }
      }
    }
  }
  ONESWEEP_STAMP(2);

  // digit of a key: a byte of it, or (RANGE) the number of splitters <= key — padding items (all-ones key) land in the last bucket
  auto digit_of = [&](UK k) -> unsigned {
    if constexpr (RANGE) {
      if (a.range_hash) return range_hash_bucket((uint64_t)k, a.range_parts);
      int lo = 0, hi = a.range_parts - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_split[mid] <= k) lo = mid + 1;
        else hi = mid;
      }
      return (unsigned)lo;
    } else {
      return (unsigned)(k >> shift) & 255u;
    }
  };
  unsigned dg[RANGE ? IPT : 1];
  if constexpr (RANGE) {
#pragma unroll
    for (int i = 0; i < IPT; ++i) dg[i] = (wbase + i * 32 >= nlim) ? (unsigned)(RADIX - 1) : digit_of(key[i]);  // padding ranks last (digit 255)
  }
  auto digit_at = [&](int i) -> unsigned {
    if constexpr (RANGE) return dg[i];
    else return (unsigned)(key[i] >> shift) & 255u;
  };
  // ---- early counts: warp-private digit histogram by shared-memory atomics (no dependency chain) ----
  uint32_t* my_hist = s_whist + warp * RADIX;
  const int distinct = warp_digit_counts<IPT>(digit_at, IPT, lane, my_hist);
  ranker_barrier(THREADS);  // (S1)
  ONESWEEP_STAMP(3);
  if constexpr (EST) {
    if (tid == 0 && pl.key_src == 0) {  // one global atomic per CTA
      const unsigned long long v = ((unsigned long long)s_misc[11] << 32) | s_misc[10];
      if (v) atomicOr(&a.ctl->vary, v);
    }
  }

  // ---- per digit: warp counts -> warp offsets; publish the aggregate ---------------------------
  uint32_t tstart = 0, count = 0;
  if (tid < RADIX) {
#pragma unroll
    for (int w = 0; w < NWARPS; ++w) {
      uint32_t c = s_whist[w * RADIX + tid];
      s_whist[w * RADIX + tid] = count;  // exclusive offset of warp w inside digit `tid`
      count += c;
    }
    const uint32_t padded = count;
    if (tid == RADIX - 1) count -= pad;
    // exclusive scan of the padded counts over digits: 8 warps of 32 digits
    uint32_t inc = warp_inclusive_sum(padded);
    if (lane == 31) s_misc[1 + warp] = inc;
    tstart = inc - padded;
  }
  ranker_barrier(THREADS);  // (S1b)
  ONESWEEP_STAMP(4);
  if (tid < RADIX) {
    uint32_t woff = 0;
#pragma unroll
    for (int w = 0; w < RADIX / 32; ++w) woff += (w < warp) ? s_misc[1 + w] : 0u;
    tstart += woff;
    s_cnt[2 * tid]     = count;
    s_cnt[2 * tid + 1] = tstart;
    // fold the tile-local digit start into the warp offsets: position = s_whist[w][d] + rank in warp
#pragma unroll
    for (int w = 0; w < NWARPS; ++w) s_whist[w * RADIX + tid] += tstart;
  }
  cta_barrier(THREADS + 32 * LBW);  // (S2) releases the look-back warps; warp offsets final
  ONESWEEP_STAMP(5);

  // ---- rank within warp (stable): peer masks + running per-warp digit offsets ---------------------
  uint32_t pos[IPT];
  warp_rank<IPT>(digit_at, IPT, distinct, lane, my_hist, s_bm + warp * RADIX, pos);
  // tile-sorted staging of the keys
#pragma unroll
  for (int i = 0; i < IPT; ++i) s_keys[pos[i]] = key[i];
  if constexpr (RANGE) {
#pragma unroll
    for (int i = 0; i < IPT; ++i) s_dig[pos[i]] = (uint8_t)dg[i];
  }
  ONESWEEP_STAMP(6);
  // row ids are fetched only now (their registers replace the dead key registers); the loads
  // overlap with the key write-out below
  VT idx[IPT];
  if (a.pairs) {
    if (pl.idx_src < 0) {
      if constexpr (CARRY) {
        // first pass: the payload column is read at the rows' input positions (coalesced)
        const VT* vsrc = static_cast<const VT*>(a.val_in) + a.portion_start;
#pragma unroll
        for (int i = 0; i < IPT; ++i) {
          const uint32_t e = wbase + i * 32;
          idx[i] = e < nlim ? ld_stream(vsrc + e) : VT(0);
        }
      } else {
#pragma unroll
        for (int i = 0; i < IPT; ++i) idx[i] = (uint32_t)(a.portion_start + wbase + i * 32);
      }
    } else {
      const VT* isrc = reinterpret_cast<const VT*>(pl.idx_src == 0 ? a.idx_bufs[0] : (pl.idx_src == 1 ? a.idx_bufs[1] : a.idx_bufs[2])) + a.portion_start;
      if (full) {
#pragma unroll
        for (int i = 0; i < IPT; ++i) idx[i] = ld_stream(isrc + wbase + i * 32);
      } else {
#pragma unroll
        for (int i = 0; i < IPT; ++i) {
          uint32_t e = wbase + i * 32;
          idx[i] = e < nlim ? ld_stream(isrc + e) : VT(0);
        }
      }
    }
  }
  cta_barrier(THREADS + 32 * LBW);  // (S4) keys staged, scatter offsets ready
  ONESWEEP_STAMP(7);

  const bool write_keys = !(a.pairs && pl.last) || a.keep_keys || pl.hybrid;
  UK* kdst = static_cast<UK*>(const_cast<void*>(pl.key_dst == 1 ? a.key_bufs[1] : a.key_bufs[2]));
  uint32_t dst[IPT];
  uint8_t dstd[RANGE ? IPT : 1];
#pragma unroll
  for (int j = 0; j < IPT; ++j) {
    const uint32_t q = j * THREADS + tid;
    UK k = s_keys[q];
    unsigned d;
    if constexpr (RANGE) d = s_dig[q];
    else d = (unsigned)(k >> shift) & 255u;
    dst[j] = s_off[d] + q;
    if constexpr (MIX || EST) {
      if (a.est_cap != 0u && dst[j] >= (d + 1u) * a.est_cap) {  // digit d's reserved range is full: the caller falls back to exact bases
        if (q < tile_n) a.ctl->overflow = 1u;
        dst[j] = 0xFFFFFFFFu;
      }
    }
    if constexpr (RANGE) {
      dstd[j] = (uint8_t)d;
      if (q < tile_n) static_cast<UK*>(s_kdst[d])[dst[j]] = untwiddle_rt<UK>(k, a.kind, desc);  // the receiver sorts raw column values
    } else if (write_keys && q < tile_n && (!(MIX || EST) || dst[j] != 0xFFFFFFFFu)) {
      if (!a.pairs && pl.last && !pl.hybrid) k = untwiddle_rt<UK>(k, a.kind, desc);
      kdst[dst[j]] = k;
    }
  }
  ONESWEEP_STAMP(9);
  if (a.pairs) {
    ranker_barrier(THREADS);
#pragma unroll
    for (int i = 0; i < IPT; ++i) s_vals[pos[i]] = idx[i];
    ONESWEEP_STAMP(10);
    ranker_barrier(THREADS);
    VT* idst = reinterpret_cast<VT*>(pl.idx_dst == 0 ? a.idx_bufs[0] : (pl.idx_dst == 1 ? a.idx_bufs[1] : a.idx_bufs[2]));
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
      const uint32_t q = j * THREADS + tid;
      if constexpr (RANGE) {
        if (q < tile_n) static_cast<VT*>(s_vdst[dstd[j]])[dst[j]] = s_vals[q];
      } else {
        if (q < tile_n && (!(MIX || EST) || dst[j] != 0xFFFFFFFFu)) idst[dst[j]] = s_vals[q];
      }
    }
    ONESWEEP_STAMP(11);
  }
}

// all passes trivial: the sorted order is the input order
template <typename UK, bool MIX = false>
__global__ void finalize_kernel(pass_args a, int64_t n, int raw, int pre_idx_buf, int carry_bytes)
{
  if (a.ctl->any_pass != 0) return;
  if (carry_bytes) {  // carried payload and no executed pass: the output is the payload column itself
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      if (carry_bytes == 8) reinterpret_cast<uint64_t*>(a.idx_bufs[0])[i] = static_cast<const uint64_t*>(a.val_in)[i];
      else reinterpret_cast<uint32_t*>(a.idx_bufs[0])[i] = static_cast<const uint32_t*>(a.val_in)[i];
      if (a.keep_keys && raw) {  // partition passes keep the (mixed) keys next to the payload
        UK k = static_cast<const UK*>(a.key_bufs[0])[i];
        if constexpr (MIX) k = (UK)mix64((uint64_t)k);
        static_cast<UK*>(const_cast<void*>(a.key_bufs[1]))[i] = k;
      }
    }
    return;
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (a.pairs) {
      if (raw) a.idx_bufs[0][i] = (int32_t)i;
      else if (pre_idx_buf != 0) a.idx_bufs[0][i] = a.idx_bufs[1][i];
      if (a.keep_keys && raw) {
        UK k = static_cast<const UK*>(a.key_bufs[0])[i];
        if constexpr (MIX) k = (UK)mix64((uint64_t)k);
        static_cast<UK*>(const_cast<void*>(a.key_bufs[1]))[i] = k;
      }
    } else {
      // keys-only (always raw): copy input to output
      static_cast<UK*>(const_cast<void*>(a.key_bufs[1]))[i] = static_cast<const UK*>(a.key_bufs[0])[i];
    }
  }
}

// Hybrid sort, second half.  The executed LSD passes ordered the rows by the key bits >= fix_shift (stable), so rows that
// agree on those bits ("segments") are contiguous and still in input order.  Each row finds its segment by walking
// outwards over the neighbouring keys in shared memory and takes its final place = segment start + number of segment
// rows that precede it in (key, input position) order.  With the plan kernel's choice of digits a segment holds a
// handful of rows (n / 2^32 = 0.23 on average for 1e9 uniform 64-bit keys after four passes), so this is one
// streaming pass: read key + payload, write payload (or the untwiddled key) a few places away.
// A walk stops after FIX_HALO rows.  A row whose walk was cut short keeps its place if every key it saw equals its own
// (a run of duplicates longer than the window: windows of neighbouring rows overlap, so if nobody objects the whole
// run is one value and already in order); otherwise it raises ctl->overflow and the host reruns the full LSD sort.
constexpr int FIX_THREADS = 256;
constexpr int FIX_IPT     = 8;
constexpr int FIX_TILE    = FIX_THREADS * FIX_IPT;
constexpr int FIX_HALO    = 64;

// Walk of one row with key k over its segment (the neighbours whose keys agree with k on the bits >= shift): key_at(o) is
// the key o rows away, lmax / rmax the rows that exist to the left / right (at most FIX_HALO). The row's final place is its
// own minus `left` plus `before`; `cut`: a walk reached FIX_HALO rows, `all_equal`: every key it saw equals k.
struct seg_walk {
  int left, before;
  bool all_equal, cut;
};
template <typename UK, int FIX_FAST, typename KeyAt>
__device__ __forceinline__ seg_walk segment_walk(const KeyAt& key_at, UK k, int shift, int lmax, int rmax)
{
  const UK pf = k >> shift;
  seg_walk w{0, 0, true, false};
  // The first FIX_FAST neighbours on each side are examined without branches (every lane of the warp does the same
  // work: a divergent walk costs the warp its LONGEST segment, which tripled the kernel's time at ~2 rows per segment);
  // only rows whose segment reaches further continue with the loops below.
  bool in_l = true, in_r = true;  // FIX_FAST = 0: no unrolled part, both walks start at the row itself
#pragma unroll
  for (int s = 1; s <= FIX_FAST; ++s) {
    const UK ol = key_at(-s);   // inside the halo: FIX_HALO >= FIX_FAST
    const UK orr = key_at(s);
    in_l = in_l && s <= lmax && (UK)(ol >> shift) == pf;
    in_r = in_r && s <= rmax && (UK)(orr >> shift) == pf;
    w.left += in_l ? 1 : 0;
    w.before += (in_l && ol <= k) ? 1 : 0;   // earlier rows win ties
    w.before += (in_r && orr < k) ? 1 : 0;
    w.all_equal = w.all_equal && (!in_l || ol == k) && (!in_r || orr == k);
  }
  int right = 0;
  if (in_l) {  // the segment extends further to the left
    for (;;) {
      if (w.left == lmax) { w.cut = lmax == FIX_HALO; break; }
      const UK o = key_at(-w.left - 1);
      if ((UK)(o >> shift) != pf) break;
      ++w.left;
      w.before += o <= k ? 1 : 0;
      w.all_equal = w.all_equal && o == k;
    }
  }
  if (in_r) {
    right = FIX_FAST;
    for (;;) {
      if (right == rmax) { w.cut = w.cut || rmax == FIX_HALO; break; }
      const UK o = key_at(right + 1);
      if ((UK)(o >> shift) != pf) break;
      ++right;
      w.before += o < k ? 1 : 0;
      w.all_equal = w.all_equal && o == k;
    }
  }
  return w;
}

template <typename UK, typename VT, int FIX_FAST>
__global__ void __launch_bounds__(FIX_THREADS) segment_fix_kernel(pass_args a, int64_t n)
{
  if (!a.ctl->hybrid || a.ctl->fix_fast != (FIX_FAST ? 1 : 0)) return;
  __shared__ UK sk[FIX_TILE + 2 * FIX_HALO];
  const int shift = a.ctl->fix_shift;
  const UK* __restrict__ keys = static_cast<const UK*>(a.ctl->fix_key_buf == 1 ? a.key_bufs[1] : a.key_bufs[2]);
  const VT* __restrict__ vin  = reinterpret_cast<const VT*>(a.ctl->fix_idx_buf == 1 ? a.idx_bufs[1] : a.idx_bufs[2]);
  VT* __restrict__ vout = reinterpret_cast<VT*>(a.idx_bufs[0]);
  UK* __restrict__ kout = static_cast<UK*>(const_cast<void*>(a.key_bufs[1]));
  const UK desc = (UK)a.desc_mask;
  const int64_t ntiles = (n + FIX_TILE - 1) / FIX_TILE;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = tile * FIX_TILE;
    __syncthreads();  // the previous tile's walks are done
    for (int q = threadIdx.x; q < FIX_TILE + 2 * FIX_HALO; q += FIX_THREADS) {
      const int64_t g = base - FIX_HALO + q;
      sk[q] = (g >= 0 && g < n) ? ld_stream(keys + g) : UK(0);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < FIX_IPT; ++j) {
      const int i = j * FIX_THREADS + threadIdx.x;
      const int64_t gi = base + i;
      if (gi >= n) continue;
      VT v{};
      if (a.pairs) v = ld_stream(vin + gi);
      const UK k  = sk[FIX_HALO + i];
      // rows to the left / right that exist (array ends are segment ends)
      const int lmax = (int)(gi < FIX_HALO ? gi : (int64_t)FIX_HALO);
      const int rmax = (int)(n - 1 - gi < FIX_HALO ? n - 1 - gi : (int64_t)FIX_HALO);
      const seg_walk w = segment_walk<UK, FIX_FAST>([&](int o) { return sk[FIX_HALO + i + o]; }, k, shift, lmax, rmax);
      int64_t dst = gi - w.left + w.before;
      if (w.cut) {
        dst = gi;
        if (!w.all_equal) atomicOr(&a.ctl->overflow, 1u);
      }
      if (a.pairs) vout[dst] = v;
      else kout[dst] = untwiddle_rt<UK>(k, a.kind, desc);
    }
  }
}

// Range tier of the hybrid plan.  The executed LSD passes cover only the top digit(s) the range id is made of (the 16-bit
// prefix for 1e9 uniform keys: ~15 K rows per range), so every range is a contiguous run of rows in input order and its keys
// agree on every bit at and above ctl->range_shift.  range_sort_kernel sorts one range per CTA in shared memory:
//   1. bucket: the next bits below the range id that vary over the input (ctl->vary), up to 2^RANGE_BUCKET_BITS buckets
//      (~2 rows per bucket at RANGE_CAP rows), so the bucket is monotone in the key; one shared-memory counting pass
//      (histogram, scan, unstable scatter of the local rows) groups the range by bucket;
//   2. order each bucket directly: a row's place is its bucket's start + the number of the bucket's rows with a smaller
//      (key, local row), so equal keys keep their input order: the stable sort, the hybrid plan's order row for row;
//   3. write: the payload window (in L2 from a prefetch issued with the key load) replaces the dead keys in shared memory
//      by a second bulk copy (estimated windows: issued before the walk of step 2, which then no longer reads the keys), and
//      every output row is written coalesced from there.
// A range longer than RANGE_CAP rows, or a bucket longer than RANGE_BUCKET_CAP rows (many equal or clustered keys), raises
// ctl->overflow (the host reruns without the range tier).
// Threads per CTA: 2^9 on the exact plan, 2^10 with estimated windows. Either way one CTA fills an SM's shared memory; the
// estimated-window kernel's walk is a chain of dependent shared-memory loads per row, and twice the warps overlap more of them.
// The CPU emulator runs every thread of a CTA as a fiber, 65 536 CTAs per call, so there the kernel keeps 2^9 threads (its
// code takes any 2^9 or 2^10) and the emulated tests keep their running time.
template <bool EST>
constexpr int range_log_threads = EST && !EMU_BUILD ? 10 : 9;
constexpr int RANGE_THREADS     = 1 << range_log_threads<false>;
constexpr int RANGE_BUCKET_BITS = 13;
constexpr int RANGE_BUCKETS     = 1 << RANGE_BUCKET_BITS;
constexpr int RANGE_BUCKET_CAP  = FIX_HALO;  // rows of one bucket: each row compares its key with all of them
constexpr int RANGE_SLOTS       = RANGE_BUCKETS + RANGE_BUCKETS / 32;  // padded counter layout of range_sort_kernel<VT, true>
constexpr int RANGE_WALK_ROWS   = 4;  // rows of one thread whose bucket walks run side by side (estimated windows)
// Unrolled walk steps of a group of RANGE_WALK_ROWS rows (estimated windows); a longer bucket finishes its row in a tail loop.
// At 1e9 uniform keys a row's bucket holds 1 + Poisson(1.86) rows, 2.86 on average, and more than 4 for ~12 % of the rows;
// a warp's 128 rows span ~45 buckets, whose largest (~6.4 rows) bounded the loop before. The phase probe (DESIGN §4.1) put
// the walk at 6.62 us per range with 4 steps, 6.89 with 5 and 8.52 with the loop as long as the largest bucket.
constexpr uint32_t RANGE_WALK_STEPS = 4;
// Estimated windows: a bucket order entry is (16-bit key digest << 15 | local row), local rows < RANGE_CAP = 2^14.
constexpr uint32_t RANGE_ROW_MASK = (1u << 15) - 1;

// Bytes in front of the keys: mbarriers, overflow flag and one scan word per warp from [16] on.
constexpr int range_head_bytes(bool est) { return est ? 256 : 128; }

size_t range_sort_smem(bool est)
{
  // scratch + keys, later the payload (one row of slack in front for the 16-byte aligned bulk copy) + bucket counters + local
  // row ids grouped by bucket (with estimated windows: and a 16-bit key digest), then in sorted order. With estimated windows
  // that is 230 672 bytes, within the 232 448 one CTA may have.
  return range_head_bytes(est) + sizeof(uint64_t) * (RANGE_CAP + 2) +
         (est ? sizeof(uint32_t) * (RANGE_SLOTS + RANGE_CAP) : sizeof(uint32_t) * RANGE_BUCKETS + sizeof(uint16_t) * RANGE_CAP);
}

// bounds[i] = first row of range i in the keys the last executed pass wrote, bounds[nranges] = n. One thread per range: a
// binary search over all rows (~30 dependent loads; the 65 537 searches run in parallel).
__global__ void range_bounds_kernel(pass_args a, int64_t n, uint32_t* __restrict__ bounds, int nranges)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > nranges) return;
  const uint64_t* __restrict__ keys = static_cast<const uint64_t*>(a.ctl->fix_key_buf == 1 ? a.key_bufs[1] : a.key_bufs[2]);
  const int sh = a.ctl->range_shift;
  const uint64_t mask = (uint64_t)nranges - 1;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)((keys[mid] >> sh) & mask) < i) lo = mid + 1;
    else hi = mid;
  }
  bounds[i] = (uint32_t)lo;
}

// Rows [0, m) of the window g (row s of its buffer) -> sdst[base + r]; returns base. The 16-byte aligned rows
// [-base, (m + base) / PER * PER - base) come by one bulk copy completing on `mbar` (the caller waits when `bulk`), the rows
// behind them by ordinary loads; a misaligned window, or one whose aligned start would lie before its buffer, takes ordinary
// loads only. The emulator replays the bulk copy with ordinary loads.
struct range_window {
  int base;
  bool bulk;
};
template <int THREADS, typename T>
__device__ __forceinline__ range_window range_window_load(T* sdst, const T* __restrict__ g, int64_t s, int m, uint32_t mbar)
{
  constexpr int PER = 16 / sizeof(T);
  const int off  = (int)((reinterpret_cast<uintptr_t>(g) & 15) / sizeof(T));
  const bool bulk = (reinterpret_cast<uintptr_t>(g) % sizeof(T)) == 0 && s >= off && m + off >= PER;
  const int bulk_rows = bulk ? (m + off) / PER * PER : 0;
  if (bulk) {
    if constexpr (EMU_BUILD) {
      for (int q = threadIdx.x; q < bulk_rows; q += THREADS) sdst[q] = g[q - off];
    } else {
      if (threadIdx.x == 0) bulk_copy_to_smem(sdst, g - off, (uint32_t)(sizeof(T) * bulk_rows), mbar);
    }
    for (int r = bulk_rows - off + (int)threadIdx.x; r < m; r += THREADS) sdst[off + r] = g[r];
  } else {
    for (int q = threadIdx.x; q < m; q += THREADS) sdst[q] = ld_stream(g + q);
  }
  return {bulk ? off : 0, bulk};
}

// Estimated-base range tier (run_est_range): the second pass left output window d7 (rows [d7 * cap, d7 * cap + cnt7[d7]) of its
// buffers, cnt7 clamped to cap) ordered by digit 6, so range (d7, d6) is contiguous inside it. Block d7, thread d6: est[i] = source
// start, est[R + i] = rows and est[2R + i] = dense destination (sum_{e < d7} cnt7[e] + offset inside the window) of range i = d7 * 256
// + d6, R = 65 536. Every range stays inside its window and every destination inside the n output rows, also after an overflow.
__global__ void __launch_bounds__(RADIX) range_est_bounds_kernel(pass_args a, uint32_t cap, uint32_t* __restrict__ est)
{
  __shared__ uint32_t s_lb[RADIX + 1];
  __shared__ uint32_t s_wsum[RADIX / 32];
  constexpr int R = RADIX * RADIX;
  const int d7 = blockIdx.x, d6 = threadIdx.x;
  const uint64_t* __restrict__ keys = static_cast<const uint64_t*>(a.ctl->fix_key_buf == 1 ? a.key_bufs[1] : a.key_bufs[2]);
  auto count = [&](int e) { return min(a.ctl->base[1][7][e] - (uint32_t)e * cap, cap); };
  const uint32_t before = warp_sum(d6 < d7 ? count(d6) : 0u);
  if ((d6 & 31) == 0) s_wsum[d6 >> 5] = before;
  const uint32_t w0 = (uint32_t)d7 * cap, wn = count(d7);
  uint32_t lo = 0, hi = wn;  // first row of the window whose digit 6 is >= d6
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if ((int)((keys[w0 + mid] >> 48) & 255u) < d6) lo = mid + 1;
    else hi = mid;
  }
  s_lb[d6] = lo;
  if (d6 == 0) s_lb[RADIX] = wn;
  __syncthreads();
  uint32_t dense = 0;
  for (int w = 0; w < RADIX / 32; ++w) dense += s_wsum[w];
  const uint32_t end = s_lb[d6 + 1];
  const int i = d7 * RADIX + d6;
  est[i]         = w0 + lo;
  est[R + i]     = end > lo ? end - lo : 0u;  // unordered keys (only after an overflow): an empty range
  est[2 * R + i] = dense + lo;
}

// Phase probe of range_sort_kernel (scripts/range_probe.py), compiled only with -DB2_RANGE_PROBE: thread 0 of CTA i writes
// clock64() at each phase boundary to g_range_probe[phase][i], its SM id and its row count behind them. The shipped build has
// none of it (its SASS is the same with and without this block).
#ifdef B2_RANGE_PROBE
constexpr int RANGE_PROBE_CTAS   = 1 << 17;
constexpr int RANGE_PROBE_STAMPS = 8;  // entry, keys waited, histogram, scan, scatter, walk, payload waited, write issued
__device__ long long g_range_probe[RANGE_PROBE_STAMPS + 2][RANGE_PROBE_CTAS];
void* g_range_probe_ptr()
{
  void* p = nullptr;
  cudaGetSymbolAddress(&p, g_range_probe);
  return p;
}
#define RANGE_PROBE_STAMP(i)                                                                  \
  do {                                                                                        \
    if (threadIdx.x == 0 && blockIdx.x < RANGE_PROBE_CTAS) g_range_probe[i][blockIdx.x] = clock64(); \
  } while (0)
#define RANGE_PROBE_SYNC() __syncthreads()
#else
#define RANGE_PROBE_STAMP(i) do {} while (0)
#define RANGE_PROBE_SYNC() do {} while (0)
#endif

// #{rows of bucket positions [start, end) with a smaller (key, local row) than (k, r)}
__device__ __attribute__((noinline)) uint32_t range_rank_keys(const uint32_t* s_ord, const uint64_t* sk, uint32_t start, uint32_t end,
                                                              uint32_t r, uint64_t k)
{
  uint32_t before = 0;
  for (uint32_t q = start; q < end; ++q) {
    const uint32_t rq = s_ord[q] & RANGE_ROW_MASK;
    const uint64_t kq = sk[rq];
    before += (kq < k || (kq == k && rq < r)) ? 1u : 0u;
  }
  return before;
}

template <typename VT, bool EST = false>
__global__ void __launch_bounds__(1 << range_log_threads<EST>, 1) range_sort_kernel(pass_args a, const uint32_t* __restrict__ bounds)
{
  RANGE_PROBE_STAMP(0);
  using UK = uint64_t;
  constexpr int LT  = range_log_threads<EST>;
  constexpr int RT  = 1 << LT;
  constexpr int IPT = RANGE_CAP / RT;  // local row ids fit 16 bits
  B2_DYNAMIC_SMEM(smem_raw);
  uint32_t* s_misc = reinterpret_cast<uint32_t*>(smem_raw);  // [0..1] / [2..3] key / payload mbarrier, [4] overflow, [16 + warp] scan
  UK* s_keys       = reinterpret_cast<UK*>(smem_raw + range_head_bytes(EST));  // [RANGE_CAP + 2]
  VT* s_vals       = reinterpret_cast<VT*>(s_keys);                          // the payload window once the keys are dead
  uint32_t* s_cnt  = reinterpret_cast<uint32_t*>(s_keys + RANGE_CAP + 2);   // [RANGE_BUCKETS] bucket counters
  uint16_t* s_perm = reinterpret_cast<uint16_t*>(s_cnt + (EST ? RANGE_SLOTS : RANGE_BUCKETS));  // [RANGE_CAP] local rows by
                                                                                                // bucket, then sorted
  // estimated windows: the bucket order holds (digest << 15 | local row) in 32 bits, [RANGE_CAP]; s_perm aliases its front
  uint32_t* s_ord  = reinterpret_cast<uint32_t*>(s_perm);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t s = bounds[blockIdx.x];
  int m;
  int64_t o = s;  // first output row
  if constexpr (EST) {  // range_est_bounds_kernel's table: source start, rows, dense destination
    m = (int)bounds[gridDim.x + blockIdx.x];
    o = bounds[2 * gridDim.x + blockIdx.x];
  } else {
    m = (int)(bounds[blockIdx.x + 1] - s);
  }
  if (m == 0) return;
  if (m > RANGE_CAP) {
    if (tid == 0) atomicOr(&a.ctl->overflow, 1u);
    return;
  }
#ifdef B2_RANGE_PROBE
  if (tid == 0 && blockIdx.x < RANGE_PROBE_CTAS) {
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    g_range_probe[RANGE_PROBE_STAMPS][blockIdx.x]     = smid;
    g_range_probe[RANGE_PROBE_STAMPS + 1][blockIdx.x] = m;
  }
#endif
  const UK* __restrict__ keys = static_cast<const UK*>(a.ctl->fix_key_buf == 1 ? a.key_bufs[1] : a.key_bufs[2]) + s;
  const VT* __restrict__ vin  = reinterpret_cast<const VT*>(a.ctl->fix_idx_buf == 1 ? a.idx_bufs[1] : a.idx_bufs[2]) + s;
  VT* __restrict__ vout = reinterpret_cast<VT*>(a.idx_bufs[0]) + o;
  UK* __restrict__ kout = static_cast<UK*>(const_cast<void*>(a.key_bufs[1])) + o;

  // bucket = the nb bits below the highest bit under the range id that varies over the input (bits between it and the range id
  // are the same in every key); nb ~ log2 m, at most RANGE_BUCKET_BITS. Thread t scans the `per` consecutive buckets t * per + j.
  // Counter of bucket b, exact plan: slot (b mod per) * RT + b / per, so the scan reads conflict-free slots j * RT + t; but
  // the walk's lookups of consecutive buckets then all hit one or two banks (16-way conflicts at per = 16). Estimated windows:
  // slot b + b / 32 (one pad word behind every 32 buckets). The walk's consecutive buckets sit in consecutive banks, and for
  // each per in {1, 2, 4, 8} the scan's reads of slots per * t + j by one warp fall in 32 distinct banks.
  const uint64_t below = a.ctl->vary & ((1ull << a.ctl->range_shift) - 1);
  const uint32_t vhi = (uint32_t)(below >> 32), vlo = (uint32_t)below;
  const int top = vhi ? 64 - __clz((int)vhi) : (vlo ? 32 - __clz((int)vlo) : 0);  // bits [0, top) may differ within a range
  const int want = m > 1 ? 32 - __clz(m - 1) : 0;                                     // ceil(log2 m)
  const int nb = min(min(want, RANGE_BUCKET_BITS), top);
  const int bshift = top - nb;
  const uint32_t bmask = (1u << nb) - 1;
  const int lp = max(nb - LT, 0);  // log2 per
  const int per = 1 << lp;
  auto bucket = [&](UK k) { return (uint32_t)(k >> bshift) & bmask; };
  // Keys of one bucket agree on every bit from bshift up, so the 16 bits below bshift (or bits [0, 16)) order two of them unless
  // they are equal: the walk then compares the whole keys.
  const int dshift = max(bshift - 16, 0);
  auto digest = [&](UK k) { return (uint32_t)(k >> dshift) << 15; };
  auto slot = [&](uint32_t b) {
    if constexpr (EST) return b + (b >> 5);
    else return ((b & (uint32_t)(per - 1)) << LT) | (b >> lp);
  };
  auto own = [&](int j) {  // slot of this thread's bucket j of the scan
    if constexpr (EST) return (int)slot((uint32_t)(tid * per + j));
    else return (j << LT) | tid;
  };

  const uint32_t mbar_k = EMU_BUILD ? 0u : (uint32_t)__cvta_generic_to_shared(s_misc);
  const uint32_t mbar_v = EMU_BUILD ? 0u : (uint32_t)__cvta_generic_to_shared(s_misc + 2);
  if constexpr (!EMU_BUILD) {
    if (tid == 0) {
      mbar_init_one(mbar_k);
      mbar_init_one(mbar_v);
    }
  }
  if (tid == 0) s_misc[4] = 0;
  const int last = EST ? (int)slot(bmask) : (int)bmask;
  for (int i = tid; i <= last; i += RT) s_cnt[i] = 0;
  __syncthreads();

  // ---- keys -> s_keys; the payload window is written in sorted order at the end: bring it into L2 meanwhile ---------------
  const range_window kw = range_window_load<RT>(s_keys, keys, s, m, mbar_k);
  if constexpr (!EMU_BUILD) {
    if (tid == 0 && a.pairs) {
      const uintptr_t lo = reinterpret_cast<uintptr_t>(vin) & ~uintptr_t(15);
      const uintptr_t hi = (reinterpret_cast<uintptr_t>(vin + m) + 15) & ~uintptr_t(15);
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(lo), "r"((uint32_t)(hi - lo)) : "memory");
    }
    if (kw.bulk) mbar_wait_phase0(mbar_k);
  }
  __syncthreads();
  RANGE_PROBE_STAMP(1);
  const UK* sk = s_keys + kw.base;

  // ---- 1. counting pass: bucket histogram, exclusive scan (overflow check), scatter of the local rows ---------------------
  for (int r = tid; r < m; r += RT) atomicAdd(&s_cnt[slot(bucket(sk[r]))], 1u);
  __syncthreads();
  RANGE_PROBE_STAMP(2);
  uint32_t c[1 << (RANGE_BUCKET_BITS - LT)];
  uint32_t tot = 0;
  bool big = false;
#pragma unroll
  for (int j = 0; j < (1 << (RANGE_BUCKET_BITS - LT)); ++j) {
    c[j] = (j < per && tid <= (int)bmask) ? s_cnt[own(j)] : 0u;
    tot += c[j];
    big = big || c[j] > (uint32_t)RANGE_BUCKET_CAP;
  }
  if (big) s_misc[4] = 1;
  const uint32_t inc = warp_inclusive_sum(tot);
  if (lane == 31) s_misc[16 + warp] = inc;
  __syncthreads();
  if (s_misc[4]) {  // uniform: read by every thread behind the barrier
    if (tid == 0) atomicOr(&a.ctl->overflow, 1u);
    return;
  }
  {
    uint32_t run = inc - tot;
    for (int w = 0; w < warp; ++w) run += s_misc[16 + w];
#pragma unroll
    for (int j = 0; j < (1 << (RANGE_BUCKET_BITS - LT)); ++j) {
      if (j < per && tid <= (int)bmask) s_cnt[own(j)] = run;
      run += c[j];
    }
  }
  __syncthreads();
  RANGE_PROBE_STAMP(3);
  if constexpr (EST) {
    for (int r = tid; r < m; r += RT) {
      const UK k = sk[r];
      s_ord[atomicAdd(&s_cnt[slot(bucket(k))], 1u)] = digest(k) | (uint32_t)r;
    }
  } else {
    for (int r = tid; r < m; r += RT) s_perm[atomicAdd(&s_cnt[slot(bucket(sk[r]))], 1u)] = (uint16_t)r;
  }
  __syncthreads();
  RANGE_PROBE_STAMP(4);

  // ---- 2. the row at bucket position p goes to bucket start + #{bucket rows with a smaller (key, local row)} --------------
  // (the counters now hold the bucket ends; consecutive positions share buckets, so a warp's walks are mostly broadcasts)
  uint32_t pk[IPT];  // destination | local row << 16
  range_window vw{0, false};
  if constexpr (EST) {
    // The walk reads the keys only for each row's bucket bounds (and for the rare whole-key rank). With a payload, every thread
    // first keeps the bounds of its rows (start | end << 16, in the slot pk takes later); the keys are then dead, and the payload
    // window replaces them while the walk runs instead of behind it. The whole-key rank then reads the keys from the input.
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
      if (tid + RT * i >= m) break;
      const uint32_t b = bucket(sk[s_ord[tid + RT * i] & RANGE_ROW_MASK]);
      pk[i] = (b ? s_cnt[slot(b - 1)] : 0u) | s_cnt[slot(b)] << 16;
    }
    const UK* kw_rank = sk;
    if (a.pairs) {
      __syncthreads();
      vw = range_window_load<RT>(s_vals, vin, s, m, mbar_v);
      kw_rank = keys;
    }
    // A row's place in its bucket is the number of the bucket's entries with a smaller digest, unless another row shares its
    // digest: that bucket is ranked again by whole keys (out of line: the unrolled walk must stay small enough for the
    // instruction cache). Entries and the bounds lo / hi lie in [0, 2^31], so the sign bit of eq - lo (eq - hi) says whether
    // eq's digest is smaller than (at most) this row's: one subtraction and one shift-add per count. The rows go in groups of
    // RANGE_WALK_ROWS: RANGE_WALK_STEPS unrolled steps walk their buckets side by side, each read clamped to its bucket's last
    // entry, whose extra reads are subtracted behind them. A bucket longer than that finishes its row alone (a warp waits for
    // its longest such tail, per row of the group). Rows past m walk the one-entry bucket [0, 1) and are not written.
#pragma unroll
    for (int i0 = 0; i0 < IPT; i0 += RANGE_WALK_ROWS) {
      if (tid + RT * i0 >= m) break;
      uint32_t e[RANGE_WALK_ROWS], start[RANGE_WALK_ROWS], end[RANGE_WALK_ROWS];
#pragma unroll
      for (int g = 0; g < RANGE_WALK_ROWS; ++g) e[g] = tid + RT * (i0 + g) < m ? s_ord[tid + RT * (i0 + g)] : 0u;
#pragma unroll
      for (int g = 0; g < RANGE_WALK_ROWS; ++g) {
        const bool in = tid + RT * (i0 + g) < m;
        start[g] = in ? pk[i0 + g] & 0xffffu : 0u;
        end[g] = in ? pk[i0 + g] >> 16 : 1u;
      }
      // entries of a smaller digest lie below lo, of at most this row's digest below hi
      auto lo = [&](int g) { return e[g] & ~RANGE_ROW_MASK; };
      auto hi = [&](int g) { return (e[g] & ~RANGE_ROW_MASK) + RANGE_ROW_MASK + 1; };
      uint32_t lt[RANGE_WALK_ROWS] = {}, le[RANGE_WALK_ROWS] = {};
#pragma unroll
      for (uint32_t q = 0; q < RANGE_WALK_STEPS; ++q) {
#pragma unroll
        for (int g = 0; g < RANGE_WALK_ROWS; ++g) {
          const uint32_t eq = s_ord[min(start[g] + q, end[g] - 1)];
          lt[g] += (eq - lo(g)) >> 31;
          le[g] += (eq - hi(g)) >> 31;
        }
      }
#pragma unroll
      for (int g = 0; g < RANGE_WALK_ROWS; ++g) {
#pragma unroll 1
        for (uint32_t q = start[g] + RANGE_WALK_STEPS; q < end[g]; ++q) {
          const uint32_t eq = s_ord[q];
          lt[g] += (eq - lo(g)) >> 31;
          le[g] += (eq - hi(g)) >> 31;
        }
      }
#pragma unroll
      for (int g = 0; g < RANGE_WALK_ROWS; ++g) {
        const uint32_t extra = RANGE_WALK_STEPS - min(end[g] - start[g], RANGE_WALK_STEPS);
        const uint32_t eq = s_ord[end[g] - 1];
        lt[g] -= extra * ((eq - lo(g)) >> 31);
        le[g] -= extra * ((eq - hi(g)) >> 31);
        const uint32_t r = e[g] & RANGE_ROW_MASK;
        if (le[g] - lt[g] > 1u) lt[g] = range_rank_keys(s_ord, kw_rank, start[g], end[g], r, kw_rank[r]);
        pk[i0 + g] = (start[g] + lt[g]) | r << 16;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < IPT; ++i) {
      const int p = tid + RT * i;
      if (p >= m) break;
      const uint32_t r = s_perm[p];
      const UK k = sk[r];
      const uint32_t b = bucket(k);
      const uint32_t end = s_cnt[slot(b)];
      const uint32_t start = b ? s_cnt[slot(b - 1)] : 0u;
      uint32_t before = 0;
      for (uint32_t q = start; q < end; ++q) {
        const uint32_t rq = s_perm[q];
        const UK kq = sk[rq];
        before += (kq < k || (kq == k && rq < r)) ? 1u : 0u;
      }
      pk[i] = (start + before) | r << 16;
    }
  }
  __syncthreads();  // the keys (pairs) and the bucket order in s_perm are dead
  RANGE_PROBE_STAMP(5);

  // ---- 3. sorted local rows -> s_perm; rows written in order from shared memory ----------------------------------------------
  if (!EST && a.pairs) vw = range_window_load<RT>(s_vals, vin, s, m, mbar_v);
#pragma unroll
  for (int i = 0; i < IPT; ++i) {
    if (tid + RT * i >= m) break;
    s_perm[pk[i] & 0xffffu] = (uint16_t)(pk[i] >> 16);
  }
  if constexpr (!EMU_BUILD) {
    if (vw.bulk) mbar_wait_phase0(mbar_v);
  }
  __syncthreads();
  RANGE_PROBE_STAMP(6);
  if (a.pairs) {
    const VT* sv = s_vals + vw.base;
    for (int r = tid; r < m; r += RT) vout[r] = sv[s_perm[r]];
  } else {
    const UK desc = (UK)a.desc_mask;
    for (int r = tid; r < m; r += RT) kout[r] = untwiddle_rt<UK>(sk[s_perm[r]], a.kind, desc);
  }
  RANGE_PROBE_SYNC();
  RANGE_PROBE_STAMP(7);
}

// descending float keys: cub sorts the (nan_bias, value) tuple descending, i.e. NaNs come first in
// DESCENDING row order (sorted_order_radix.cu:41-50,121-131). The stable pass above leaves them
// ascending; reverse that prefix.
__global__ void reverse_nan_prefix_kernel(int32_t* idx, const uint32_t* nan_count)
{
  const uint32_t m = *nan_count;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m / 2; i += stride) {
    int32_t x = idx[i], y = idx[m - 1 - i];
    idx[i] = y;
    idx[m - 1 - i] = x;
  }
}

// ------------------------------------------------------------------------------------------------
// 4. null compaction (single nullable column)
// ------------------------------------------------------------------------------------------------
constexpr int CP_THREADS = 256;
constexpr int CP_ROWS    = 2048;  // rows per CTA = 64 mask words

__global__ void __launch_bounds__(CP_THREADS) valid_count_kernel(const uint32_t* __restrict__ mask, int64_t bit_offset,
                                                                  int64_t n, uint32_t* __restrict__ tile_valid)
{
  // each warp counts one tile of CP_ROWS rows
  const int64_t tile = (int64_t)blockIdx.x * (CP_THREADS / 32) + (threadIdx.x >> 5);
  const int64_t ntiles = (n + CP_ROWS - 1) / CP_ROWS;
  if (tile >= ntiles) return;
  const int64_t row0 = tile * CP_ROWS;
  const int64_t last_word = (bit_offset + n - 1) >> 5;
  uint32_t c = 0;
  for (int w = lane_id(); w < CP_ROWS / 32; w += 32) {
    int64_t r = row0 + (int64_t)w * 32;
    if (r < n) {
      uint32_t bits = load_mask_word_unaligned(mask, bit_offset + r, last_word);
      int64_t rem = n - r;
      if (rem < 32) bits &= (1u << rem) - 1u;
      c += __popc(bits);
    }
  }
  c = warp_sum(c);
  if (lane_id() == 0) tile_valid[tile] = c;
}

// single-CTA exclusive scan over tile counts (ntiles <= ~1M); also writes total
__global__ void __launch_bounds__(1024) scan_tiles_kernel(uint32_t* __restrict__ tile_valid, int64_t ntiles,
                                                          uint32_t* __restrict__ total)
{
  __shared__ uint32_t wsum[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t b = 0; b < ntiles; b += 1024) {
    int64_t i = b + threadIdx.x;
    uint32_t v = i < ntiles ? tile_valid[i] : 0;
    uint32_t inc = warp_inclusive_sum(v);
    if (lane_id() == 31) wsum[threadIdx.x >> 5] = inc;
    __syncthreads();
    uint32_t woff = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += wsum[w];
    uint32_t c = carry;
    if (i < ntiles) tile_valid[i] = c + woff + inc - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + woff + inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

template <typename UK>
__global__ void __launch_bounds__(CP_THREADS) compact_kernel(const UK* __restrict__ keys, const uint32_t* __restrict__ mask,
                                                             int64_t bit_offset, int64_t n, int kind, UK desc_mask,
                                                             const uint32_t* __restrict__ tile_valid_excl,
                                                             UK* __restrict__ out_keys, int32_t* __restrict__ out_valid_idx,
                                                             int32_t* __restrict__ out_null_idx)
{
  __shared__ uint32_t wcount[CP_ROWS / 32];  // valid count per 32-row word
  const int64_t tile = blockIdx.x;
  const int64_t row0 = tile * CP_ROWS;
  const int64_t last_word = (bit_offset + n - 1) >> 5;
  const uint32_t vbase = tile_valid_excl[tile];
  const uint32_t nbase = (uint32_t)row0 - vbase;
  // 64 words per tile; thread t<64 loads word t
  uint32_t bits = 0;
  if (threadIdx.x < CP_ROWS / 32) {
    int64_t r = row0 + (int64_t)threadIdx.x * 32;
    if (r < n) {
      bits = load_mask_word_unaligned(mask, bit_offset + r, last_word);
      int64_t rem = n - r;
      if (rem < 32) bits &= (1u << rem) - 1u;
    }
    wcount[threadIdx.x] = __popc(bits);
  }
  __syncthreads();
  // each warp handles words warp, warp+8, ... ; prefix of earlier words by summing smem (<=64 adds)
  for (int w = threadIdx.x >> 5; w < CP_ROWS / 32; w += CP_THREADS / 32) {
    int64_t r = row0 + (int64_t)w * 32 + lane_id();
    uint32_t before = 0;
    for (int j = lane_id(); j < w; j += 32) before += wcount[j];
    before = warp_sum(before);
    bool in = r < n;
    bool valid = false;
    if (in) {
      // recompute this word's bits (cheap, L1-resident)
      uint32_t wb = load_mask_word_unaligned(mask, bit_offset + row0 + (int64_t)w * 32, last_word);
      valid = (wb >> lane_id()) & 1u;
    }
    unsigned vb = __ballot_sync(0xffffffffu, valid);
    unsigned nb = __ballot_sync(0xffffffffu, in && !valid);
    if (valid) {
      uint32_t o = vbase + before + __popc(vb & lanemask_lt());
      out_keys[o]      = twiddle_rt<UK>(keys[r], kind, desc_mask);
      out_valid_idx[o] = (int32_t)r;
    } else if (in) {
      uint32_t o = nbase + ((uint32_t)w * 32 - before) + __popc(nb & lanemask_lt());
      out_null_idx[o] = (int32_t)r;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host driver
// ------------------------------------------------------------------------------------------------
// Rows per portion of a one-sweep pass with `tile`-row tiles: whole tiles, and few enough rows for 32-bit positions inside the
// portion. B2_SORT_PORTION=<rows> (test hook) lowers it.
int64_t portion_rows(int tile)
{
  static const int64_t lim = [] {
    const char* e = std::getenv("B2_SORT_PORTION");
    int64_t v = e ? std::atoll(e) : 0;
    if (v <= 0) v = (int64_t(1) << 30) - 16384;
    return v;
  }();
  return std::max<int64_t>(tile, lim / tile * tile);
}

// The one-sweep passes of one call: `passes` passes over n rows, each split into portions. One allocation holds a head that
// zero_head() clears (control block, `hist_bytes` of digit histograms, one tile counter per (pass, portion), `tail_bytes` for
// the caller) and behind it the look-back rows of every (pass, portion), which run() zeroes right before that portion's launch,
// so that passes the plan skips cost nothing (1e9 rows: 163 MB per executed pass instead of 1.3 GB per sort).
// extra_tiles: look-back rows for that many tiles more per (pass, portion) (the estimated-base second pass has up to 256 partial
// tiles in the middle of its sequence).
template <typename UK, typename Shape, typename VT, bool CARRY, bool MIX, bool RANGE = false, bool EST = false>
struct onesweep_passes {
  static constexpr int TILE = Shape::tile;
  // every instantiation declares the RANGE arrays behind s_misc, only RANGE launches allocate them
  static constexpr size_t SMEM = (sizeof(UK) > sizeof(VT) ? sizeof(UK) : sizeof(VT)) * (size_t)TILE +
                                 sizeof(uint32_t) * (2 * (Shape::threads / 32) * RADIX + 3 * RADIX + 16) +
                                 (RANGE ? (sizeof(UK) + 2 * sizeof(void*)) * RADIX + (size_t)TILE : 0);
  static constexpr size_t CTL_BYTES = (sizeof(sort_ctl) + 255) / 256 * 256;
  const int64_t n, plim, nportions;
  const size_t hist_bytes, cnt_bytes, head_bytes, status_per;
  dbuf work;

  onesweep_passes(int64_t rows, int passes, size_t hist, size_t tail_bytes, cudaStream_t stream, int extra_tiles = 0)
    : n(rows), plim(portion_rows(TILE)), nportions((n + plim - 1) / plim), hist_bytes(hist),
      cnt_bytes((sizeof(uint32_t) * passes * nportions + 255) / 256 * 256), head_bytes(CTL_BYTES + hist_bytes + cnt_bytes + tail_bytes),
      status_per(sizeof(uint32_t) * RADIX * (size_t)((std::min(n, plim) + TILE - 1) / TILE + extra_tiles)),
      work(head_bytes + status_per * passes * nportions, stream)
  {
    static std::atomic<uint64_t> attr_done{0};  // per device: the opt-in to > 48 KB of dynamic shared memory is a per-context setting
    once_per_device(attr_done, [] {
      B2_CUDA_TRY(cudaFuncSetAttribute(onesweep_kernel<UK, Shape, VT, CARRY, MIX, RANGE, EST>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)SMEM));
    });
  }
  sort_ctl* ctl() const { return work.as<sort_ctl>(); }
  uint32_t* hist() const { return reinterpret_cast<uint32_t*>(work.as<char>() + CTL_BYTES); }
  void* tail() const { return work.as<char>() + CTL_BYTES + hist_bytes + cnt_bytes; }
  void zero_head(cudaStream_t stream) const { B2_CUDA_TRY(cudaMemsetAsync(work.ptr, 0, head_bytes, stream)); }

  // pass number `slot` of this call, portion by portion (a.pass is the digit it sorts by)
  void run(pass_args& a, int slot, const char* scope, cudaStream_t stream, int extra_tiles = 0) const
  {
    for (int64_t q = 0; q < nportions; ++q) {
      const int64_t start = q * plim;
      const int64_t pn = std::min(plim, n - start);
      const int64_t ntiles = (pn + TILE - 1) / TILE + extra_tiles;
      a.portion_start = start;
      a.portion_n = (uint32_t)pn;
      a.portion_parity = (int)(q & 1);
      a.has_next_portion = q + 1 < nportions;
      a.status = reinterpret_cast<uint32_t*>(work.as<char>() + head_bytes + (size_t)(slot * nportions + q) * status_per);
      a.tile_counter = reinterpret_cast<uint32_t*>(work.as<char>() + CTL_BYTES + hist_bytes) + slot * nportions + q;
      B2_CUDA_TRY(cudaMemsetAsync(a.status, 0, sizeof(uint32_t) * RADIX * (size_t)ntiles, stream));
      prof_scope ps(scope, stream);
      B2_LAUNCH((onesweep_kernel<UK, Shape, VT, CARRY, MIX, RANGE, EST>), (unsigned)ntiles, Shape::threads + 32 * LBW, SMEM, stream, a);
    }
  }
};

// B2_SORT_HYBRID=0 switches the partial-LSD + fix-up plan off; B2_SORT_HYBRID_MIN=<rows> moves its lower size limit
// (tests run it on small inputs).
// range tier of the hybrid plan: from this size on by default (measured on the H100: DESIGN.md §4.1); B2_SORT_RANGE=0 / 1
// (test hook) forces it off / on wherever the plan finds it feasible
constexpr int64_t RANGE_MIN_ROWS = int64_t(1) << 27;
int range_env()
{
  static int v = [] {
    const char* e = std::getenv("B2_SORT_RANGE");
    return e ? (std::atoi(e) != 0 ? 1 : 0) : -1;
  }();
  return v;
}

int64_t hybrid_min_rows()
{
  static int64_t v = [] {
    const char* off = std::getenv("B2_SORT_HYBRID");
    if (off && std::atoi(off) == 0) return INT64_MAX;
    const char* e = std::getenv("B2_SORT_HYBRID_MIN");
    return e ? (int64_t)std::atoll(e) : (int64_t(1) << 16);
  }();
  return v;
}

// ---- range tier with estimated bases (no histogram) ---------------------------------------------------------------------------
// Buffers: keys 0 raw -> 1 (first window buffer) -> 2 (second), payload implicit / carried -> 2 -> 1; the range sort reads key 2 /
// payload 1 and writes payload 0 (pairs) or key 1, which the host then points at the keys-only output.
__global__ void range_est_plan_kernel(sort_ctl* ctl, uint32_t cap)
{
  const int d = threadIdx.x;  // 256 threads
  ctl->base[0][6][d] = (uint32_t)d * cap;
  ctl->base[0][7][d] = (uint32_t)d * cap;
  if (d < 8) {
    pass_plan pl{};
    pl.trivial = d < 6;
    if (d >= 6) {
      pl.key_src = d == 6 ? 0 : 1;
      pl.key_dst = d == 6 ? 1 : 2;
      pl.idx_src = d == 6 ? -1 : 2;
      pl.idx_dst = d == 6 ? 2 : 1;
      pl.last    = d == 7;
      pl.hybrid  = 1;
    }
    ctl->plan[d] = pl;
  }
  if (d == 0) {
    ctl->any_pass    = 2;
    ctl->hybrid      = 1;
    ctl->range       = 1;
    ctl->range_shift = 48;
    ctl->range_bits  = 16;
    ctl->fix_shift   = 48;
    ctl->fix_key_buf = 2;
    ctl->fix_idx_buf = 1;
    ctl->overflow    = 0;
  }
}

// Tiles of the second pass from the first pass's window ends: tile_first[d] = sum_{e<d} ceil(cnt6[e] / tile), tile t = (window d,
// offset) reads rows [d * cap + offset, + min(tile, cnt6[d] - offset)); the last tile is flagged. Counts are clamped to cap, so an
// overflowed window never sends a reader past its buffer. Entries past the last tile stay zero (zero_head).
__global__ void range_est_tiles_kernel(const sort_ctl* ctl, uint32_t cap, int tile, uint2* __restrict__ tiles)
{
  __shared__ uint32_t s_wsum[RADIX / 32];
  const int d = threadIdx.x;  // 256 threads
  const uint32_t cnt = min(ctl->base[1][6][d] - (uint32_t)d * cap, cap);
  const uint32_t nt = (cnt + (uint32_t)tile - 1) / (uint32_t)tile;
  const uint32_t inc = warp_inclusive_sum(nt);
  if ((d & 31) == 31) s_wsum[d >> 5] = inc;
  __syncthreads();
  uint32_t first = inc - nt, total = 0;
  for (int w = 0; w < RADIX / 32; ++w) {
    first += w < (d >> 5) ? s_wsum[w] : 0u;
    total += s_wsum[w];
  }
  for (uint32_t k = 0; k < nt; ++k) {
    const uint32_t off = k * (uint32_t)tile;
    const uint32_t t = first + k;
    tiles[t] = make_uint2((uint32_t)d * cap + off, min((uint32_t)tile, cnt - off) | (t + 1 == total ? 0x80000000u : 0u));
  }
}

// The range tier's two one-sweep passes into estimated digit windows of `cap` rows (digit d of pass p owns rows [d * cap, (d + 1) *
// cap) of its output), then range_sort_kernel from the second pass's windows into the dense output. k1 / k2 / v1 / v2 hold 256 * cap
// rows each (v*: pairs only; v2 is the second pass's destination). Returns false when a window, a range or a bucket overflowed:
// the output is then incomplete and the caller runs the exact plan.
template <typename UK, typename Shape, typename VT, bool CARRY>
bool run_est_range(const UK* raw_keys, UK* keys_out, UK* k1, UK* k2, int32_t* idx_out, int32_t* v1, int32_t* v2, int64_t n, uint32_t cap,
                   int kind, UK desc_mask, bool pairs, const void* val_in, cudaStream_t stream)
{
  static_assert(sizeof(UK) == 8, "the estimated-base range tier sorts 64-bit keys");
  constexpr int TILE = Shape::tile;
  const int64_t ntiles = (n + TILE - 1) / TILE + RADIX;  // window ends add at most 256 partial tiles
  // the look-back rows behind the tile table are read and written in 16-byte groups: keep them 256-byte aligned
  const size_t table_bytes = (sizeof(uint2) * ntiles + 255) / 256 * 256;
  const onesweep_passes<UK, Shape, VT, CARRY, false, false, true> passes(n, 2, 0, table_bytes, stream, RADIX);
  {
    static std::atomic<uint64_t> attr_done{0};
    once_per_device(attr_done, [] {
      B2_CUDA_TRY(cudaFuncSetAttribute(range_sort_kernel<VT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)range_sort_smem(true)));
    });
  }
  sort_ctl* const ctl = passes.ctl();
  uint2* const tiles = static_cast<uint2*>(passes.tail());
  passes.zero_head(stream);
  B2_LAUNCH(range_est_plan_kernel, 1, RADIX, 0, stream, ctl, cap);
  pass_args a{};
  a.key_bufs[0] = raw_keys;
  a.key_bufs[1] = k1;
  a.key_bufs[2] = k2;
  a.idx_bufs[0] = idx_out;
  a.idx_bufs[1] = v2;
  a.idx_bufs[2] = v1;
  a.ctl = ctl;
  a.kind = kind;
  a.pairs = pairs ? 1 : 0;
  a.val_in = val_in;
  a.desc_mask = (uint64_t)desc_mask;
  a.est_cap = cap;
  a.pass = 6;
  passes.run(a, 0, "onesweep", stream);
  B2_LAUNCH(range_est_tiles_kernel, 1, RADIX, 0, stream, (const sort_ctl*)ctl, cap, TILE, tiles);
  a.pass = 7;
  a.est_tiles = tiles;
  passes.run(a, 1, "onesweep", stream, RADIX);
  a.key_bufs[1] = keys_out;  // the range sort's keys-only destination
  dbuf bounds(sizeof(uint32_t) * 3 * RADIX * RADIX, stream);
  {
    prof_scope ps("range_bounds", stream);
    B2_LAUNCH(range_est_bounds_kernel, RADIX, RADIX, 0, stream, a, cap, bounds.as<uint32_t>());
  }
  {
    prof_scope ps("segment_fix", stream);  // the range sort
    B2_LAUNCH((range_sort_kernel<VT, true>), RADIX * RADIX, 1 << range_log_threads<true>, range_sort_smem(true), stream, a, bounds.as<const uint32_t>());
  }
  uint32_t overflow = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&overflow, &ctl->overflow, sizeof(overflow), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  return overflow == 0;
}

// Sort `n` keys.
//  raw_keys != nullptr : keys are the user's raw column (twiddled on load, implicit row ids)
//  raw_keys == nullptr : keys are pre-twiddled in bufA with explicit row ids in idx buffer pre_idx_buf
//  pairs: idx_out receives the permutation ; keys-only: bufA is the OUTPUT, bufB the temp.
template <typename UK, typename Shape, typename VT = uint32_t, bool CARRY = false, bool MIX = false>
void run_radix_cfg(const UK* raw_keys, UK* bufA, UK* bufB, int32_t* idx_out, int32_t* idx_tmp, int32_t* idx_tmp2, int pre_idx_buf, int64_t n,
                   int kind, bool descending, bool pairs, cudaStream_t stream, int first_pass = 0, int last_pass = 7,
                   bool keep_keys = false, const void* val_in = nullptr, uint32_t* top_digit_base_out = nullptr, uint32_t est_cap = 0,
                   void* est_buf = nullptr)
{
  constexpr int NP = sizeof(UK);
  const bool raw = raw_keys != nullptr;
  const UK desc_mask = descending ? ~UK(0) : UK(0);

  // est_cap != 0 (est_range_capacity): the range tier with estimated bases first. Its windows hold 256 * est_cap rows: bufB and
  // est_buf (keys-only), bufA, bufB, idx_tmp and est_buf (pairs) are that large. An overflow falls back to the exact plan below.
  if constexpr (sizeof(UK) == 8 && !MIX) {
    if (est_cap != 0 && raw && first_pass == 0 && last_pass >= NP - 1 && !keep_keys) {
      const bool done =
        pairs ? run_est_range<UK, Shape, VT, CARRY>(raw_keys, bufA, bufA, bufB, idx_out, static_cast<int32_t*>(est_buf), idx_tmp, n, est_cap,
                                                    kind, desc_mask, true, val_in, stream)
              : run_est_range<UK, Shape, VT, CARRY>(raw_keys, bufA, static_cast<UK*>(est_buf), bufB, nullptr, nullptr, nullptr, n, est_cap,
                                                    kind, desc_mask, false, val_in, stream);
      if (done) return;
    }
  }

  const onesweep_passes<UK, Shape, VT, CARRY, MIX> passes(n, NP, sizeof(uint32_t) * NP * RADIX, 0, stream);
  sort_ctl* const ctl = passes.ctl();
  uint32_t* const ghist = passes.hist();
  if constexpr (sizeof(UK) == 8 && !MIX) {
    static std::atomic<uint64_t> attr_done{0};
    once_per_device(attr_done, [] {
      B2_CUDA_TRY(cudaFuncSetAttribute(range_sort_kernel<VT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)range_sort_smem(false)));
    });
  }

  // Hybrid plan (64-bit raw keys, full sort): LSD passes over the top digits only, then segment_fix_kernel. The plan
  // kernel decides on the device; the host learns the outcome from one 4-byte read-back after the fix-up.
  bool try_hybrid = sizeof(UK) == 8 && !MIX && raw && first_pass == 0 && last_pass >= NP - 1 && !keep_keys && n >= hybrid_min_rows();
  // Its range tier (range_sort_kernel) from RANGE_MIN_ROWS rows on; B2_SORT_RANGE=0 / 1 (test hook) switches it off / on at
  // any size. The host reads the plan back to size the range launches.
  const int force_range = range_env();
  bool try_range = try_hybrid && force_range != 0 && (force_range == 1 || n >= RANGE_MIN_ROWS);

  for (;;) {
    passes.zero_head(stream);
    {
      int grid = (int)std::min<int64_t>((n + 512 * 16 - 1) / (512 * 16), num_sms() * 4);
      grid = std::max(grid, 1);
      const UK* hkeys = raw ? raw_keys : bufA;
      uint32_t* nanp = (raw && kind == (int)key_kind::FLOAT) ? &ctl->nan_count : nullptr;
      // digits that can be executed at all: [first_pass, last_pass]
      const uint32_t span_mask = ((last_pass >= NP - 1 ? (1u << NP) : (1u << (last_pass + 1))) - 1u) & ~((1u << std::max(first_pass, 0)) - 1u);
      if (try_hybrid) {
        // two-phase: the top four digits first (half the shared-memory atomics); the low four only if the plan needs them
        {
          prof_scope ps("histogram", stream);
          B2_LAUNCH((histogram_kernel<UK, MIX>), grid, 512, 0, stream, hkeys, n, raw ? 1 : 0, kind, desc_mask, ghist, nanp, 0xf0u,
                    (const int32_t*)nullptr, &ctl->vary);
        }
        B2_LAUNCH(plan_kernel, 1, RADIX, 0, stream, ghist, NP, (uint32_t)n, raw ? 1 : 0, pre_idx_buf, ctl, first_pass, last_pass, 1, 1,
                  try_range ? 1 : 0);
        {
          prof_scope ps("histogram", stream);
          B2_LAUNCH((histogram_kernel<UK, MIX>), grid, 512, 0, stream, hkeys, n, raw ? 1 : 0, kind, desc_mask, ghist, (uint32_t*)nullptr, 0x0fu,
                    &ctl->need_low, (unsigned long long*)nullptr);
        }
        B2_LAUNCH(plan_kernel, 1, RADIX, 0, stream, ghist, NP, (uint32_t)n, raw ? 1 : 0, pre_idx_buf, ctl, first_pass, last_pass, 1, 2,
                  try_range ? 1 : 0);
      } else {
        {
          prof_scope ps("histogram", stream);
          B2_LAUNCH((histogram_kernel<UK, MIX>), grid, 512, 0, stream, hkeys, n, raw ? 1 : 0, kind, desc_mask, ghist, nanp, span_mask,
                    (const int32_t*)nullptr, (unsigned long long*)nullptr);
        }
        B2_LAUNCH(plan_kernel, 1, RADIX, 0, stream, ghist, NP, (uint32_t)n, raw ? 1 : 0, pre_idx_buf, ctl, first_pass, last_pass, 0, 0);
      }
    }

    {
      static const int force_fix = [] {  // test hook: B2_SORT_FIX_FAST=0/1 overrides the plan's choice of the fix-up flavour
        const char* e = std::getenv("B2_SORT_FIX_FAST");
        return e ? (std::atoi(e) != 0 ? 1 : 0) : -1;
      }();
      if (force_fix >= 0 && try_hybrid) B2_LAUNCH(set_fix_fast_kernel, 1, 1, 0, stream, ctl, force_fix);
    }
    pass_args a{};
    a.key_bufs[0] = raw_keys;
    a.key_bufs[1] = bufA;
    a.key_bufs[2] = bufB;
    a.idx_bufs[0] = idx_out;
    a.idx_bufs[1] = idx_tmp;
    a.idx_bufs[2] = idx_tmp2;
    a.ctl = ctl;
    a.kind = kind;
    a.pairs = pairs ? 1 : 0;
    a.keep_keys = keep_keys ? 1 : 0;
    a.val_in = val_in;
    a.desc_mask = (uint64_t)desc_mask;
    // Large inputs: read the plan back (one small copy + sync, ~20 us against milliseconds of passes) and launch only the
    // passes it executes — a skipped pass would otherwise start one CTA per tile just to return (163 K CTAs at 1e9 rows).
    // Small inputs launch every digit's kernel and stay free of host synchronisation.
    uint32_t skip_mask = 0;
    bool plan_hybrid = true;
    int range_bits = 0;  // range tier: the range id has range_bits bits
    static const int64_t readback_min = [] {
      const char* e = std::getenv("B2_SORT_PLAN_READBACK_MIN");  // test hook
      return e ? (int64_t)std::atoll(e) : (int64_t(1) << 22);
    }();
    if (n >= readback_min || try_range) {
      pass_plan hp[8];
      int32_t hflag = 0, hrange[3] = {0, 0, 0};  // ctl->range, range_shift, range_bits
      B2_CUDA_TRY(cudaMemcpyAsync(hp, &ctl->plan[0], sizeof(pass_plan) * 8, cudaMemcpyDeviceToHost, stream));
      B2_CUDA_TRY(cudaMemcpyAsync(&hflag, &ctl->hybrid, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
      if (try_range) B2_CUDA_TRY(cudaMemcpyAsync(hrange, &ctl->range, sizeof(hrange), cudaMemcpyDeviceToHost, stream));
      B2_CUDA_TRY(cudaStreamSynchronize(stream));
      for (int p = 0; p < NP; ++p)
        if (hp[p].trivial) skip_mask |= 1u << p;
      plan_hybrid = hflag != 0;
      range_bits = hrange[0] ? hrange[2] : 0;
    }
    for (int p = std::max(0, first_pass); p < NP && p <= last_pass; ++p) {
      if ((skip_mask >> p) & 1u) continue;
      a.pass = p;
      passes.run(a, p, "onesweep", stream);
    }
    if constexpr (sizeof(UK) == 8 && !MIX) {
      if (try_hybrid && plan_hybrid && range_bits) {
        const int nranges = 1 << range_bits;
        dbuf bounds(sizeof(uint32_t) * (nranges + 1), stream);
        {
          prof_scope ps("range_bounds", stream);
          B2_LAUNCH(range_bounds_kernel, (nranges + 256) / 256, 256, 0, stream, a, n, bounds.as<uint32_t>(), nranges);
        }
        prof_scope ps("segment_fix", stream);  // the range sort replaces the segment fix-up
        B2_LAUNCH((range_sort_kernel<VT>), nranges, RANGE_THREADS, range_sort_smem(false), stream, a, bounds.as<const uint32_t>());
      } else if (try_hybrid && plan_hybrid) {
        const int64_t ntiles = (n + FIX_TILE - 1) / FIX_TILE;
        const int grid = (int)std::min<int64_t>(ntiles, num_sms() * 8);
        prof_scope ps("segment_fix", stream);
        B2_LAUNCH((segment_fix_kernel<UK, VT, 0>), grid, FIX_THREADS, 0, stream, a, n);  // the plan's ctl->fix_fast picks one of the two
        B2_LAUNCH((segment_fix_kernel<UK, VT, 3>), grid, FIX_THREADS, 0, stream, a, n);
      }
    }
    {
      int grid = (int)std::min<int64_t>((n + 255) / 256, num_sms() * 8);
      B2_LAUNCH((finalize_kernel<UK, MIX>), std::max(grid, 1), 256, 0, stream, a, n, raw ? 1 : 0, pre_idx_buf, CARRY ? (int)sizeof(VT) : 0);
    }
    if (!try_hybrid || !plan_hybrid) break;
    uint32_t overflow = 0;
    B2_CUDA_TRY(cudaMemcpyAsync(&overflow, &ctl->overflow, sizeof(overflow), cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    if (!overflow) break;
    if (range_bits) {  // a range did not fit (or held unequal keys beyond the walk window): the hybrid plan without the range tier
      try_range = false;
      continue;
    }
    try_hybrid = false;  // a segment was longer than the fix-up window (digits not independent): full LSD sort of the untouched input
  }
  if (pairs && raw && kind == (int)key_kind::FLOAT && descending) {
    B2_LAUNCH(reverse_nan_prefix_kernel, num_sms() * 4, 256, 0, stream, idx_out, &ctl->nan_count);
  }
  if (top_digit_base_out)  // start offset of every value of the most significant digit (partition boundaries)
    B2_CUDA_TRY(cudaMemcpyAsync(top_digit_base_out, &ctl->base[0][NP - 1][0], sizeof(uint32_t) * RADIX, cudaMemcpyDeviceToDevice, stream));
}

// tile shape of the row-id passes (and of the payload-carrying ones, except 8-byte keys with 8-byte payloads)
template <typename UK>
using key_tile = std::conditional_t<sizeof(UK) == 8, tile_384x16, tile_512x16>;

template <typename UK>
void run_radix(const UK* raw_keys, UK* bufA, UK* bufB, int32_t* idx_out, int32_t* idx_tmp, int pre_idx_buf, int64_t n,
               int kind, bool descending, bool pairs, cudaStream_t stream, int32_t* idx_tmp2 = nullptr, uint32_t est_cap = 0,
               void* est_buf = nullptr)
{
  run_radix_cfg<UK, key_tile<UK>>(raw_keys, bufA, bufB, idx_out, idx_tmp, idx_tmp2, pre_idx_buf, n, kind, descending, pairs, stream, 0, 7,
                                  false, nullptr, nullptr, est_cap, est_buf);
}

// The 64-bit key kernels are instantiated here, ahead of the narrower key types that the sort entry points below instantiate.
// How nvcc inlines the device helpers shared by the histogram, finalize and gather kernels depends on the order in which the
// kernels are instantiated; this order gives every kernel the code the sort was measured with.
template void run_radix_cfg<uint64_t, tile_384x16>(const uint64_t*, uint64_t*, uint64_t*, int32_t*, int32_t*, int32_t*, int, int64_t, int, bool,
                                                   bool, cudaStream_t, int, int, bool, const void*, uint32_t*, uint32_t, void*);

}  // namespace

// Stable partial sort of n 64-bit packed join keys by the two most significant bytes of mix64(key) (passes 6 and 7
// only): the kernels apply mix64 on load (histogram of the two needed digits only), so keys_out / idx_out receive
// mix64(key) and the original positions grouped by its top 16 bits. Used by the partitioned join (radix_join.cu).
void radix_partition_top16_mix(const uint64_t* packed_keys, int64_t n, uint64_t* keys_out, int32_t* idx_out, cudaStream_t stream)
{
  dbuf b(sizeof(uint64_t) * n, stream), it(sizeof(int32_t) * n, stream);
  run_radix_cfg<uint64_t, tile_384x16, uint32_t, false, true>(packed_keys, keys_out, b.as<uint64_t>(), idx_out, it.as<int32_t>(), nullptr, 0,
                                                              n, (int)key_kind::UNSIGNED, false, true, stream, 6, 7, true);
}

// One stable partition pass by the top byte of mix64(key), carrying one 4- or 8-byte payload column next to the mixed
// keys (hash groupby: rows of a group meet in one of 256 partitions; mix64 is undone with unmix64). part_base[d] =
// first row of partition d.
void radix_partition_mix_carry(const uint64_t* keys, const void* vals, int val_bytes, int64_t n, uint64_t* mixed_keys_out, void* vals_out,
                               uint32_t* part_base, cudaStream_t stream)
{
  dbuf b(sizeof(uint64_t) * n, stream), vt((size_t)val_bytes * n, stream);
  if (val_bytes == 8)
    run_radix_cfg<uint64_t, tile_384x16, uint64_t, true, true>(keys, mixed_keys_out, b.as<uint64_t>(), static_cast<int32_t*>(vals_out),
                                                                vt.as<int32_t>(), nullptr, 0, n, (int)key_kind::UNSIGNED, false, true, stream,
                                                                7, 7, true, vals, part_base);
  else
    run_radix_cfg<uint64_t, tile_384x16, uint32_t, true, true>(keys, mixed_keys_out, b.as<uint64_t>(), static_cast<int32_t*>(vals_out),
                                                                vt.as<int32_t>(), nullptr, 0, n, (int)key_kind::UNSIGNED, false, true, stream,
                                                                7, 7, true, vals, part_base);
}

namespace {
// plan of the single executed pass `pass` with estimated bases: digit d starts at d * cap
__global__ void est_plan_kernel(sort_ctl* ctl, int pass, uint32_t cap)
{
  const int d = threadIdx.x;  // 256 threads
  ctl->base[0][pass][d] = (uint32_t)d * cap;
  if (d < 8) {
    pass_plan pl{};
    pl.trivial = d != pass;
    if (d == pass) {
      pl.key_src = 0;
      pl.idx_src = -1;
      pl.key_dst = 1;
      pl.idx_dst = 0;
      pl.last    = 1;
      pl.hybrid  = 0;
    }
    ctl->plan[d] = pl;
  }
  if (d == 0) {
    ctl->any_pass = 1;
    ctl->hybrid   = 0;
    ctl->overflow = 0;
  }
}

// MIX: counts[b] = sampled rows (every `stride`-th) whose mix64(key) has top byte b. Otherwise the keys are twiddled as the sort's
// passes twiddle them (kind, desc_mask) and counts[b] / counts[256 + b] count digit 7 / digit 6 = b.
template <bool MIX = true>
__global__ void __launch_bounds__(256) est_sample_kernel(const uint64_t* __restrict__ keys, int64_t n, int64_t stride, unsigned int* __restrict__ counts,
                                                         int kind = 0, uint64_t desc_mask = 0)
{
  constexpr int NC = MIX ? 1 : 2;
  __shared__ unsigned int sh[NC * RADIX];
  for (int c = 0; c < NC; ++c) sh[c * RADIX + threadIdx.x] = 0;
  __syncthreads();
  const int64_t m = (n + stride - 1) / stride;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    if constexpr (MIX) {
      atomicAdd(&sh[(unsigned)(mix64(keys[i * stride]) >> 56)], 1u);
    } else {
      const uint64_t k = twiddle_rt<uint64_t>(keys[i * stride], kind, desc_mask);
      atomicAdd(&sh[(unsigned)(k >> 56)], 1u);
      atomicAdd(&sh[RADIX + (unsigned)((k >> 48) & 255u)], 1u);
    }
  }
  __syncthreads();
  for (int c = 0; c < NC; ++c)
    if (sh[c * RADIX + threadIdx.x]) atomicAdd(&counts[c * RADIX + threadIdx.x], sh[c * RADIX + threadIdx.x]);
}

template <typename VT>
bool est_pass_impl(const uint64_t* keys, const void* vals, int64_t n, uint32_t cap, uint64_t* mixed_keys_out, void* vals_out, uint32_t* part_base,
                   uint32_t* part_end, cudaStream_t stream)
{
  constexpr int PASS = 7;
  const onesweep_passes<uint64_t, tile_384x16, VT, true, true> passes(n, 1, 0, 0, stream);  // one portion: n <= portion_rows()
  sort_ctl* const ctl = passes.ctl();
  passes.zero_head(stream);
  B2_LAUNCH(est_plan_kernel, 1, RADIX, 0, stream, ctl, PASS, cap);
  pass_args a{};
  a.key_bufs[0] = keys;
  a.key_bufs[1] = mixed_keys_out;
  a.key_bufs[2] = mixed_keys_out;
  a.idx_bufs[0] = static_cast<int32_t*>(vals_out);
  a.idx_bufs[1] = static_cast<int32_t*>(vals_out);
  a.idx_bufs[2] = static_cast<int32_t*>(vals_out);
  a.ctl = ctl;
  a.kind = (int)key_kind::UNSIGNED;
  a.pairs = 1;
  a.keep_keys = 1;
  a.val_in = vals;
  a.desc_mask = 0;
  a.pass = PASS;
  a.est_cap = cap;
  passes.run(a, 0, "onesweep", stream);
  B2_CUDA_TRY(cudaMemcpyAsync(part_base, &ctl->base[0][PASS][0], sizeof(uint32_t) * RADIX, cudaMemcpyDeviceToDevice, stream));
  B2_CUDA_TRY(cudaMemcpyAsync(part_end, &ctl->base[1][PASS][0], sizeof(uint32_t) * RADIX, cudaMemcpyDeviceToDevice, stream));
  uint32_t overflow = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&overflow, &ctl->overflow, sizeof(overflow), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  return overflow == 0;
}
}  // namespace

// Rows per partition to reserve for the histogram-free partition pass below, or 0 when a strided sample of the keys says the
// partitions are too uneven for it (few distinct keys, hot keys): max sampled share + 5 sigma of the sampling noise must fit.
uint32_t radix_partition_est_capacity(const uint64_t* keys, int64_t n, cudaStream_t stream)
{
  static const int64_t min_rows = [] {
    const char* e = std::getenv("B2_GROUPBY_EST_MIN");  // test hook
    return e ? (int64_t)std::atoll(e) : (int64_t(1) << 22);
  }();
  if (n < min_rows || n > portion_rows(tile_384x16::tile)) return 0;
  if (const char* e = std::getenv("B2_GROUPBY_EST_CAP")) return (uint32_t)std::max(1, std::atoi(e));  // test hook: forces the overflow fallback
  const int64_t want = int64_t(1) << 20;
  const int64_t stride = std::max<int64_t>(1, n / want);
  const int64_t m = (n + stride - 1) / stride;
  dbuf cnt(sizeof(unsigned int) * RADIX, stream);
  B2_CUDA_TRY(cudaMemsetAsync(cnt.ptr, 0, cnt.bytes, stream));
  B2_LAUNCH((est_sample_kernel<true>), num_sms() * 4, 256, 0, stream, keys, n, stride, cnt.as<unsigned int>(), 0, (uint64_t)0);
  unsigned int h[RADIX];
  B2_CUDA_TRY(cudaMemcpyAsync(h, cnt.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  unsigned int mx = 0;
  for (int d = 0; d < RADIX; ++d) mx = std::max(mx, h[d]);
  const double cap = (double)(n / RADIX) * 1.25 + 4096.0;
  const double worst = ((double)mx + 5.0 * std::sqrt((double)mx) + 1.0) * ((double)n / (double)m);
  if (worst > cap || cap * RADIX >= 4.0e9) return 0;
  return (uint32_t)cap;
}

// radix_partition_mix_carry without the histogram: the pass runs with estimated bases (partition d owns rows [d * cap, (d + 1) * cap) of
// the outputs, which hold 256 * cap rows) and reports the exact end of every partition in part_end[d]. Returns false when a partition
// overflowed its range (the outputs are then incomplete: run radix_partition_mix_carry).
bool radix_partition_mix_carry_est(const uint64_t* keys, const void* vals, int val_bytes, int64_t n, uint32_t cap, uint64_t* mixed_keys_out,
                                   void* vals_out, uint32_t* part_base, uint32_t* part_end, cudaStream_t stream)
{
  if (val_bytes == 8) return est_pass_impl<uint64_t>(keys, vals, n, cap, mixed_keys_out, vals_out, part_base, part_end, stream);
  return est_pass_impl<uint32_t>(keys, vals, n, cap, mixed_keys_out, vals_out, part_base, part_end, stream);
}

namespace {
// bucket b of a key = number of splitters <= key (twiddled order); counts[b] += rows of bucket b
template <typename UK>
__global__ void __launch_bounds__(512) range_count_kernel(const UK* __restrict__ keys, int64_t n, int kind, const UK* __restrict__ splitters, int P,
                                                          unsigned long long* __restrict__ counts)
{
  __shared__ UK sp[RADIX];
  __shared__ unsigned int cnt[RADIX];
  for (int i = threadIdx.x; i < RADIX; i += blockDim.x) {
    sp[i]  = (splitters != nullptr && i < P - 1) ? splitters[i] : ~UK(0);
    cnt[i] = 0;
  }
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const UK k = twiddle_rt<UK>(ld_stream(keys + i), kind, UK(0));
    int lo = 0, hi = P - 1;
    if (splitters == nullptr) lo = hi = (int)range_hash_bucket((uint64_t)k, P);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (sp[mid] <= k) lo = mid + 1;
      else hi = mid;
    }
    atomicAdd(&cnt[lo], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < P; i += blockDim.x)
    if (cnt[i]) atomicAdd(&counts[i], (unsigned long long)cnt[i]);
}
template <typename UK>
__global__ void twiddle_splitters_kernel(const UK* __restrict__ raw, int m, int kind, UK* __restrict__ out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) out[i] = twiddle_rt<UK>(raw[i], kind, UK(0));
}
}  // namespace

// Range partition of one null-free 8-byte integer-like key column (and optionally one null-free 4- / 8-byte payload column) straight
// into P destination buffers — local or PEER memory (sharded sort: the partition pass is the bucket exchange).
// Step 1 (range_partition_counts): rows per bucket, so that the ranks can agree on where each one writes.
// Step 2 (range_partition_scatter): ONE one-sweep pass (stable; per-(tile, bucket) runs of ~6144 / P rows, i.e. 6 KB NVLink
// writes at P = 8) whose digit is the bucket; key_dst[b] / val_dst[b] = address of this rank's first row of bucket b.
void range_partition_counts(const b2_column_view& keys, const void* splitters, int P, int64_t* out_counts, cudaStream_t stream)
{
  using UK = uint64_t;
  const int64_t n = keys.size;
  const int kind = is_signed_id(storage_type(keys.type_id)) ? (int)key_kind::SIGNED : (int)key_kind::UNSIGNED;
  for (int b = 0; b < P; ++b) out_counts[b] = 0;
  if (n == 0) return;
  dbuf cnt(sizeof(unsigned long long) * RADIX, stream), sp(sizeof(UK) * RADIX, stream);
  B2_CUDA_TRY(cudaMemsetAsync(cnt.ptr, 0, cnt.bytes, stream));
  const bool hashed = splitters == nullptr;  // no splitters: hash partition (range_hash_bucket)
  if (P > 1 && !hashed) B2_LAUNCH((twiddle_splitters_kernel<UK>), 1, RADIX, 0, stream, static_cast<const UK*>(splitters), P - 1, kind, sp.as<UK>());
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 511) / 512, num_sms() * 4));
  {
    prof_scope ps("range_count", stream);
    B2_LAUNCH((range_count_kernel<UK>), grid, 512, 0, stream, static_cast<const UK*>(keys.data) + keys.offset, n, kind,
              hashed ? static_cast<const UK*>(nullptr) : sp.as<UK>(), P, cnt.as<unsigned long long>());
  }
  unsigned long long h[RADIX];
  B2_CUDA_TRY(cudaMemcpyAsync(h, cnt.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  for (int b = 0; b < P; ++b) out_counts[b] = (int64_t)h[b];
}

template <typename VT, bool CARRY>
static void range_scatter_impl(const b2_column_view& keys, const void* vals, const void* splitters, int P, void* const* key_dst, void* const* val_dst,
                               cudaStream_t stream)
{
  using UK = uint64_t;
  const int64_t n = keys.size;
  const int kind = is_signed_id(storage_type(keys.type_id)) ? (int)key_kind::SIGNED : (int)key_kind::UNSIGNED;
  // tail: splitters and per-bucket destination pointers
  const onesweep_passes<UK, tile_384x16, VT, CARRY, false, true> passes(n, 1, 0, sizeof(UK) * RADIX + 2 * sizeof(void*) * RADIX, stream);
  passes.zero_head(stream);
  sort_ctl* const ctl = passes.ctl();
  auto* d_split  = static_cast<UK*>(passes.tail());
  auto* d_kdst   = reinterpret_cast<void**>(d_split + RADIX);
  auto* d_vdst   = d_kdst + RADIX;
  if (P > 1 && splitters != nullptr) B2_LAUNCH((twiddle_splitters_kernel<UK>), 1, RADIX, 0, stream, static_cast<const UK*>(splitters), P - 1, kind, d_split);
  B2_CUDA_TRY(cudaMemcpyAsync(d_kdst, key_dst, sizeof(void*) * P, cudaMemcpyHostToDevice, stream));
  if (CARRY) B2_CUDA_TRY(cudaMemcpyAsync(d_vdst, val_dst, sizeof(void*) * P, cudaMemcpyHostToDevice, stream));
  // the plan of the single pass 0: executed, raw keys, last pass (keys-only mode untwiddles what it writes); base = 0: positions
  // count from the start of each bucket's run
  pass_plan pl{};
  pl.trivial = 0; pl.key_src = 0; pl.key_dst = 1; pl.idx_src = -1; pl.idx_dst = 0; pl.last = 1; pl.hybrid = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&ctl->plan[0], &pl, sizeof(pl), cudaMemcpyHostToDevice, stream));

  pass_args a{};
  a.key_bufs[0] = static_cast<const UK*>(keys.data) + keys.offset;
  a.ctl = ctl;
  a.kind = kind;
  a.pairs = CARRY ? 1 : 0;
  a.val_in = vals;
  a.desc_mask = 0;
  a.range_splitters = d_split;
  a.range_key_dst = d_kdst;
  a.range_val_dst = d_vdst;
  a.range_parts = P;
  a.range_hash = (P > 1 && splitters == nullptr) ? 1 : 0;
  a.pass = 0;
  passes.run(a, 0, "range_scatter", stream);
}

void range_partition_scatter(const b2_column_view& keys, const b2_column_view* values, const void* splitters, int P, void* const* key_dst,
                             void* const* val_dst, cudaStream_t stream)
{
  if (keys.size == 0) return;
  if (values == nullptr) return range_scatter_impl<uint32_t, false>(keys, nullptr, splitters, P, key_dst, nullptr, stream);
  const int vw = type_width(values->type_id);
  const void* vin = static_cast<const char*>(values->data) + (size_t)values->offset * vw;
  if (vw == 8) range_scatter_impl<uint64_t, true>(keys, vin, splitters, P, key_dst, val_dst, stream);
  else range_scatter_impl<uint32_t, true>(keys, vin, splitters, P, key_dst, val_dst, stream);
}

namespace {

// B2_SORT_EST=0 / 1 (test hook): the range tier with estimated bases off / on at any size where it applies; B2_SORT_EST_CAP=<rows>
// (test hook) sets its window size without sampling (small values force the overflow fallback).
int est_env()
{
  static int v = [] {
    const char* e = std::getenv("B2_SORT_EST");
    return e ? (std::atoi(e) != 0 ? 1 : 0) : -1;
  }();
  return v;
}

// Rows per digit window of the range tier with estimated bases (run_est_range), or 0 for the exact plan. It applies where the range
// tier is tried (64-bit raw keys, from RANGE_MIN_ROWS rows on), on one portion, and not where the NaN count is needed (row ids of
// descending float keys). A strided sample of 2^20 keys, twiddled as the passes twiddle them, must show both top digits varying, an
// expected range length n * coll6 * coll7 + 5 sigma within RANGE_CAP, and a worst digit share (max sampled count + 5 sigma of the
// sampling noise, scaled to n) within the groupby's bound n / 256 * 1.25 + 4096; cap is that share rounded up to 16 rows, so that
// window starts stay 16-byte aligned for the bulk tile loads, and no larger: the four window buffers hold 256 * cap rows each.
template <typename UK>
uint32_t est_range_capacity(const UK* raw_keys, int64_t n, int kind, bool descending, bool pairs, int tile, cudaStream_t stream)
{
  if constexpr (sizeof(UK) != 8) {
    return 0;
  } else {
    const int force = est_env();
    if (force == 0 || n < 2 || n > portion_rows(tile)) return 0;
    if (pairs && kind == (int)key_kind::FLOAT && descending) return 0;
    if (range_env() == 0 || hybrid_min_rows() == INT64_MAX) return 0;
    if (force != 1 && (n < RANGE_MIN_ROWS || n < hybrid_min_rows())) return 0;
    if (const char* e = std::getenv("B2_SORT_EST_CAP")) return (uint32_t)std::max(1, std::atoi(e));
    const int64_t stride = std::max<int64_t>(1, n >> 20);
    const int64_t m = (n + stride - 1) / stride;
    dbuf cnt(sizeof(unsigned int) * 2 * RADIX, stream);
    B2_CUDA_TRY(cudaMemsetAsync(cnt.ptr, 0, cnt.bytes, stream));
    {
      prof_scope ps("est_sample", stream);
      const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((m + 255) / 256, num_sms() * 4));
      B2_LAUNCH((est_sample_kernel<false>), grid, 256, 0, stream, reinterpret_cast<const uint64_t*>(raw_keys), n, stride, cnt.as<unsigned int>(),
                kind, (uint64_t)(descending ? ~UK(0) : UK(0)));
    }
    unsigned int h[2 * RADIX];
    B2_CUDA_TRY(cudaMemcpyAsync(h, cnt.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    unsigned int mx[2] = {0, 0};
    double coll[2] = {0.0, 0.0};
    for (int c = 0; c < 2; ++c)
      for (int d = 0; d < RADIX; ++d) {
        mx[c] = std::max(mx[c], h[c * RADIX + d]);
        const double f = (double)h[c * RADIX + d] / (double)m;
        coll[c] += f * f;
      }
    if (mx[0] >= (unsigned)m || mx[1] >= (unsigned)m) return 0;  // a top digit is constant in the sample
    const double e = (double)n * coll[0] * coll[1];
    if (e + 5.0 * std::sqrt(e) > (double)RANGE_CAP) return 0;
    const double top = (double)std::max(mx[0], mx[1]);
    const double worst = (top + 5.0 * std::sqrt(top) + 1.0) * ((double)n / (double)m);
    if (worst > (double)(n / RADIX) * 1.25 + 4096.0) return 0;
    const uint64_t cap = ((uint64_t)std::ceil(worst) + 15) / 16 * 16;
    if (cap * RADIX >= 4000000000ull) return 0;
    return (uint32_t)cap;
  }
}

int kind_of(int32_t storage_id)
{
  if (is_float_id(storage_id)) return (int)key_kind::FLOAT;
  if (is_signed_id(storage_id)) return (int)key_kind::SIGNED;
  return (int)key_kind::UNSIGNED;  // unsigned ints and BOOL8
}

template <typename UK>
column_ptr sorted_order_single(const b2_column_view& col, bool ascending, bool nulls_before, cudaStream_t stream)
{
  const int64_t n = col.size;
  const int sid   = storage_type(col.type_id);
  const int kind  = kind_of(sid);
  auto out = make_column(B2_INT32, col.size, false, stream);
  const UK* data = static_cast<const UK*>(col.data) + col.offset;
  int32_t* out_idx = out->data.as<int32_t>();

  if (!has_nulls(col)) {
    // estimated-base range tier: the temporaries are its windows (256 * cap rows), also for the exact plan it falls back to
    const uint32_t cap = est_range_capacity<UK>(data, n, kind, !ascending, true, key_tile<UK>::tile, stream);
    const int64_t rows = cap ? std::max<int64_t>(n, (int64_t)RADIX * cap) : n;
    dbuf a(sizeof(UK) * rows, stream), b(sizeof(UK) > 1 ? sizeof(UK) * rows : 0, stream), it(sizeof(int32_t) * rows, stream);
    dbuf ev(cap ? sizeof(int32_t) * RADIX * (size_t)cap : 0, stream);
    run_radix<UK>(data, a.as<UK>(), b.as<UK>(), out_idx, it.as<int32_t>(), 0, n, kind, !ascending, true, stream, nullptr, cap, ev.ptr);
    return out;
  }
  // nullable: nulls first iff (null_order == BEFORE) xor descending (sort_column_impl.cuh:35-57)
  const bool nulls_first = nulls_before != !ascending;
  const int64_t n_null  = col.null_count;
  const int64_t n_valid = n - n_null;
  const int64_t ntiles = (n + CP_ROWS - 1) / CP_ROWS;
  dbuf tv(sizeof(uint32_t) * (ntiles + 1), stream);
  B2_LAUNCH(valid_count_kernel, (unsigned)((ntiles + 7) / 8), CP_THREADS, 0, stream, col.null_mask, (int64_t)col.offset, n,
            tv.as<uint32_t>());
  B2_LAUNCH(scan_tiles_kernel, 1, 1024, 0, stream, tv.as<uint32_t>(), ntiles, tv.as<uint32_t>() + ntiles);
  dbuf a(sizeof(UK) * std::max<int64_t>(n_valid, 1), stream), b(sizeof(UK) * std::max<int64_t>(n_valid, 1), stream);
  dbuf it(sizeof(int32_t) * std::max<int64_t>(n_valid, 1), stream), it2(sizeof(int32_t) * std::max<int64_t>(n_valid, 1), stream);
  int32_t* valid_out = out_idx + (nulls_first ? n_null : 0);
  int32_t* null_out  = out_idx + (nulls_first ? 0 : n_valid);
  const UK desc_mask = ascending ? UK(0) : ~UK(0);
  // compaction writes explicit row ids into the TEMP idx buffer (buffer 1); the plan then makes the
  // last executed pass land in buffer 0 = valid_out.
  B2_LAUNCH((compact_kernel<UK>), (unsigned)ntiles, CP_THREADS, 0, stream, data, col.null_mask, (int64_t)col.offset, n,
            kind, desc_mask, tv.as<uint32_t>(), a.as<UK>(), it.as<int32_t>(), null_out);
  if (n_valid > 0)
    run_radix<UK>(nullptr, a.as<UK>(), b.as<UK>(), valid_out, it.as<int32_t>(), 1, n_valid, kind, !ascending, true, stream,
                  it2.as<int32_t>());
  return out;
}

}  // namespace

bool is_radix_sortable(const b2_column_view& c) { return !has_nulls(c) && is_fixed_width(c.type_id); }

// cudf::detail::sorted_order(column_view) — cpp/src/sort/sort_column.cu:22-44
static column_ptr sorted_order_column(const b2_column_view& col, bool ascending, bool nulls_before, cudaStream_t stream)
{
  switch (type_width(col.type_id)) {
    case 1: return sorted_order_single<uint8_t>(col, ascending, nulls_before, stream);
    case 2: return sorted_order_single<uint16_t>(col, ascending, nulls_before, stream);
    case 4: return sorted_order_single<uint32_t>(col, ascending, nulls_before, stream);
    case 8: return sorted_order_single<uint64_t>(col, ascending, nulls_before, stream);
    default: B2_FAIL(B2_ERR_DATA_TYPE, "sorted_order: unsupported (non fixed-width) key type");
  }
}

// ---- multi-column lexicographic order (sort_impl.cuh:61-93): LSD over columns, last to first ----
namespace {
template <typename UK>
__global__ void gather_twiddle_kernel(const UK* __restrict__ keys, const uint32_t* __restrict__ mask, int64_t bit_offset,
                                      const int32_t* __restrict__ perm, int64_t n, int kind, UK desc_mask,
                                      UK* __restrict__ out_keys, uint8_t* __restrict__ out_null)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    int32_t r = perm ? perm[i] : (int32_t)i;
    bool valid = mask == nullptr || bit_is_set(mask, bit_offset + r);
    out_keys[i] = valid ? twiddle_rt<UK>(keys[r], kind, desc_mask) : UK(0);
    if (out_null) out_null[i] = valid ? 0 : 1;
  }
}
// stable 2-way partition of perm by flag (0 first when zero_first) — used for the null "digit"
__global__ void flag_count_kernel(const uint8_t* __restrict__ flag, int64_t n, uint32_t* __restrict__ tile_ones)
{
  // one warp per 1024 elements
  const int64_t tile = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int64_t ntiles = (n + 1023) / 1024;
  if (tile >= ntiles) return;
  uint32_t c = 0;
  for (int j = 0; j < 32; ++j) {
    int64_t i = tile * 1024 + j * 32 + lane_id();
    c += (i < n && flag[i]) ? 1u : 0u;
  }
  c = warp_sum(c);
  if (lane_id() == 0) tile_ones[tile] = c;
}
__global__ void flag_partition_kernel(const uint8_t* __restrict__ flag, const int32_t* __restrict__ perm_in, int64_t n,
                                      const uint32_t* __restrict__ tile_ones_excl, const uint32_t* __restrict__ total_ones,
                                      int ones_first, int32_t* __restrict__ perm_out)
{
  const int64_t tile = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int64_t ntiles = (n + 1023) / 1024;
  if (tile >= ntiles) return;
  const uint32_t tot1 = *total_ones;
  const uint32_t tot0 = (uint32_t)n - tot1;
  uint32_t ones_before = tile_ones_excl[tile];
  uint32_t zeros_before = (uint32_t)(tile * 1024) - ones_before;
  for (int j = 0; j < 32; ++j) {
    int64_t i = tile * 1024 + j * 32 + lane_id();
    bool in = i < n;
    bool f = in && flag[i];
    unsigned b1 = __ballot_sync(0xffffffffu, f);
    unsigned b0 = __ballot_sync(0xffffffffu, in && !f);
    if (in) {
      uint32_t o = f ? (ones_first ? 0u : tot0) + ones_before + __popc(b1 & lanemask_lt())
                     : (ones_first ? tot1 : 0u) + zeros_before + __popc(b0 & lanemask_lt());
      perm_out[o] = perm_in[i];
    }
    ones_before += __popc(b1);
    zeros_before += __popc(b0);
  }
}
__global__ void compose_perm_kernel(const int32_t* __restrict__ perm, const int32_t* __restrict__ order, int64_t n,
                                    int32_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = perm[order[i]];
}

template <typename UK>
void lex_step(const b2_column_view& col, bool ascending, bool nulls_before, int32_t*& perm, int32_t*& perm_alt,
              bool& have_perm, dbuf& ka, dbuf& kb, dbuf& kc, dbuf& ord, dbuf& otmp, dbuf& nullflag, dbuf& tiles, cudaStream_t stream)
{
  const int64_t n = col.size;
  const int kind  = kind_of(storage_type(col.type_id));
  const UK desc_mask = ascending ? UK(0) : ~UK(0);
  const bool nullable = has_nulls(col);
  const int grid = (int)std::min<int64_t>((n + 255) / 256, num_sms() * 16);
  B2_LAUNCH((gather_twiddle_kernel<UK>), grid, 256, 0, stream, static_cast<const UK*>(col.data) + col.offset,
            nullable ? col.null_mask : nullptr, (int64_t)col.offset, have_perm ? perm : nullptr, n, kind, desc_mask,
            ka.as<UK>(), nullable ? nullflag.as<uint8_t>() : nullptr);
  // sort positions 0..n-1 by the gathered key: explicit ids = iota in buffer 1 (otmp), result in ord
  // (raw=false path wants explicit ids; generate iota cheaply through the same compose kernel is
  // not possible, so run with pre-twiddled keys + implicit ids by treating them as UNSIGNED raw.)
  run_radix<UK>(ka.as<UK>(), kb.as<UK>(), kc.as<UK>(), ord.as<int32_t>(), otmp.as<int32_t>(), 0, n,
                (int)key_kind::UNSIGNED, false, true, stream);
  // perm' = perm ∘ ord
  if (have_perm) {
    B2_LAUNCH(compose_perm_kernel, grid, 256, 0, stream, perm, ord.as<int32_t>(), n, perm_alt);
    std::swap(perm, perm_alt);
  } else {
    B2_CUDA_TRY(cudaMemcpyAsync(perm, ord.ptr, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, stream));
    have_perm = true;
  }
  if (nullable) {
    // null flag of the rows in the new order, then a stable partition (the null "digit")
    const bool nulls_first = nulls_before != !ascending;
    const int64_t ntiles = (n + 1023) / 1024;
    // flags in new order: gather nullflag (indexed by old position) through ord
    // reuse kb as byte scratch
    uint8_t* f2 = kb.as<uint8_t>();
    // f2[i] = nullflag[ord[i]]
    B2_LAUNCH((gather_twiddle_kernel<uint8_t>), grid, 256, 0, stream, nullflag.as<uint8_t>(), (const uint32_t*)nullptr,
              (int64_t)0, ord.as<int32_t>(), n, (int)key_kind::UNSIGNED, (uint8_t)0, f2, (uint8_t*)nullptr);
    B2_LAUNCH(flag_count_kernel, (unsigned)((ntiles + 7) / 8), 256, 0, stream, f2, n, tiles.as<uint32_t>());
    B2_LAUNCH(scan_tiles_kernel, 1, 1024, 0, stream, tiles.as<uint32_t>(), ntiles, tiles.as<uint32_t>() + ntiles);
    B2_LAUNCH(flag_partition_kernel, (unsigned)((ntiles + 7) / 8), 256, 0, stream, f2, perm, n, tiles.as<uint32_t>(),
              tiles.as<uint32_t>() + ntiles, nulls_first ? 1 : 0, perm_alt);
    std::swap(perm, perm_alt);
  }
}
}  // namespace

// cudf::detail::sorted_order(table_view) — cpp/src/sort/sort_impl.cuh:31-96
column_ptr sorted_order(const std::vector<b2_column_view>& keys, const std::vector<uint8_t>& order,
                        const std::vector<uint8_t>& null_prec, bool /*stable: every path here is stable*/,
                        cudaStream_t stream)
{
  if (keys.empty() || keys[0].size == 0) return make_column(B2_INT32, 0, false, stream);
  B2_EXPECTS(order.empty() || order.size() == keys.size(), B2_ERR_LOGIC,
             "Mismatch between number of columns and column order.");
  B2_EXPECTS(null_prec.empty() || null_prec.size() == keys.size(), B2_ERR_LOGIC,
             "Mismatch between number of columns and null_precedence size.");
  auto asc = [&](size_t i) { return order.empty() ? true : order[i] == B2_ASCENDING; };
  auto before = [&](size_t i) { return null_prec.empty() ? true : null_prec[i] == B2_NULL_BEFORE; };
  if (keys.size() == 1) return sorted_order_column(keys[0], asc(0), before(0), stream);

  const int64_t n = keys[0].size;
  auto out = make_column(B2_INT32, (int32_t)n, false, stream);
  dbuf alt(sizeof(int32_t) * n, stream), ka(8 * n, stream), kb(8 * n, stream), kc(8 * n, stream), ord(sizeof(int32_t) * n, stream),
    otmp(sizeof(int32_t) * n, stream), nullflag(n, stream), tiles(sizeof(uint32_t) * ((n + 1023) / 1024 + 1), stream);
  int32_t* perm = out->data.as<int32_t>();
  int32_t* perm_alt = alt.as<int32_t>();
  bool have_perm = false;
  for (size_t c = keys.size(); c-- > 0;) {
    const auto& col = keys[c];
    switch (type_width(col.type_id)) {
      case 1: lex_step<uint8_t>(col, asc(c), before(c), perm, perm_alt, have_perm, ka, kb, kc, ord, otmp, nullflag, tiles, stream); break;
      case 2: lex_step<uint16_t>(col, asc(c), before(c), perm, perm_alt, have_perm, ka, kb, kc, ord, otmp, nullflag, tiles, stream); break;
      case 4: lex_step<uint32_t>(col, asc(c), before(c), perm, perm_alt, have_perm, ka, kb, kc, ord, otmp, nullflag, tiles, stream); break;
      case 8: lex_step<uint64_t>(col, asc(c), before(c), perm, perm_alt, have_perm, ka, kb, kc, ord, otmp, nullflag, tiles, stream); break;
      default: B2_FAIL(B2_ERR_DATA_TYPE, "sorted_order: unsupported (non fixed-width) key type");
    }
  }
  if (perm != out->data.as<int32_t>()) {
    B2_CUDA_TRY(cudaMemcpyAsync(out->data.ptr, perm, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, stream));
    // `alt` now aliases the live result until the copy has run; it is freed stream-ordered after it.
  }
  return out;
}

// sort_by_key of ONE non-null 4- or 8-byte values column by ONE non-null fixed-width key column carries the payload
// through the passes instead of row ids: no random-access gather afterwards (a random 8-byte read
// fetches a whole DRAM burst, many times the bytes it uses). B2_SORT_CARRY=0 selects the row-id + gather path for every shape.
bool sort_carry_enabled()
{
  static bool v = [] {
    const char* e = std::getenv("B2_SORT_CARRY");
    return !e || std::atoi(e) != 0;
  }();
  return v;
}
bool sort_carry_applicable(const b2_column_view& keys, const b2_column_view& values, bool ascending)
{
  const int vw = type_width(values.type_id);
  const bool float_desc = is_float_id(storage_type(keys.type_id)) && !ascending;  // NaN-prefix reversal works on row ids only
  return sort_carry_enabled() && is_radix_sortable(keys) && !has_nulls(values) && (vw == 4 || vw == 8) && !float_desc &&
         keys.size == values.size && keys.size > 0;
}
column_ptr sort_by_key_carry(const b2_column_view& keys, const b2_column_view& values, bool ascending, cudaStream_t stream)
{
  const int64_t n = keys.size;
  const int kind = kind_of(storage_type(keys.type_id));
  auto out = make_column(values.type_id, (int32_t)n, false, stream);
  const int vw = type_width(values.type_id);
  const void* vin = static_cast<const char*>(values.data) + (size_t)values.offset * vw;
  auto go = [&](auto ktag, auto vtag) {
    using UK = decltype(ktag);
    using VT = decltype(vtag);
    // 8-byte payloads on 8-byte keys: 512 x 20 tiles, one CTA per SM, keys by one bulk async copy per tile: 13.2 instead of
    // 16.0 ms per 1e9-row pass on the H100 (DESIGN.md §4.1)
    using Shape = std::conditional_t<sizeof(UK) == 8 && sizeof(VT) == 8, tile_512x20_bulk, key_tile<UK>>;
    const UK* kin = static_cast<const UK*>(keys.data) + keys.offset;
    // estimated-base range tier: the temporaries are its windows (256 * cap rows), also for the exact plan it falls back to
    const uint32_t cap = est_range_capacity<UK>(kin, n, kind, !ascending, true, Shape::tile, stream);
    const int64_t rows = cap ? std::max<int64_t>(n, (int64_t)RADIX * cap) : n;
    dbuf vtmp((size_t)vw * rows, stream), a(sizeof(UK) * rows, stream), b(sizeof(UK) > 1 ? sizeof(UK) * rows : 0, stream);
    dbuf ev(cap ? (size_t)vw * RADIX * cap : 0, stream);
    run_radix_cfg<UK, Shape, VT, true>(kin, a.as<UK>(), b.as<UK>(), out->data.as<int32_t>(), vtmp.as<int32_t>(), nullptr, 0, n, kind, !ascending,
                                       true, stream, 0, 7, false, vin, nullptr, cap, ev.ptr);
  };
  auto by_key = [&](auto vtag) {
    switch (type_width(keys.type_id)) {
      case 1: go(uint8_t{}, vtag); break;
      case 2: go(uint16_t{}, vtag); break;
      case 4: go(uint32_t{}, vtag); break;
      default: go(uint64_t{}, vtag); break;
    }
  };
  if (vw == 8) by_key(uint64_t{}); else by_key(uint32_t{});
  return out;
}

// cudf::detail::sort_radix — cpp/src/sort/sort_radix.cu:151-161 (integer / chrono / bool keys;
// float columns go through sorted_order + gather so that NaN payloads and -0/+0 survive)
column_ptr sort_single_column(const b2_column_view& col, bool ascending, cudaStream_t stream)
{
  const int64_t n = col.size;
  auto out = make_column(col.type_id, col.size, false, stream);
  if (n == 0) return out;
  const int kind = kind_of(storage_type(col.type_id));
  B2_EXPECTS(kind != (int)key_kind::FLOAT, B2_ERR_LOGIC, "keys-only radix path is for integer-like keys");
  auto run = [&](auto tag) {
    using UK = decltype(tag);
    const UK* kin = static_cast<const UK*>(col.data) + col.offset;
    // estimated-base range tier: the temporary and a second key buffer are its windows (256 * cap rows)
    const uint32_t cap = est_range_capacity<UK>(kin, n, kind, !ascending, false, key_tile<UK>::tile, stream);
    const int64_t rows = cap ? std::max<int64_t>(n, (int64_t)RADIX * cap) : n;
    dbuf tmp(sizeof(UK) > 1 ? sizeof(UK) * rows : 0, stream), ev(cap ? sizeof(UK) * RADIX * (size_t)cap : 0, stream);
    run_radix<UK>(kin, out->data.as<UK>(), tmp.as<UK>(), nullptr, nullptr, 0, n, kind, !ascending, false, stream, nullptr, cap, ev.ptr);
  };
  switch (type_width(col.type_id)) {
    case 1: run(uint8_t{}); break;
    case 2: run(uint16_t{}); break;
    case 4: run(uint32_t{}); break;
    case 8: run(uint64_t{}); break;
    default: B2_FAIL(B2_ERR_DATA_TYPE, "sort: unsupported key type");
  }
  return out;
}

}  // namespace b2

#ifdef B2_ONESWEEP_PROBE
// scripts/onesweep_probe.py: clears / copies out the phase stamps of the last onesweep_kernel launches (row-major
// [2][ONESWEEP_PROBE_STAMPS + 1][ONESWEEP_PROBE_TILES] int64).
extern "C" B2_API int b2_onesweep_probe_reset(void)
{
  return (int)cudaMemset(b2::g_onesweep_probe_ptr(), 0, sizeof(b2::g_onesweep_probe));
}
extern "C" B2_API int b2_onesweep_probe_read(long long* out, int* stamps, int* tiles)
{
  *stamps = b2::ONESWEEP_PROBE_STAMPS;
  *tiles  = b2::ONESWEEP_PROBE_TILES;
  return (int)cudaMemcpy(out, b2::g_onesweep_probe_ptr(), sizeof(b2::g_onesweep_probe), cudaMemcpyDeviceToHost);
}
#endif

#ifdef B2_RANGE_PROBE
// scripts/range_probe.py: clears / copies out the phase stamps of the last range_sort_kernel launches (row-major
// [RANGE_PROBE_STAMPS + 2][RANGE_PROBE_CTAS] int64).
extern "C" B2_API int b2_range_probe_reset(void)
{
  return (int)cudaMemset(b2::g_range_probe_ptr(), 0, sizeof(long long) * (b2::RANGE_PROBE_STAMPS + 2) * b2::RANGE_PROBE_CTAS);
}
extern "C" B2_API int b2_range_probe_read(long long* out, int* stamps, int* ctas)
{
  *stamps = b2::RANGE_PROBE_STAMPS;
  *ctas   = b2::RANGE_PROBE_CTAS;
  return (int)cudaMemcpy(out, b2::g_range_probe_ptr(), sizeof(long long) * (b2::RANGE_PROBE_STAMPS + 2) * b2::RANGE_PROBE_CTAS,
                         cudaMemcpyDeviceToHost);
}
#endif

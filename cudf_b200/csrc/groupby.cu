// groupby.cu — hash groupby-aggregate (SUM / MIN / MAX / COUNT / MEAN) and the sort-based grouped scan.
//
// Replaces cpp/src/groupby/groupby.cu:40-71,186-259 (dispatch, validation, empty results),
// cpp/src/groupby/hash/{groupby.cu,compute_groupby.cu,compute_single_pass_aggs.cuh,
// compute_global_memory_aggs.cuh,single_pass_functors.cuh,output_utils.cu,
// hash_compound_agg_finalizer.cu,extract_single_pass_aggs.cpp} and the cuco::static_set they use;
// element semantics from cpp/include/cudf/detail/aggregation/device_aggregators.cuh:99-112,337-446
// and result types from cpp/include/cudf/detail/aggregation/aggregation.hpp:879-970.
// Grouped scan: cpp/src/groupby/sort/{scan.cpp,group_scan_util.cuh:77-128,sort_helper.cu}.
//
// One fused kernel per aggregate() call: every row packs its key (key_pack.cuh), finds or claims its
// group slot with ONE 128-bit CAS on {key, representative row, nullbits} (linear probing), then
// updates that slot's accumulators with L2 atomics: a per-slot row counter shared by all requests
// plus one 8-byte accumulator per value aggregation (int64 / uint64 / double / order-preserving
// int64 for float MIN/MAX) and a valid counter per nullable value column.  The table starts at a
// size that keeps slots + accumulators L2-resident (2^21 slots) and grows x8 after a device-side
// overflow signal (one host sync per aggregate(), the reference also syncs once:
// compute_single_pass_aggs.cuh:111-122).  The reference instead sizes its set for N rows and
// aggregates into a sparse N-row table.  A finalize kernel converts accumulators to the reference
// result types, builds null masks (group with zero valid values -> null) and MEAN = SUM / COUNT.
#include "common.cuh"
#include "device_utils.cuh"
#include "key_pack.cuh"

#include <algorithm>
#include <cstdlib>

namespace b2 {
namespace {

constexpr int MAX_OPS = 24;

enum acc_kind : int8_t { ACC_I64 = 0, ACC_U64 = 1, ACC_F64 = 2 };
enum op_kind : int8_t { OPK_SUM = 0, OPK_MIN = 1, OPK_MAX = 2, OPK_SUMSQ = 3, OPK_PROD = 4, OPK_ARGMIN = 5, OPK_ARGMAX = 6 };

struct value_op {
  const void* src;
  const uint32_t* mask;  // null when the column has no nulls
  int32_t offset;
  int8_t src_type;       // storage type id (B2_INT8 ... B2_BOOL8)
  int8_t acc;            // acc_kind
  int8_t op;             // op_kind
  int8_t pad;
  unsigned long long* accum;  // [slots]
  int32_t* vcount;            // [slots] valid-value counter of the source column (shared by its ops) or null
  int32_t bump_vcount;        // only the first op of a column bumps the shared counter
};

struct value_ops {
  value_op op[MAX_OPS];
  int32_t n;
};

struct gb_ctl {
  unsigned int ngroups;
  unsigned int overflow;
};

// order-preserving double <-> int64 (for MIN/MAX of floats with integer atomics). Every NaN maps to the positive quiet NaN,
// which orders above +inf: MIN / MAX rank NaN above +inf whatever its sign, as scan_reduce.cu's binop does.
__device__ __forceinline__ long long f64_to_ordered(double v)
{
  if (v != v) return 0x7ff8000000000000ll;
  long long b = __double_as_longlong(v);
  return b >= 0 ? b : (b ^ 0x7fffffffffffffffll);
}
__device__ __forceinline__ double ordered_to_f64(long long o)
{
  return __longlong_as_double(o >= 0 ? o : (o ^ 0x7fffffffffffffffll));
}

__device__ __forceinline__ void load_value(const value_op& op, int64_t e, long long& iv, unsigned long long& uv, double& fv)
{
  // values are streamed once: evict-first loads keep the group table and accumulators L2-resident
  switch (op.src_type) {
    case B2_INT8: iv = __ldcs(static_cast<const signed char*>(op.src) + e); break;
    case B2_INT16: iv = __ldcs(static_cast<const short*>(op.src) + e); break;
    case B2_INT32: iv = __ldcs(static_cast<const int*>(op.src) + e); break;
    case B2_INT64: iv = __ldcs(static_cast<const long long*>(op.src) + e); break;
    case B2_UINT8: uv = __ldcs(static_cast<const unsigned char*>(op.src) + e); iv = (long long)uv; break;
    case B2_UINT16: uv = __ldcs(static_cast<const unsigned short*>(op.src) + e); iv = (long long)uv; break;
    case B2_UINT32: uv = __ldcs(static_cast<const unsigned int*>(op.src) + e); iv = (long long)uv; break;
    case B2_UINT64: uv = __ldcs(static_cast<const unsigned long long*>(op.src) + e); iv = (long long)uv; break;
    case B2_BOOL8: uv = __ldcs(static_cast<const unsigned char*>(op.src) + e) != 0; iv = (long long)uv; break;
    case B2_FLOAT32: fv = __ldcs(static_cast<const float*>(op.src) + e); break;
    default: fv = __ldcs(static_cast<const double*>(op.src) + e); break;
  }
}

// WIDE (keys wider than 8 bytes): the slot holds a 64-bit hash of the row; a hash hit is confirmed by comparing the
// key columns of this row with the slot's representative row (key_pack.cuh).
// SQ: the request contains SUM_OF_SQUARES accumulators (M2 / VARIANCE / STD are derived from SUM, SUM_OF_SQUARES and
// COUNT in the finalize step: cpp/src/groupby/common/m2_var_std.cu:35-62) or PRODUCT accumulators (a CAS loop per
// update: device_aggregators.cuh:323-335 atomic_mul).
template <bool WIDE = false, bool SQ = false>
__global__ void __launch_bounds__(256) groupby_kernel(key_cols kc, int64_t n, bool skip_null_keys, slot_t* __restrict__ table,
                                                      uint32_t mask, uint32_t cap, int32_t* __restrict__ gsize,
                                                      int32_t* __restrict__ slot_gid, int32_t* __restrict__ rep_rows, value_ops ops,
                                                      gb_ctl* ctl)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  slot_t empty;
  memset(&empty, 0xff, sizeof(empty));
  int iter = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride, ++iter) {
    // table too small -> the host grows it and reruns. Polled rarely: a per-row volatile read of one
    // word turned a single L2 slice into the bottleneck.
    if ((iter & 63) == 0 && *reinterpret_cast<volatile unsigned int*>(&ctl->overflow)) return;
    uint64_t key;
    uint32_t nb;
    if constexpr (WIDE) hash_row_wide(kc, r, key, nb);
    else pack_row(kc, r, key, nb);
    if (skip_null_keys && nb) continue;
    uint32_t i = slot_hash(key, nb, mask);
    int probes = 0;
    while (true) {
      // a full table (overflow in progress) must not trap the probe loop
      if (((++probes) & 127) == 0 && *reinterpret_cast<volatile unsigned int*>(&ctl->overflow)) return;
      // cheap read first: most rows find their group already present
      slot_t cur = load_slot_volatile(&table[i]);
      if (cur.row == -1) {
        const slot_t want{key, (int32_t)r, nb};
        cur = cas128(&table[i], empty, want);
        if (cur.row == -1) {  // we created the group
          const unsigned int g = atomicAdd(&ctl->ngroups, 1u);
          if (g >= cap) { atomicExch(&ctl->overflow, 1u); return; }
          slot_gid[i] = (int32_t)g;
          rep_rows[g] = (int32_t)r;
          break;
        }
      }
      if constexpr (WIDE) {
        if (cur.key == key && cur.nullbits == nb && rows_equal_wide(kc, r, kc, cur.row)) break;
      } else {
        if (cur.key == key && cur.nullbits == nb) break;
      }
      i = (i + 1) & mask;
    }
    atomicAdd(&gsize[i], 1);
    for (int k = 0; k < ops.n; ++k) {
      const value_op& op = ops.op[k];
      const int64_t e = r + op.offset;
      if (op.mask != nullptr) {
        if (!bit_is_set(op.mask, e)) continue;
        if (op.bump_vcount) atomicAdd(&op.vcount[i], 1);
      }
      long long iv = 0;
      unsigned long long uv = 0;
      double fv = 0;
      load_value(op, e, iv, uv, fv);
      unsigned long long* a = op.accum + i;
      if constexpr (SQ) {
        if (op.op == OPK_SUMSQ) {  // device_aggregators.cuh:309-321: value * value in the target type
          if (op.acc == ACC_F64) atomicAdd(reinterpret_cast<double*>(a), fv * fv);
          else if (op.acc == ACC_I64) atomicAdd(a, (unsigned long long)iv * (unsigned long long)iv);
          else atomicAdd(a, uv * uv);
          continue;
        }
        if (op.op == OPK_ARGMIN || op.op == OPK_ARGMAX) {
          // global_memory_aggregator.cuh:155-200: the accumulator holds a row index (sentinel -1); a row replaces the
          // holder when its value is strictly better — or equal with a smaller row index, which makes ties
          // deterministic (the reference keeps whichever tied row arrived first)
          const bool want_max = op.op == OPK_ARGMAX;
          unsigned long long seen = *reinterpret_cast<volatile unsigned long long*>(a);
          while (true) {
            bool better = seen == ~0ull;
            if (!better) {
              const int64_t held = (int64_t)seen;
              long long hi_ = 0;
              unsigned long long hu = 0;
              double hf = 0;
              load_value(op, held + op.offset, hi_, hu, hf);
              if (op.acc == ACC_F64) {
                // the order of MIN / MAX: NaN ranks above +inf, and NaNs tie
                const bool fn = fv != fv, hn = hf != hf;
                const bool beats = want_max ? (!hn && (fn || fv > hf)) : (!fn && (hn || fv < hf));
                better = beats || ((fn ? hn : fv == hf) && r < held);
              }
              else if (op.acc == ACC_I64) better = (want_max ? iv > hi_ : iv < hi_) || (iv == hi_ && r < held);
              else better = (want_max ? uv > hu : uv < hu) || (uv == hu && r < held);
            }
            if (!better) break;
            const unsigned long long prev = atomicCAS(a, seen, (unsigned long long)r);
            if (prev == seen) break;
            seen = prev;
          }
          continue;
        }
        if (op.op == OPK_PROD) {
          unsigned long long seen = *reinterpret_cast<volatile unsigned long long*>(a), want;
          do {
            const unsigned long long cur = seen;
            if (op.acc == ACC_F64) want = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)cur) * fv);
            else if (op.acc == ACC_I64) want = cur * (unsigned long long)iv;
            else want = cur * uv;
            seen = atomicCAS(a, cur, want);
            if (seen == cur) break;
          } while (true);
          continue;
        }
      }
      if (op.acc == ACC_F64) {
        if (op.op == OPK_SUM) atomicAdd(reinterpret_cast<double*>(a), fv);
        else if (op.op == OPK_MIN) atomicMin(reinterpret_cast<long long*>(a), f64_to_ordered(fv));
        else atomicMax(reinterpret_cast<long long*>(a), f64_to_ordered(fv));
      } else if (op.acc == ACC_I64) {
        if (op.op == OPK_SUM) atomicAdd(a, (unsigned long long)iv);
        else if (op.op == OPK_MIN) atomicMin(reinterpret_cast<long long*>(a), iv);
        else atomicMax(reinterpret_cast<long long*>(a), iv);
      } else {
        if (op.op == OPK_SUM) atomicAdd(a, uv);
        else if (op.op == OPK_MIN) atomicMin(a, uv);
        else atomicMax(a, uv);
      }
    }
  }
}

// ---- partitioned path (large inputs, one 8-byte integer key column, one value column) ---------------------------------
// The L2-atomic kernel above is bound by the rate of global atomics at many groups. Here the rows are first
// partitioned by the top byte of mix64(key) (one one-sweep pass carrying the value: radix_sort.cu), so that all rows of a
// group sit in one of 256 contiguous partitions; a CTA then aggregates a chunk of ONE partition in a shared-memory table
// (mixed key, row count, up to three accumulators) and merges each of its groups into the global table once — the
// role of the reference's shared-memory pre-aggregation (cpp/src/groupby/hash/compute_shared_memory_aggs.cu:261-355),
// which on its own gives up at this many groups (compute_mapping_indices.cuh:92-152 cardinality limit).
// Groups that do not fit in the shared table (more than ~4.9 K groups in a partition) go to the global table row by row.
constexpr int PGB_THREADS = 1024;
constexpr int PGB_MAX_OPS = 3;
// rows per work item of the aggregation kernel: about 12 items per SM (tail balance), between 2^15 and 2^19 rows (every item merges its
// groups into the global table once, so larger items merge less)
inline uint32_t pgb_chunk_rows(int64_t n)
{
  uint32_t c = 1u << 15;
  while (c < (1u << 19) && (int64_t)c * 2 * (num_sms() * 12) <= n) c <<= 1;
  return c;
}
constexpr bool PGB_EST_DEFAULT = true;   // histogram-free partition pass (radix_partition_mix_carry_est): one read of the keys less
constexpr uint64_t PGB_EMPTY = ~0ull;

struct pgb_args {
  const uint64_t* mkeys;     // mix64(key), partitioned
  const void* vals;          // carried value bits (val_bytes each) or null
  int32_t val_bytes;
  int32_t src_type;          // storage type id of the value column
  const uint32_t* part_base; // [256] first row of each partition
  const uint32_t* part_end;  // [256] one past its last row (partitions need not be adjacent: estimated bases leave gaps)
  uint32_t n;
  const uint32_t* item_start;  // [257] first work item of each partition (exclusive scan of chunk counts)
  uint32_t* item_counter;
  uint32_t chunk;            // rows per work item
  uint32_t smem_slots;       // power of two
  uint32_t smem_limit;       // groups accepted in the shared table
  int32_t nops;
  int8_t op[PGB_MAX_OPS];    // op_kind
  int8_t acc[PGB_MAX_OPS];   // acc_kind
  unsigned long long* accum[PGB_MAX_OPS];  // global accumulators [slots]
  unsigned long long init[PGB_MAX_OPS];
};

// find or claim the global slot of `key` (same protocol as groupby_kernel); -1: table overflow signalled
__device__ __forceinline__ int64_t global_slot(slot_t* __restrict__ table, uint32_t mask, uint32_t cap, uint64_t key, int32_t* __restrict__ slot_gid,
                                               gb_ctl* ctl)
{
  slot_t empty;
  memset(&empty, 0xff, sizeof(empty));
  uint32_t i = slot_hash(key, 0u, mask);
  int probes = 0;
  while (true) {
    if (((++probes) & 127) == 0 && *reinterpret_cast<volatile unsigned int*>(&ctl->overflow)) return -1;
    slot_t cur = load_slot_volatile(&table[i]);
    if (cur.row == -1) {
      const slot_t want{key, 0, 0u};
      cur = cas128(&table[i], empty, want);
      if (cur.row == -1) {
        const unsigned int g = atomicAdd(&ctl->ngroups, 1u);
        if (g >= cap) { atomicExch(&ctl->overflow, 1u); return -1; }
        slot_gid[i] = (int32_t)g;
        return i;
      }
    }
    if (cur.key == key && cur.nullbits == 0u) return i;
    i = (i + 1) & mask;
  }
}

__device__ __forceinline__ unsigned long long pgb_value_bits(const pgb_args& a, uint32_t r)
{
  // accumulator-typed bits of the row's value: int64 / uint64 sums wrap identically, so integers share one form
  if (a.val_bytes == 8) {
    const unsigned long long b = __ldcs(static_cast<const unsigned long long*>(a.vals) + r);
    return b;  // INT64 / UINT64 / FLOAT64 bits
  }
  const unsigned int b = __ldcs(static_cast<const unsigned int*>(a.vals) + r);
  if (a.src_type == B2_FLOAT32) {
    float f;
    memcpy(&f, &b, 4);
    return (unsigned long long)__double_as_longlong((double)f);
  }
  if (a.src_type == B2_INT32) return (unsigned long long)(long long)(int)b;
  return (unsigned long long)b;
}

template <bool SHARED>
__device__ __forceinline__ void pgb_combine(unsigned long long* a, int8_t op, int8_t acc, unsigned long long v)
{
  // v: partial result in accumulator form (SUM: plain bits; MIN / MAX of floats: order-preserving int64)
  if (op == OPK_SUM) {
    if (acc == ACC_F64) atomicAdd(reinterpret_cast<double*>(a), __longlong_as_double((long long)v));
    else atomicAdd(a, v);
  } else if (acc == ACC_U64) {
    if (op == OPK_MIN) atomicMin(a, v); else atomicMax(a, v);
  } else {
    if (op == OPK_MIN) atomicMin(reinterpret_cast<long long*>(a), (long long)v);
    else atomicMax(reinterpret_cast<long long*>(a), (long long)v);
  }
}

__global__ void pgb_items_kernel(const uint32_t* __restrict__ part_base, uint32_t* __restrict__ part_end, bool ends_given, uint32_t n, uint32_t chunk,
                                 uint32_t* __restrict__ item_start)
{
  // 256 threads: chunks per partition, exclusive scan; adjacent partitions (exact bases): part_end is derived here
  __shared__ uint32_t wt[8];
  const int d = threadIdx.x;
  const uint32_t b = part_base[d], e = ends_given ? part_end[d] : (d == 255 ? n : part_base[d + 1]);
  if (!ends_given) part_end[d] = e;
  const uint32_t c = (e - b + chunk - 1) / chunk;
  const uint32_t inc = warp_inclusive_sum(c);
  if ((d & 31) == 31) wt[d >> 5] = inc;
  __syncthreads();
  uint32_t off = 0;
  for (int w = 0; w < (d >> 5); ++w) off += wt[w];
  item_start[d] = off + inc - c;
  if (d == 255) item_start[256] = off + inc;
}

// MODE: 0 generic (any supported ops, decided at run time), 1 = one SUM of an 8-byte float column, 2 = one SUM of an 8-byte
// integer column, 3 = no value ops (counts only). The specialised forms drop the per-row dispatch: the generic kernel spends
// ~150 instructions per row and is issue-bound.
template <int MODE>
__device__ __forceinline__ void pgb_apply(const pgb_args& a, unsigned long long* acc, size_t stride, uint32_t slot, unsigned long long vb, unsigned long long vo,
                                          bool shared_mem)
{
  if constexpr (MODE == 1) {
    atomicAdd(reinterpret_cast<double*>(acc + slot), __longlong_as_double((long long)vb));
  } else if constexpr (MODE == 2) {
    atomicAdd(acc + slot, vb);
  } else if constexpr (MODE == 0) {
    for (int k = 0; k < a.nops; ++k) {
      if (shared_mem) pgb_combine<true>(acc + (size_t)k * stride + slot, a.op[k], a.acc[k], a.op[k] == OPK_SUM ? vb : vo);
      else pgb_combine<false>(a.accum[k] + slot, a.op[k], a.acc[k], a.op[k] == OPK_SUM ? vb : vo);
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(PGB_THREADS, 1) pgb_agg_kernel(pgb_args a, slot_t* __restrict__ table, uint32_t mask, uint32_t cap,
                                                                 int32_t* __restrict__ gsize, int32_t* __restrict__ slot_gid, gb_ctl* ctl)
{
  B2_DYNAMIC_SMEM(smem_raw);
  const uint32_t S = a.smem_slots;
  unsigned long long* s_key = reinterpret_cast<unsigned long long*>(smem_raw);
  unsigned long long* s_acc = s_key + S;                                       // [nops][S]
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(s_acc + (size_t)a.nops * S);   // [S]
  __shared__ uint32_t s_item, s_fill;
  __shared__ uint32_t s_start[257];
  for (int i = threadIdx.x; i < 257; i += PGB_THREADS) s_start[i] = a.item_start[i];
  __syncthreads();
  const uint32_t total = s_start[256];
  while (true) {
    if (threadIdx.x == 0) {
      s_item = *reinterpret_cast<volatile unsigned int*>(&ctl->overflow) ? 0xffffffffu : atomicAdd(a.item_counter, 1u);
      s_fill = 0;
    }
    for (uint32_t i = threadIdx.x; i < S; i += PGB_THREADS) {
      s_key[i] = PGB_EMPTY;
      s_cnt[i] = 0;
      for (int k = 0; k < a.nops; ++k) s_acc[(size_t)k * S + i] = a.init[k];
    }
    __syncthreads();
    const uint32_t item = s_item;
    if (item >= total) return;  // also: global table overflow seen by thread 0 (the host grows the table and reruns)
    // partition of this item: last d with s_start[d] <= item
    int lo = 0, hi = 255;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_start[mid] <= item) lo = mid; else hi = mid - 1;
    }
    const uint32_t pb = a.part_base[lo], pe = a.part_end[lo];
    const uint32_t r0 = pb + (item - s_start[lo]) * a.chunk;
    const uint32_t r1 = min(pe, r0 + a.chunk);
    constexpr int U = 4;  // rows in flight per thread
    for (uint32_t rb = r0 + threadIdx.x; rb < r1; rb += U * PGB_THREADS) {
      unsigned long long mks[U], vbs[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t r = rb + u * PGB_THREADS;
        mks[u] = r < r1 ? __ldcs(a.mkeys + r) : 0ull;
        if constexpr (MODE == 1 || MODE == 2) vbs[u] = r < r1 ? __ldcs(static_cast<const unsigned long long*>(a.vals) + r) : 0ull;
        else if constexpr (MODE == 3) vbs[u] = 0ull;
        else vbs[u] = (r < r1 && a.nops) ? pgb_value_bits(a, r) : 0ull;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
      if (rb + u * PGB_THREADS >= r1) continue;  // (not `break`: keeps the loop fully unrolled and mks / vbs in registers)
      const unsigned long long mk = mks[u];
      const unsigned long long vb = vbs[u];
      // accumulator form of the value for MIN / MAX of floats (generic kernel only)
      unsigned long long vo = vb;
      if constexpr (MODE == 0) vo = (a.nops && a.acc[0] == ACC_F64) ? (unsigned long long)f64_to_ordered(__longlong_as_double((long long)vb)) : vb;
      int64_t slot = -1;
      if (mk != PGB_EMPTY) {
        uint32_t i = (uint32_t)mk & (S - 1);
        for (int probes = 0; probes < 64; ++probes) {
          unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(&s_key[i]);
          if (k == PGB_EMPTY) {
            if (*reinterpret_cast<volatile uint32_t*>(&s_fill) >= a.smem_limit) break;
            k = atomicCAS(&s_key[i], PGB_EMPTY, mk);
            if (k == PGB_EMPTY) { atomicAdd(&s_fill, 1u); k = mk; }
          }
          if (k == mk) { slot = i; break; }
          i = (i + 1) & (S - 1);
        }
      }
      if (slot >= 0) {
        atomicAdd(&s_cnt[slot], 1u);
        pgb_apply<MODE>(a, s_acc, S, (uint32_t)slot, vb, vo, true);
      } else {
        // shared table full (or the reserved key value): this row goes to the global table directly
        const int64_t g = global_slot(table, mask, cap, unmix64(mk), slot_gid, ctl);
        if (g >= 0) {
          atomicAdd(&gsize[g], 1);
          pgb_apply<MODE>(a, MODE == 0 ? nullptr : a.accum[0], 0, (uint32_t)g, vb, vo, false);
        }
      }
      }
    }
    __syncthreads();
    // merge this item's groups into the global table
    for (uint32_t i = threadIdx.x; i < S; i += PGB_THREADS) {
      const unsigned long long mk = s_key[i];
      if (mk == PGB_EMPTY) continue;
      const int64_t g = global_slot(table, mask, cap, unmix64(mk), slot_gid, ctl);
      if (g < 0) continue;
      atomicAdd(&gsize[g], (int32_t)s_cnt[i]);
      if constexpr (MODE == 0) {
        for (int k = 0; k < a.nops; ++k) pgb_combine<false>(a.accum[k] + g, a.op[k], a.acc[k], s_acc[(size_t)k * S + i]);
      } else {
        pgb_apply<MODE>(a, a.accum[0], 0, (uint32_t)g, s_acc[i], 0ull, false);
      }
    }
    __syncthreads();
  }
}

// keys of the partitioned path: group g's key is the packed key stored in its slot (one 8-byte integer column)
__global__ void pgb_keys_kernel(const slot_t* __restrict__ table, int64_t slots, const int32_t* __restrict__ slot_gid, uint64_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride)
    if (table[s].row != -1) out[slot_gid[s]] = table[s].key;
}

__global__ void fill_u64_kernel(unsigned long long* p, int64_t n, unsigned long long v)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

// finalize one output column: walk the slots, write dense group g = slot_gid[s]
struct out_spec {
  const unsigned long long* accum;  // null for counts
  const int32_t* vcount;            // null: column without nulls
  const int32_t* gsize;
  int8_t acc;       // acc_kind of accum
  int8_t op;        // op_kind
  int8_t mode;      // 0 value (SUM/MIN/MAX/SUM_OF_SQUARES), 1 MEAN, 2 COUNT_VALID, 3 COUNT_ALL, 5 M2, 6 VARIANCE, 7 STD
  int8_t pad;
  int32_t out_type; // storage type id of the output column
  void* out;
  uint32_t* out_mask;  // null: no mask
  unsigned long long* null_count;
  // appended last so that the layout seen by the validated kernels does not move
  const unsigned long long* accum2;  // modes 5-7: SUM_OF_SQUARES accumulator (accum = SUM accumulator)
  int32_t ddof;
};

template <bool EXT = false>
__global__ void __launch_bounds__(256) finalize_kernel(const slot_t* __restrict__ table, int64_t slots,
                                                       const int32_t* __restrict__ slot_gid, out_spec o)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long nulls = 0;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += stride) {
    if (table[s].row == -1) continue;
    const int32_t g = slot_gid[s];
    const int32_t nvalid = o.vcount ? o.vcount[s] : o.gsize[s];
    if (o.mode == 2) { static_cast<int32_t*>(o.out)[g] = nvalid; continue; }
    if (o.mode == 3) { static_cast<int32_t*>(o.out)[g] = o.gsize[s]; continue; }
    const unsigned long long raw = o.accum[s];
    if constexpr (EXT) {
      if (o.mode >= 5) {  // M2 / VARIANCE / STD (m2_var_std.cu:35-62,150-196), always FLOAT64
        const unsigned long long raw2 = o.accum2[s];
        const double sum   = o.acc == ACC_F64 ? __longlong_as_double((long long)raw) : (double)(long long)raw;
        const double sumsq = o.acc == ACC_F64 ? __longlong_as_double((long long)raw2) : (double)(long long)raw2;
        const double m2 = nvalid == 0 ? 0.0 : sumsq - sum * sum / nvalid;
        double out = m2;
        bool valid = true;
        if (o.mode != 5) {
          const int df = nvalid - o.ddof;
          valid = nvalid != 0 && df > 0;
          out = valid ? (o.mode == 6 ? m2 / df : sqrt(m2 / df)) : 0.0;
        }
        static_cast<double*>(o.out)[g] = out;
        if (o.out_mask) {
          if (valid) atomicOr(&o.out_mask[g >> 5], 1u << (g & 31));
          else ++nulls;
        }
        continue;
      }
    }
    if (o.mode == 1) {
      // SUM of any integral source is an int64 (aggregation.hpp:950-956): unsigned sources are read back as signed too
      double sum = o.acc == ACC_F64 ? __longlong_as_double((long long)raw) : (double)(long long)raw;
      static_cast<double*>(o.out)[g] = nvalid > 0 ? sum / (double)nvalid : 0.0;
    } else {
      double fv = 0;
      long long iv = (long long)raw;
      if (o.acc == ACC_F64) fv = o.op == OPK_SUM ? __longlong_as_double((long long)raw) : ordered_to_f64((long long)raw);
      switch (o.out_type) {
        case B2_INT8: static_cast<int8_t*>(o.out)[g] = (int8_t)iv; break;
        case B2_INT16: static_cast<int16_t*>(o.out)[g] = (int16_t)iv; break;
        case B2_INT32: static_cast<int32_t*>(o.out)[g] = (int32_t)iv; break;
        case B2_INT64: static_cast<int64_t*>(o.out)[g] = iv; break;
        case B2_UINT8: case B2_BOOL8: static_cast<uint8_t*>(o.out)[g] = (uint8_t)raw; break;
        case B2_UINT16: static_cast<uint16_t*>(o.out)[g] = (uint16_t)raw; break;
        case B2_UINT32: static_cast<uint32_t*>(o.out)[g] = (uint32_t)raw; break;
        case B2_UINT64: static_cast<uint64_t*>(o.out)[g] = raw; break;
        case B2_FLOAT32: static_cast<float*>(o.out)[g] = (float)fv; break;
        default: static_cast<double*>(o.out)[g] = fv; break;
      }
    }
    if (o.out_mask) {
      if (nvalid > 0) atomicOr(&o.out_mask[g >> 5], 1u << (g & 31));
      else ++nulls;
    }
  }
  if (o.null_count) {
    nulls = warp_sum(nulls);
    if (lane_id() == 0 && nulls) atomicAdd(o.null_count, nulls);
  }
}

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, num_sms() * 16)); }

// result type rules: aggregation.hpp:879-970
int32_t result_type(int32_t kind, int32_t src)
{
  switch (kind) {
    case B2_AGG_SUM: case B2_AGG_SUM_OF_SQUARES: case B2_AGG_PRODUCT: return is_float_id(src) ? src : B2_INT64;
    case B2_AGG_M2: case B2_AGG_VARIANCE: case B2_AGG_STD: return B2_FLOAT64;
    case B2_AGG_MIN: case B2_AGG_MAX: return src;
    case B2_AGG_COUNT_VALID: case B2_AGG_COUNT_ALL: case B2_AGG_ARGMAX: case B2_AGG_ARGMIN: return B2_INT32;
    case B2_AGG_MEAN: return B2_FLOAT64;
    default: B2_FAIL(B2_ERR_INVALID_ARGUMENT, "unsupported groupby aggregation on the hash path (SUM/PRODUCT/MIN/MAX/ARGMIN/ARGMAX/COUNT/MEAN/SUM_OF_SQUARES/M2/VARIANCE/STD)");
  }
}

// B2_AGG_WITH_DDOF: bit 30 says "ddof given", bits 8..23 hold it; the plain kind means ddof = 1 (aggregation.hpp:231-260)
inline int32_t base_kind(int32_t k) { return (k & (1 << 30)) ? (k & 0xFF) : k; }
inline int32_t kind_ddof(int32_t k) { return (k & (1 << 30)) ? ((k >> 8) & 0xFFFF) : 1; }
inline bool needs_sumsq(int32_t kind) { return kind == B2_AGG_SUM_OF_SQUARES || kind == B2_AGG_M2 || kind == B2_AGG_VARIANCE || kind == B2_AGG_STD; }

unsigned long long acc_init(int8_t acc, int8_t op)
{
  if (op == OPK_SUM || op == OPK_SUMSQ) return 0ull;
  if (op == OPK_PROD) return acc == ACC_F64 ? 0x3FF0000000000000ull /* 1.0 */ : 1ull;
  if (op == OPK_ARGMIN || op == OPK_ARGMAX) return ~0ull;  // ARG*_SENTINEL
  if (acc == ACC_U64) return op == OPK_MIN ? ~0ull : 0ull;
  // I64, and F64 in ordered-int64 space
  return op == OPK_MIN ? (unsigned long long)INT64_MAX : (unsigned long long)INT64_MIN;
}

}  // namespace
}  // namespace b2

using namespace b2;

struct b2_groupby {
  std::vector<b2_column_view> keys;
  int32_t null_handling = B2_NULL_EXCLUDE;
  bool keys_are_sorted  = false;
  std::vector<uint8_t> order, nprec;
};

namespace b2 {

struct request_view {
  b2_column_view values;
  std::vector<int32_t> kinds;
};

static void empty_results(const b2_groupby& gb, const std::vector<request_view>& reqs, cudaStream_t stream, table_ptr& keys_out,
                          table_ptr& res_out)
{
  keys_out = std::make_unique<b2_table>();
  for (auto& k : gb.keys) keys_out->cols.push_back(make_column(k.type_id, 0, false, stream));
  res_out = std::make_unique<b2_table>();
  for (auto& r : reqs)
    for (int32_t kind : r.kinds) res_out->cols.push_back(make_column(result_type(base_kind(kind), r.values.type_id), 0, false, stream));
}

bool groupby_needs_sort_path(const b2_groupby& gb, const std::vector<request_view>& reqs);
void groupby_aggregate_sorted(const b2_groupby& gb, const std::vector<request_view>& reqs, cudaStream_t stream, table_ptr& keys_out,
                              table_ptr& res_out);

// cudf::groupby::groupby::aggregate — groupby.cu:220-237 -> hash path
void groupby_aggregate(const b2_groupby& gb, const std::vector<request_view>& reqs, cudaStream_t stream, table_ptr& keys_out,
                       table_ptr& res_out)
{
  if (groupby_needs_sort_path(gb, reqs)) return groupby_aggregate_sorted(gb, reqs, stream, keys_out, res_out);
  const int64_t n = gb.keys.empty() ? 0 : gb.keys[0].size;
  for (auto& r : reqs) {
    validate_column(r.values);
    B2_EXPECTS(r.values.size == n, B2_ERR_LOGIC, "Size mismatch between request values and groupby keys.");
    B2_EXPECTS(!r.kinds.empty(), B2_ERR_LOGIC, "Empty aggregation request");  // verify_valid_requests
    for (int32_t raw_kind : r.kinds) {
      const int32_t kind = base_kind(raw_kind);
      (void)result_type(kind, r.values.type_id);
      if (kind == B2_AGG_SUM || kind == B2_AGG_MEAN || kind == B2_AGG_PRODUCT || needs_sumsq(kind))
        B2_EXPECTS(is_numeric(r.values.type_id), B2_ERR_LOGIC, "SUM/PRODUCT/MEAN/SUM_OF_SQUARES/M2/VARIANCE/STD need a numeric values column");
    }
  }
  if (n == 0) return empty_results(gb, reqs, stream, keys_out, res_out);

  const bool wide = keys_are_wide(gb.keys);
  key_cols kc = make_key_cols(gb.keys, true);
  bool keys_nullable = false;
  for (auto& k : gb.keys) keys_nullable |= has_nulls(k);
  const bool skip_null_keys = keys_nullable && gb.null_handling == B2_NULL_EXCLUDE;

  // ---- partitioned path? (one null-free 8-byte integer key column, all value data from ONE null-free 4- / 8-byte column,
  // SUM / MIN / MAX / MEAN / COUNT only, large input) ----
  bool use_pgb = false;
  const b2_column_view* pgb_val = nullptr;
  {
    static const int64_t min_rows = [] {
      const char* e = std::getenv("B2_GROUPBY_PARTITION_ROWS");  // 0 switches the path off
      const int64_t v = e ? std::atoll(e) : (int64_t(1) << 24);
      return v <= 0 ? INT64_MAX : v;
    }();
    bool ok = n >= min_rows && gb.keys.size() == 1 && type_width(gb.keys[0].type_id) == 8 && !is_float_id(storage_type(gb.keys[0].type_id)) &&
              !keys_nullable;
    int data_ops = 0;
    for (auto& r : reqs) {
      if (!ok) break;
      if (has_nulls(r.values)) { ok = false; break; }
      bool needs_data = false;
      bool has_sum = false;
      for (int32_t raw_kind : r.kinds) {
        const int32_t kind = base_kind(raw_kind);
        if (kind == B2_AGG_COUNT_VALID || kind == B2_AGG_COUNT_ALL) continue;
        if (kind == B2_AGG_SUM || kind == B2_AGG_MEAN) { needs_data = true; if (!has_sum) { has_sum = true; ++data_ops; } continue; }
        if (kind == B2_AGG_MIN || kind == B2_AGG_MAX) { needs_data = true; ++data_ops; continue; }
        ok = false;
      }
      if (!needs_data) continue;
      const int w = type_width(r.values.type_id);
      if (w != 4 && w != 8) ok = false;
      if (pgb_val && (pgb_val->data != r.values.data || pgb_val->offset != r.values.offset || pgb_val->type_id != r.values.type_id)) ok = false;
      if (pgb_val && ok) ok = false;  // one request carries the data column (keeps the op bookkeeping below one-to-one)
      pgb_val = &r.values;
    }
    use_pgb = ok && data_ops <= PGB_MAX_OPS;
  }
  dbuf pgb_keys, pgb_vals, pgb_base, pgb_items;
  bool pgb_ends_given = false;
  if (use_pgb) {
    prof_scope ps("groupby_partition", stream);
    const int vb = pgb_val ? type_width(pgb_val->type_id) : 0;
    pgb_base  = dbuf(sizeof(uint32_t) * 512, stream);  // [256] first row, [256] end of each partition
    pgb_items = dbuf(sizeof(uint32_t) * 258, stream);
    const uint64_t* kin = static_cast<const uint64_t*>(gb.keys[0].data) + gb.keys[0].offset;
    // Histogram-free partition pass when a sample of the keys says the partitions are even enough (B2_GROUPBY_EST=0: never):
    // partition d gets a fixed range of `cap` rows, the pass reports where each one ended.
    static const bool est_enabled = [] {
      const char* e = std::getenv("B2_GROUPBY_EST");
      return e ? std::atoi(e) != 0 : PGB_EST_DEFAULT;
    }();
    const uint32_t est_cap = est_enabled ? radix_partition_est_capacity(kin, n, stream) : 0u;
    if (est_cap) {
      const int cb = vb ? vb : 8;
      pgb_keys = dbuf(sizeof(uint64_t) * 256 * (size_t)est_cap, stream);
      pgb_vals = dbuf((size_t)cb * 256 * (size_t)est_cap, stream);
      const void* vin = vb ? static_cast<const void*>(static_cast<const char*>(pgb_val->data) + (size_t)pgb_val->offset * vb) : static_cast<const void*>(kin);
      pgb_ends_given = radix_partition_mix_carry_est(kin, vin, cb, n, est_cap, pgb_keys.as<uint64_t>(), pgb_vals.ptr, pgb_base.as<uint32_t>(),
                                                     pgb_base.as<uint32_t>() + 256, stream);
      if (!pgb_ends_given) {  // a partition overflowed its range (the sample missed a hot spot): exact bases below
        pgb_keys = dbuf();
        pgb_vals = dbuf();
      }
    }
    if (pgb_ends_given) {
      // partitioned by the estimated bases
    } else if (vb) {
      pgb_keys  = dbuf(sizeof(uint64_t) * n, stream);
      pgb_vals = dbuf((size_t)vb * n, stream);
      radix_partition_mix_carry(kin, static_cast<const char*>(pgb_val->data) + (size_t)pgb_val->offset * vb, vb, n, pgb_keys.as<uint64_t>(),
                                pgb_vals.ptr, pgb_base.as<uint32_t>(), stream);
    } else {  // counts only: the key column doubles as the carried payload
      pgb_keys = dbuf(sizeof(uint64_t) * n, stream);
      pgb_vals = dbuf(sizeof(uint64_t) * n, stream);
      radix_partition_mix_carry(kin, kin, 8, n, pgb_keys.as<uint64_t>(), pgb_vals.ptr, pgb_base.as<uint32_t>(), stream);
    }
  }

  // ---- plan the accumulators ----
  struct col_plan { int32_t* vcount = nullptr; bool bumped = false; };
  uint64_t max_slots = 16;
  while (max_slots < 2ull * (uint64_t)n) max_slots <<= 1;
  uint64_t slots = std::min<uint64_t>(max_slots, 1ull << 21);

  while (true) {
    const uint32_t cap = (uint32_t)std::min<uint64_t>((uint64_t)n, (uint64_t)(slots * 0.6));
    dbuf table(slots * sizeof(slot_t), stream);
    B2_CUDA_TRY(cudaMemsetAsync(table.ptr, 0xff, table.bytes, stream));
    dbuf gsize(sizeof(int32_t) * slots, stream), slot_gid(sizeof(int32_t) * slots, stream);
    B2_CUDA_TRY(cudaMemsetAsync(gsize.ptr, 0, gsize.bytes, stream));
    dbuf rep_rows(sizeof(int32_t) * (size_t)cap, stream);
    dbuf ctl(sizeof(gb_ctl), stream);
    B2_CUDA_TRY(cudaMemsetAsync(ctl.ptr, 0, sizeof(gb_ctl), stream));

    value_ops ops{};
    std::vector<dbuf> accs;                      // one per value op
    std::vector<dbuf> vcounts(reqs.size());      // one per nullable value column
    struct slot_of { int op_index; };            // (request, kind) -> op index or -1
    std::vector<std::vector<int>> op_of(reqs.size()), op2_of(reqs.size());  // op2: SUM_OF_SQUARES partner of M2/VAR/STD
    bool any_sumsq = false;
    for (size_t q = 0; q < reqs.size(); ++q) {
      const auto& v = reqs[q].values;
      const int32_t st = storage_type(v.type_id);
      const bool nullable = has_nulls(v);
      bool bumped = false;
      const int op_begin = ops.n;
      // MEAN / SUM / M2 / VARIANCE / STD of the same column share one SUM accumulator; SUM_OF_SQUARES / M2 / VARIANCE /
      // STD share one SUM_OF_SQUARES accumulator
      int sum_op = -1, sumsq_op = -1;
      auto new_op = [&](int8_t opk) {
        B2_EXPECTS(ops.n < MAX_OPS, B2_ERR_INVALID_ARGUMENT, "too many aggregations in one groupby call");
        value_op& op = ops.op[ops.n];
        op.src      = v.data;
        op.mask     = nullable ? v.null_mask : nullptr;
        op.offset   = v.offset;
        op.src_type = (int8_t)st;
        const bool sumlike = opk == OPK_SUM || opk == OPK_SUMSQ || opk == OPK_PROD;
        op.acc      = is_float_id(st) ? ACC_F64 : ((is_signed_id(st) || sumlike) ? ACC_I64 : ACC_U64);
        if (sumlike && !is_float_id(st) && !is_signed_id(st)) op.acc = ACC_U64;  // same bits as int64 sums
        op.op       = opk;
        accs.emplace_back(sizeof(unsigned long long) * slots, stream);
        op.accum = accs.back().as<unsigned long long>();
        B2_LAUNCH(fill_u64_kernel, grid_for((int64_t)slots), 256, 0, stream, op.accum, (int64_t)slots, acc_init(op.acc, opk));
        return ops.n++;
      };
      for (int32_t raw_kind : reqs[q].kinds) {
        const int32_t kind = base_kind(raw_kind);
        if (kind == B2_AGG_COUNT_VALID || kind == B2_AGG_COUNT_ALL) { op_of[q].push_back(-1); op2_of[q].push_back(-1); continue; }
        if (kind == B2_AGG_MIN || kind == B2_AGG_MAX) {
          op_of[q].push_back(new_op(kind == B2_AGG_MIN ? OPK_MIN : OPK_MAX));
          op2_of[q].push_back(-1);
          continue;
        }
        if (kind == B2_AGG_ARGMIN || kind == B2_AGG_ARGMAX) {
          op_of[q].push_back(new_op(kind == B2_AGG_ARGMIN ? OPK_ARGMIN : OPK_ARGMAX));
          op2_of[q].push_back(-1);
          any_sumsq = true;  // handled by the extended kernel instantiation
          continue;
        }
        if (kind == B2_AGG_PRODUCT) {
          op_of[q].push_back(new_op(OPK_PROD));
          op2_of[q].push_back(-1);
          any_sumsq = true;  // the extended kernel instantiation also carries the PRODUCT update
          continue;
        }
        const bool want_sum = kind != B2_AGG_SUM_OF_SQUARES;  // SUM, MEAN, M2, VARIANCE, STD
        if (want_sum && sum_op < 0) sum_op = new_op(OPK_SUM);
        if (needs_sumsq(kind) && sumsq_op < 0) { sumsq_op = new_op(OPK_SUMSQ); any_sumsq = true; }
        op_of[q].push_back(kind == B2_AGG_SUM_OF_SQUARES ? sumsq_op : sum_op);
        op2_of[q].push_back(kind == B2_AGG_SUM_OF_SQUARES ? -1 : (needs_sumsq(kind) ? sumsq_op : -1));
      }
      if (nullable) {
        vcounts[q] = dbuf(sizeof(int32_t) * slots, stream);
        B2_CUDA_TRY(cudaMemsetAsync(vcounts[q].ptr, 0, vcounts[q].bytes, stream));
        // the shared valid counter is bumped by the column's first value op, or by a dedicated
        // pseudo-op when the request only has counts
        bool any_op = false;
        for (int k = op_begin; k < ops.n; ++k) {
          ops.op[k].vcount = vcounts[q].as<int32_t>();
          if (!bumped) { ops.op[k].bump_vcount = 1; bumped = true; }
          any_op = true;
        }
        if (!any_op) {
          B2_EXPECTS(ops.n < MAX_OPS, B2_ERR_INVALID_ARGUMENT, "too many aggregations in one groupby call");
          value_op& op = ops.op[ops.n++];
          op.src = v.data; op.mask = v.null_mask; op.offset = v.offset; op.src_type = (int8_t)st;
          op.acc = ACC_U64; op.op = OPK_MAX;  // harmless accumulate into a scratch array
          accs.emplace_back(sizeof(unsigned long long) * slots, stream);
          op.accum = accs.back().as<unsigned long long>();
          op.vcount = vcounts[q].as<int32_t>();
          op.bump_vcount = 1;
        }
      }
    }

    if (use_pgb) {
      prof_scope ps("groupby_aggregate", stream);
      pgb_args pa{};
      pa.mkeys = pgb_keys.as<uint64_t>();
      pa.vals  = pgb_val ? pgb_vals.ptr : nullptr;
      pa.val_bytes = pgb_val ? type_width(pgb_val->type_id) : 0;
      pa.src_type  = pgb_val ? storage_type(pgb_val->type_id) : B2_INT64;
      pa.part_base = pgb_base.as<uint32_t>();
      pa.part_end  = pgb_base.as<uint32_t>() + 256;
      pa.n = (uint32_t)n;
      pa.item_start = pgb_items.as<uint32_t>();
      pa.item_counter = pgb_items.as<uint32_t>() + 257;
      pa.chunk = pgb_chunk_rows(n);
      pa.nops = ops.n;
      for (int k = 0; k < ops.n; ++k) {
        pa.op[k] = ops.op[k].op; pa.acc[k] = ops.op[k].acc; pa.accum[k] = ops.op[k].accum; pa.init[k] = acc_init(ops.op[k].acc, ops.op[k].op);
      }
      pa.smem_slots = ops.n <= 1 ? 8192u : 4096u;
      {
        static const uint32_t forced = [] {  // test hook: a tiny shared table exercises the spill to the global table
          const char* e = std::getenv("B2_GROUPBY_SMEM_SLOTS");
          uint32_t v = e ? (uint32_t)std::atoi(e) : 0u;
          while (v & (v - 1)) v &= v - 1;  // power of two
          return v;
        }();
        if (forced >= 16 && forced < pa.smem_slots) pa.smem_slots = forced;
      }
      pa.smem_limit = pa.smem_slots * 6 / 10;
      const size_t smem = (size_t)pa.smem_slots * (8 + 8 * (size_t)ops.n + 4);
      static std::atomic<uint64_t> attr_done{0};
      once_per_device(attr_done, [] {
        B2_CUDA_TRY(cudaFuncSetAttribute(pgb_agg_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 20));
        B2_CUDA_TRY(cudaFuncSetAttribute(pgb_agg_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 20));
        B2_CUDA_TRY(cudaFuncSetAttribute(pgb_agg_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 20));
        B2_CUDA_TRY(cudaFuncSetAttribute(pgb_agg_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 20));
      });
      B2_CUDA_TRY(cudaMemsetAsync(pa.item_counter, 0, sizeof(uint32_t), stream));
      B2_LAUNCH(pgb_items_kernel, 1, 256, 0, stream, pa.part_base, pgb_base.as<uint32_t>() + 256, pgb_ends_given, pa.n, pa.chunk,
                pgb_items.as<uint32_t>());
      int mode = 0;
      if (ops.n == 0) mode = 3;
      else if (ops.n == 1 && pa.op[0] == OPK_SUM && pa.val_bytes == 8) mode = pa.acc[0] == ACC_F64 ? 1 : 2;
#define B2_PGB(M) B2_LAUNCH((pgb_agg_kernel<M>), num_sms(), PGB_THREADS, smem, stream, pa, table.as<slot_t>(), (uint32_t)(slots - 1), cap, \
                            gsize.as<int32_t>(), slot_gid.as<int32_t>(), ctl.as<gb_ctl>())
      switch (mode) {
        case 1: B2_PGB(1); break;
        case 2: B2_PGB(2); break;
        case 3: B2_PGB(3); break;
        default: B2_PGB(0); break;
      }
#undef B2_PGB
    } else {
      prof_scope ps("groupby_aggregate", stream);
#define B2_GB(W, Q)                                                                                                                    \
  B2_LAUNCH((groupby_kernel<W, Q>), grid_for(n), 256, 0, stream, kc, n, skip_null_keys, table.as<slot_t>(), (uint32_t)(slots - 1), cap, \
            gsize.as<int32_t>(), slot_gid.as<int32_t>(), rep_rows.as<int32_t>(), ops, ctl.as<gb_ctl>())
      if (wide) { if (any_sumsq) B2_GB(true, true); else B2_GB(true, false); }
      else      { if (any_sumsq) B2_GB(false, true); else B2_GB(false, false); }
#undef B2_GB
    }
    gb_ctl h{};
    B2_CUDA_TRY(cudaMemcpyAsync(&h, ctl.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    if (h.overflow) {
      B2_EXPECTS(slots < max_slots, B2_ERR_LOGIC, "groupby: hash table overflow at maximum size");
      slots = std::min<uint64_t>(max_slots, slots * 8);
      continue;  // buffers are released (stream-ordered) and rebuilt at the new size
    }
    const int32_t G = (int32_t)h.ngroups;

    // ---- outputs ----
    if (use_pgb) {
      keys_out = std::make_unique<b2_table>();
      keys_out->cols.push_back(make_column(gb.keys[0].type_id, G, false, stream));
      if (G > 0)
        B2_LAUNCH(pgb_keys_kernel, grid_for((int64_t)slots), 256, 0, stream, table.as<slot_t>(), (int64_t)slots, slot_gid.as<int32_t>(),
                  keys_out->cols[0]->data.as<uint64_t>());
    } else {
      keys_out = gather_table(gb.keys, rep_rows.as<int32_t>(), G, false, stream);
    }
    res_out  = std::make_unique<b2_table>();
    for (size_t q = 0; q < reqs.size(); ++q) {
      const auto& v = reqs[q].values;
      const bool nullable = has_nulls(v);
      for (size_t j = 0; j < reqs[q].kinds.size(); ++j) {
        const int32_t kind = base_kind(reqs[q].kinds[j]);
        const int32_t rt   = result_type(kind, v.type_id);
        const bool counts  = kind == B2_AGG_COUNT_VALID || kind == B2_AGG_COUNT_ALL;
        const bool var_std = kind == B2_AGG_VARIANCE || kind == B2_AGG_STD;  // null where count - ddof <= 0 (m2_var_std.cu:150-196)
        const bool ext     = var_std || kind == B2_AGG_M2;
        // result has a mask only when the input column has nulls (output_utils.cu:67-86); counts and M2 never;
        // VARIANCE / STD build theirs from the group counts
        auto col = make_column(rt, G, var_std || (nullable && !counts && kind != B2_AGG_M2), stream);
        if (G > 0) {
          out_spec o{};
          o.gsize  = gsize.as<int32_t>();
          o.vcount = nullable ? vcounts[q].as<int32_t>() : nullptr;
          o.out    = col->data.ptr;
          o.out_type = storage_type(rt);
          if (counts) {
            o.mode = kind == B2_AGG_COUNT_VALID ? 2 : 3;
          } else {
            const value_op& op = ops.op[op_of[q][j]];
            o.accum = op.accum;
            o.acc   = op.acc;
            o.op    = (op.op == OPK_SUMSQ || op.op == OPK_PROD) ? (int8_t)OPK_SUM : op.op;  // finalize: "plain accumulator bits", like SUM
            if (op.op == OPK_ARGMIN || op.op == OPK_ARGMAX) { o.acc = ACC_I64; o.op = OPK_SUM; }  // a row index, stored as INT32
            o.mode  = kind == B2_AGG_MEAN ? 1 : (kind == B2_AGG_M2 ? 5 : (kind == B2_AGG_VARIANCE ? 6 : (kind == B2_AGG_STD ? 7 : 0)));
            if (ext) {
              o.accum2 = ops.op[op2_of[q][j]].accum;
              o.ddof   = kind_ddof(reqs[q].kinds[j]);
            }
            if (var_std || (nullable && kind != B2_AGG_M2)) {
              o.out_mask = col->mask.as<uint32_t>();
              col->pending = dbuf(sizeof(unsigned long long), stream);
              col->pending_stream = stream;
              col->null_count = -1;
              B2_CUDA_TRY(cudaMemsetAsync(col->pending.ptr, 0, sizeof(unsigned long long), stream));
              o.null_count = col->pending.as<unsigned long long>();
            }
          }
          if (ext)
            B2_LAUNCH((finalize_kernel<true>), grid_for((int64_t)slots), 256, 0, stream, table.as<slot_t>(), (int64_t)slots,
                      slot_gid.as<int32_t>(), o);
          else
            B2_LAUNCH((finalize_kernel<false>), grid_for((int64_t)slots), 256, 0, stream, table.as<slot_t>(), (int64_t)slots,
                      slot_gid.as<int32_t>(), o);
        }
        res_out->cols.push_back(std::move(col));
      }
    }
    return;
  }
}

// ---- grouped scan: sort keys (stable), permute values, segmented inclusive scan -----------------
namespace {

// head[i] = 1 when sorted row i starts a new group (packed key differs from row i-1)
template <bool WIDE = false>
__global__ void group_heads_kernel(key_cols kc, const int32_t* __restrict__ order, int64_t n, uint8_t* __restrict__ head)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint8_t h = 1;
    if (i > 0) {
      if constexpr (WIDE) {
        h = rows_equal_wide(kc, order[i - 1], kc, order[i]) ? 0 : 1;
      } else {
        uint64_t k0, k1;
        uint32_t n0, n1;
        pack_row(kc, order[i - 1], k0, n0);
        pack_row(kc, order[i], k1, n1);
        h = (k0 != k1 || n0 != n1) ? 1 : 0;
      }
    }
    head[i] = h;
  }
}

// Single-CTA-per-tile segmented scan in three steps (tile aggregates -> carries -> apply).
// Element = (value as 8-byte accumulator, valid flag); op: SUM / MIN / MAX / COUNT.
constexpr int SEG_TILE = 2048;

// MIN / MAX rank NaN above +inf (scan_reduce.cu's binop), so NaN is MIN's identity for doubles
template <typename A, int OPK>
__device__ __forceinline__ A seg_apply(A a, A b)
{
  if (OPK == OPK_SUM) return a + b;
  if (OPK == OPK_MIN) return (b < a || a != a) ? b : a;  // a != a: a is NaN (false for integers)
  return (a < b || b != b) ? b : a;
}
template <typename A, int OPK>
__device__ __forceinline__ A seg_identity()
{
  if (OPK == OPK_SUM) return A(0);
  if (OPK == OPK_MIN) return sizeof(A) == 8 && ((A)-1 < A(0)) ? (A)INT64_MAX : (A)~0ull;
  return ((A)-1 < A(0)) ? (A)INT64_MIN : A(0);
}
template <> __device__ __forceinline__ double seg_identity<double, OPK_MIN>() { return __longlong_as_double(0x7ff8000000000000ll); }
template <> __device__ __forceinline__ double seg_identity<double, OPK_MAX>() { return __longlong_as_double(0xfff0000000000000ll); }

template <typename A>
__device__ __forceinline__ A load_acc(const void* src, int32_t st, int64_t e)
{
  switch (st) {
    case B2_INT8: return (A) static_cast<const int8_t*>(src)[e];
    case B2_INT16: return (A) static_cast<const int16_t*>(src)[e];
    case B2_INT32: return (A) static_cast<const int32_t*>(src)[e];
    case B2_INT64: return (A) static_cast<const int64_t*>(src)[e];
    case B2_UINT8: return (A) static_cast<const uint8_t*>(src)[e];
    case B2_UINT16: return (A) static_cast<const uint16_t*>(src)[e];
    case B2_UINT32: return (A) static_cast<const uint32_t*>(src)[e];
    case B2_UINT64: return (A) static_cast<const uint64_t*>(src)[e];
    case B2_BOOL8: return (A)(static_cast<const uint8_t*>(src)[e] != 0);
    case B2_FLOAT32: return (A) static_cast<const float*>(src)[e];
    default: return (A) static_cast<const double*>(src)[e];
  }
}
template <typename A>
__device__ __forceinline__ void store_acc(void* dst, int32_t st, int64_t i, A a)
{
  switch (st) {
    case B2_INT8: static_cast<int8_t*>(dst)[i] = (int8_t)a; break;
    case B2_INT16: static_cast<int16_t*>(dst)[i] = (int16_t)a; break;
    case B2_INT32: static_cast<int32_t*>(dst)[i] = (int32_t)a; break;
    case B2_INT64: static_cast<int64_t*>(dst)[i] = (int64_t)a; break;
    case B2_UINT8: case B2_BOOL8: static_cast<uint8_t*>(dst)[i] = (uint8_t)a; break;
    case B2_UINT16: static_cast<uint16_t*>(dst)[i] = (uint16_t)a; break;
    case B2_UINT32: static_cast<uint32_t*>(dst)[i] = (uint32_t)a; break;
    case B2_UINT64: static_cast<uint64_t*>(dst)[i] = (uint64_t)a; break;
    case B2_FLOAT32: static_cast<float*>(dst)[i] = (float)a; break;
    default: static_cast<double*>(dst)[i] = (double)a; break;
  }
}

struct seg_args {
  const void* src;          // original (unsorted) values; null for COUNT_ALL
  const uint32_t* mask;     // original validity or null
  int32_t offset;
  int32_t src_type;
  const int32_t* order;     // sorted row -> source row
  const uint8_t* head;
  int64_t n;
  int32_t count_mode;       // 1: element value is 1 per valid row (COUNT)
  void* out;
  int32_t out_type;
  uint32_t* out_mask;       // validity of the permuted values (null when source has no nulls)
  unsigned long long* out_valid_count;
};

// one thread scans one tile sequentially in phase A/C (tiles are small; this is not the headline
// path) — phase A: tile summary {has_head, prefix-before-first-head, suffix-after-last-head}
template <typename A, int OPK>
__global__ void seg_tile_summary_kernel(seg_args a, A* __restrict__ tail, uint8_t* __restrict__ has_head)
{
  const int64_t ntiles = (a.n + SEG_TILE - 1) / SEG_TILE;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntiles) return;
  const int64_t b = t * SEG_TILE, e = min(a.n, b + SEG_TILE);
  A run = seg_identity<A, OPK>();
  uint8_t hh = 0;
  for (int64_t i = b; i < e; ++i) {
    if (a.head[i]) { run = seg_identity<A, OPK>(); hh = 1; }
    const int64_t r = a.order[i];
    const bool valid = a.mask == nullptr || bit_is_set(a.mask, r + a.offset);
    if (valid) run = seg_apply<A, OPK>(run, a.count_mode ? A(1) : load_acc<A>(a.src, a.src_type, r + a.offset));
  }
  tail[t] = run;        // running value at the end of the tile (since the last head, or whole tile)
  has_head[t] = hh;
}
// phase B: sequential carry over tiles (ntiles = n/2048: tiny)
template <typename A, int OPK>
__global__ void seg_carry_kernel(A* __restrict__ tail, const uint8_t* __restrict__ has_head, int64_t ntiles, A* __restrict__ carry)
{
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  A c = seg_identity<A, OPK>();
  for (int64_t t = 0; t < ntiles; ++t) {
    carry[t] = c;  // value carried INTO tile t (applies until its first head)
    c = has_head[t] ? tail[t] : seg_apply<A, OPK>(c, tail[t]);
  }
}
template <typename A, int OPK>
__global__ void seg_apply_kernel(seg_args a, const A* __restrict__ carry)
{
  const int64_t ntiles = (a.n + SEG_TILE - 1) / SEG_TILE;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntiles) return;
  const int64_t b = t * SEG_TILE, e = min(a.n, b + SEG_TILE);
  A run = carry[t];
  unsigned long long nvalid = 0;
  for (int64_t i = b; i < e; ++i) {
    if (a.head[i]) run = seg_identity<A, OPK>();
    const int64_t r = a.order[i];
    const bool valid = a.mask == nullptr || bit_is_set(a.mask, r + a.offset);
    if (valid) {
      run = seg_apply<A, OPK>(run, a.count_mode ? A(1) : load_acc<A>(a.src, a.src_type, r + a.offset));
      ++nvalid;
      if (a.out_mask) atomicOr(&a.out_mask[i >> 5], 1u << (i & 31));
    }
    store_acc<A>(a.out, a.out_type, i, run);
  }
  if (a.out_valid_count && nvalid) atomicAdd(a.out_valid_count, nvalid);
}

template <typename A, int OPK>
void run_seg_scan(seg_args a, cudaStream_t stream)
{
  const int64_t ntiles = (a.n + SEG_TILE - 1) / SEG_TILE;
  dbuf tail(sizeof(A) * ntiles, stream), carry(sizeof(A) * ntiles, stream), hh(ntiles, stream);
  const int grid = (int)((ntiles + 127) / 128);
  B2_LAUNCH((seg_tile_summary_kernel<A, OPK>), grid, 128, 0, stream, a, tail.as<A>(), hh.as<uint8_t>());
  B2_LAUNCH((seg_carry_kernel<A, OPK>), 1, 32, 0, stream, tail.as<A>(), hh.as<uint8_t>(), ntiles, carry.as<A>());
  B2_LAUNCH((seg_apply_kernel<A, OPK>), grid, 128, 0, stream, a, carry.as<A>());
}

}  // namespace

// cudf::groupby::groupby::scan — groupby.cu:240-259 -> sort_scan
void groupby_scan(const b2_groupby& gb, const std::vector<request_view>& reqs, cudaStream_t stream, table_ptr& keys_out,
                  table_ptr& res_out)
{
  const int64_t n_all = gb.keys.empty() ? 0 : gb.keys[0].size;
  for (auto& r : reqs) {
    validate_column(r.values);
    B2_EXPECTS(r.values.size == n_all, B2_ERR_LOGIC, "Size mismatch between request values and groupby keys.");
    for (int32_t kind : r.kinds)
      B2_EXPECTS(kind == B2_AGG_SUM || kind == B2_AGG_MIN || kind == B2_AGG_MAX || kind == B2_AGG_COUNT_VALID || kind == B2_AGG_COUNT_ALL,
                 B2_ERR_INVALID_ARGUMENT, "unsupported groupby scan aggregation (SUM/MIN/MAX/COUNT)");
  }
  if (n_all == 0) return empty_results(gb, reqs, stream, keys_out, res_out);
  key_cols kc = make_key_cols(gb.keys, true);

  // sorted order of the keys (ascending, nulls first), null-key rows dropped under EXCLUDE
  std::vector<uint8_t> asc(gb.keys.size(), B2_ASCENDING), before(gb.keys.size(), B2_NULL_BEFORE);
  auto order_col = sorted_order(gb.keys, asc, before, true, stream);
  const int32_t* order = order_col->data.as<int32_t>();
  int64_t n = n_all;
  bool keys_nullable = false;
  for (auto& k : gb.keys) keys_nullable |= has_nulls(k);
  if (keys_nullable && gb.null_handling == B2_NULL_EXCLUDE) {
    // rows with any null key sort first only for single-column keys; in general count and filter them
    int32_t nulls = 0;
    dbuf m = bitmask_and(gb.keys, (int32_t)n_all, &nulls, stream);
    if (nulls > 0) {
      B2_EXPECTS(gb.keys.size() == 1, B2_ERR_INVALID_ARGUMENT,
                 "groupby scan with null keys under EXCLUDE supports a single key column on this path");
      order += nulls;  // ascending, nulls BEFORE: the null-key rows are the first `nulls` entries
      n -= nulls;
    }
  }
  keys_out = gather_table(gb.keys, order, (int32_t)n, false, stream);
  res_out  = std::make_unique<b2_table>();
  if (n == 0) {
    for (auto& r : reqs)
      for (int32_t kind : r.kinds) res_out->cols.push_back(make_column(result_type(kind, r.values.type_id), 0, false, stream));
    return;
  }
  dbuf head(n, stream);
  if (keys_are_wide(gb.keys)) B2_LAUNCH((group_heads_kernel<true>), grid_for(n), 256, 0, stream, kc, order, n, head.as<uint8_t>());
  else B2_LAUNCH((group_heads_kernel<false>), grid_for(n), 256, 0, stream, kc, order, n, head.as<uint8_t>());

  for (auto& r : reqs) {
    const auto& v = r.values;
    const int32_t st = storage_type(v.type_id);
    const bool nullable = has_nulls(v);
    for (int32_t kind : r.kinds) {
      const bool counts = kind == B2_AGG_COUNT_VALID || kind == B2_AGG_COUNT_ALL;
      const int32_t rt = result_type(kind, v.type_id);
      auto col = make_column(rt, (int32_t)n, nullable && !counts, stream);
      seg_args a{};
      a.src = v.data; a.mask = (nullable && kind != B2_AGG_COUNT_ALL) ? v.null_mask : nullptr; a.offset = v.offset; a.src_type = st;
      a.order = order; a.head = head.as<uint8_t>(); a.n = n; a.count_mode = counts ? 1 : 0;
      a.out = col->data.ptr; a.out_type = storage_type(rt);
      if (nullable && !counts) {
        a.out_mask = col->mask.as<uint32_t>();
        col->pending = dbuf(sizeof(unsigned long long), stream);
        col->pending_stream = stream;
        col->pending_is_valid_count = true;
        col->null_count = -1;
        B2_CUDA_TRY(cudaMemsetAsync(col->pending.ptr, 0, sizeof(unsigned long long), stream));
        a.out_valid_count = col->pending.as<unsigned long long>();
      }
      const bool flt = is_float_id(st) && !counts;
      const bool uns = !is_signed_id(st) && !flt && !counts;
      if (counts || kind == B2_AGG_SUM) {
        if (flt) run_seg_scan<double, OPK_SUM>(a, stream);
        else run_seg_scan<long long, OPK_SUM>(a, stream);
      } else if (kind == B2_AGG_MIN) {
        if (flt) run_seg_scan<double, OPK_MIN>(a, stream);
        else if (uns) run_seg_scan<unsigned long long, OPK_MIN>(a, stream);
        else run_seg_scan<long long, OPK_MIN>(a, stream);
      } else {
        if (flt) run_seg_scan<double, OPK_MAX>(a, stream);
        else if (uns) run_seg_scan<unsigned long long, OPK_MAX>(a, stream);
        else run_seg_scan<long long, OPK_MAX>(a, stream);
      }
      res_out->cols.push_back(std::move(col));
    }
  }
}

// ---- sort-based aggregate -----------------------------------------------------------------------------------------------
// cudf::groupby falls back to its sort-based implementation when the keys are declared pre-sorted or when a requested
// aggregation has no hash implementation (cpp/src/groupby/groupby.cu:76-99 dispatch_aggregation, cpp/src/groupby/sort/
// aggregate.cpp, sort_helper.cu; per-aggregation group_*.cu).  Here: stable sorted order of the keys (radix_sort.cu) ->
// group boundaries -> values gathered into group order -> one segmented reduction per aggregation (scan_reduce.cu); the
// order-dependent ones (NTH_ELEMENT, NUNIQUE, MEDIAN) read the group order / a second order by (keys, values).
// Output: one row per group in ascending key order (nulls first), the sort path's order in the reference.
namespace {

__global__ void gb_offsets_kernel(const uint8_t* __restrict__ head, const int32_t* __restrict__ gid_incl, int64_t n, int32_t G,
                                  int32_t* __restrict__ offsets)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (head[i]) offsets[gid_incl[i] - 1] = (int32_t)i;
    if (i == 0) offsets[G] = (int32_t)n;
  }
}
__global__ void gb_head32_kernel(const uint8_t* __restrict__ head, int64_t n, int32_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = head[i];
}
__global__ void gb_rep_rows_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ offsets, int32_t G, int32_t* __restrict__ rep)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) rep[g] = order[offsets[g]];
}
__global__ void gb_sizes_kernel(const int32_t* __restrict__ offsets, int32_t G, int32_t* __restrict__ out)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) out[g] = offsets[g + 1] - offsets[g];
}
__global__ void gb_valid_flags_kernel(const uint32_t* __restrict__ mask, int64_t n, int32_t* __restrict__ flags)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) flags[i] = (mask == nullptr || bit_is_set(mask, i)) ? 1 : 0;
}
// NTH_ELEMENT: gather map into the group-ordered values; out-of-range picks become nulls (INT32_MIN is out of bounds for gather)
__global__ void gb_nth_map_kernel(const int32_t* __restrict__ offsets, int32_t G, int32_t nth, int32_t* __restrict__ map)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int32_t size = offsets[g + 1] - offsets[g];
  const int32_t idx = nth >= 0 ? nth : size + nth;
  map[g] = (idx >= 0 && idx < size) ? offsets[g] + idx : INT32_MIN;
}
// values as doubles (and their squares) / as wrapped 64-bit integers squared: inputs of SUM_OF_SQUARES / M2 / VARIANCE / STD
__global__ void gb_squares_kernel(const void* __restrict__ src, int32_t st, int64_t n, double* __restrict__ x, double* __restrict__ x2,
                                  long long* __restrict__ i2)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double d = 0;
    long long w = 0;
    switch (st) {
      case B2_INT8: w = static_cast<const int8_t*>(src)[i]; d = (double)w; break;
      case B2_INT16: w = static_cast<const int16_t*>(src)[i]; d = (double)w; break;
      case B2_INT32: w = static_cast<const int32_t*>(src)[i]; d = (double)w; break;
      case B2_INT64: w = static_cast<const int64_t*>(src)[i]; d = (double)w; break;
      case B2_UINT8: case B2_BOOL8: w = static_cast<const uint8_t*>(src)[i]; d = (double)w; break;
      case B2_UINT16: w = static_cast<const uint16_t*>(src)[i]; d = (double)w; break;
      case B2_UINT32: w = static_cast<const uint32_t*>(src)[i]; d = (double)w; break;
      case B2_UINT64: { const unsigned long long u = static_cast<const unsigned long long*>(src)[i]; w = (long long)u; d = (double)u; break; }
      case B2_FLOAT32: d = static_cast<const float*>(src)[i]; break;
      default: d = static_cast<const double*>(src)[i]; break;
    }
    if (x) x[i] = d;
    if (x2) x2[i] = d * d;
    if (i2) i2[i] = (long long)((unsigned long long)w * (unsigned long long)w);
  }
}
// MEAN of an integral column on the sort path, as the reference's (aggregate.cpp:275-298: a DIV of the SUM and COUNT_VALID results,
// in double) and the hash path's finalize_kernel: the group's wrapped INT64 SUM over its valid count. In place: sum and out may alias.
__global__ void gb_int_mean_kernel(const long long* sum, const int32_t* __restrict__ cnt, int32_t G, double* out)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int32_t c = cnt[g];
  const long long s = sum[g];
  out[g] = c > 0 ? (double)s / (double)c : 0.0;
}
// The sort path's M2 / VARIANCE / STD take two passes, as the reference's sort path does (cpp/src/groupby/sort/group_m2.cu:34-58,
// group_std.cu:19-52, aggregate.cpp:303-353): the group MEAN first, then per valid row (x - mean)^2, divided by (n - ddof) for
// VARIANCE / STD, summed per group. Null rows and rows of a group with n <= ddof contribute 0.
__global__ void gb_dev2_kernel(const double* __restrict__ x, const uint32_t* __restrict__ mask, const int32_t* __restrict__ gid_incl, int64_t n,
                               const double* __restrict__ mean, const int32_t* __restrict__ cnt, int var, int32_t ddof, double* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double t = 0.0;
    if (mask == nullptr || bit_is_set(mask, i)) {
      const int32_t g = gid_incl[i] - 1;
      const double d = x[i] - mean[g];
      t = d * d;
      if (var) {
        const int32_t df = cnt[g] - ddof;
        t = df > 0 ? t / df : 0.0;
      }
    }
    out[i] = t;
  }
}
// VARIANCE / STD from the per-group sum of gb_dev2_kernel's terms: null where the group has no valid value or n <= ddof
__global__ void gb_var_std_kernel(const double* __restrict__ s, const int32_t* __restrict__ cnt, int32_t G, int32_t ddof, int is_std,
                                  double* __restrict__ out, uint32_t* __restrict__ out_mask, unsigned long long* __restrict__ valid_count)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int32_t n = cnt[g];
  const bool valid = n != 0 && n - ddof > 0;
  out[g] = valid ? (is_std ? sqrt(s[g]) : s[g]) : 0.0;
  if (valid) {
    atomicOr(&out_mask[g >> 5], 1u << (g & 31));
    atomicAdd(valid_count, 1ull);
  }
}
// NUNIQUE: rows are ordered by (keys, value) with null values last inside a group; a valid row counts when it opens its group
// or differs from its predecessor (floats: -0 == +0, NaN == NaN as in the reference's equality comparator)
template <typename T>
__global__ void gb_distinct_flags_kernel(const T* __restrict__ v, const uint32_t* __restrict__ mask, const int32_t* __restrict__ gid_incl, int64_t n,
                                         int is_float, int32_t* __restrict__ flags)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  auto norm = [&](T b) -> T {
    if (!is_float) return b;
    if constexpr (sizeof(T) == 4) {
      if ((b << 1) == 0) return 0;
      if ((b & 0x7fffffffu) > 0x7f800000u) return (T)0x7fc00000u;
    } else if constexpr (sizeof(T) == 8) {
      if ((b << 1) == 0) return 0;
      if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return (T)0x7ff8000000000000ull;
    }
    return b;
  };
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool valid = mask == nullptr || bit_is_set(mask, i);
    int32_t f = 0;
    if (valid) {
      const bool first = i == 0 || gid_incl[i] != gid_incl[i - 1];
      f = (first || norm(v[i]) != norm(v[i - 1])) ? 1 : 0;
    }
    flags[i] = f;
  }
}
// a * b rounded on its own: never contracted into an FMA with the add it feeds
__device__ __forceinline__ double mul_rn(double a, double b)
{
#ifdef B2_EMU  // tests/emu: a plain C++ build for x86-64 has no FMA to contract into
  return a * b;
#else
  return __dmul_rn(a, b);
#endif
}
// MEDIAN = 0.5 quantile with linear interpolation over the group's valid values (sorted ascending, NaN then nulls last):
// (1 - f) * a + f * b as the reference's interpolate::linear (cpp/src/quantiles/quantiles_util.hpp:23-36,73-89), so an odd
// count whose middle value is +-inf gives NaN (0 * inf) and {-inf, 5} gives -inf. Both products are rounded on their own, not
// contracted into an FMA: with f in {0, 0.5} they are exact except for subnormal halves, whose rounding is then fixed.
__global__ void gb_median_kernel(const double* __restrict__ x, const int32_t* __restrict__ offsets, const int32_t* __restrict__ valid_cnt, int32_t G,
                                 double* __restrict__ out, uint32_t* __restrict__ out_mask, unsigned long long* __restrict__ valid_count)
{
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const int32_t m = valid_cnt[g];
  if (m == 0) { out[g] = 0.0; return; }
  const double pos = (m - 1) * 0.5;
  const int32_t lo = (int32_t)floor(pos), hi = (int32_t)ceil(pos);
  const double a = x[offsets[g] + lo], b = x[offsets[g] + hi], frac = pos - lo;
  out[g] = mul_rn(1.0 - frac, a) + mul_rn(frac, b);
  atomicOr(&out_mask[g >> 5], 1u << (g & 31));
  atomicAdd(valid_count, 1ull);
}

constexpr int32_t AGG_MEDIAN = 14, AGG_NUNIQUE = 18, AGG_NTH_ELEMENT = 19;  // aggregation::Kind values (aggregation.hpp:78-121)
// B2_AGG_WITH_DDOF carries a 16-bit parameter: ddof for VARIANCE / STD, n (signed) for NTH_ELEMENT
inline int32_t kind_param_signed(int32_t k) { return (k & (1 << 30)) ? (int32_t)(int16_t)((k >> 8) & 0xFFFF) : 0; }

int32_t sorted_result_type(int32_t kind, int32_t src)
{
  switch (kind) {
    case AGG_MEDIAN: return B2_FLOAT64;
    case AGG_NUNIQUE: return B2_INT32;
    case AGG_NTH_ELEMENT: return src;
    default: return result_type(kind, src);
  }
}

void mark_pending_valid(b2_column& c, cudaStream_t stream)
{
  c.pending = dbuf(sizeof(unsigned long long), stream);
  c.pending_stream = stream;
  c.pending_is_valid_count = true;
  c.null_count = -1;
  B2_CUDA_TRY(cudaMemsetAsync(c.pending.ptr, 0, sizeof(unsigned long long), stream));
}

}  // namespace

bool groupby_needs_sort_path(const b2_groupby& gb, const std::vector<request_view>& reqs)
{
  if (gb.keys_are_sorted) return true;
  if (const char* e = std::getenv("B2_GROUPBY_SORT")) if (std::atoi(e) != 0) return true;  // test hook
  for (auto& r : reqs)
    for (int32_t raw : r.kinds) {
      const int32_t k = base_kind(raw);
      if (k == AGG_MEDIAN || k == AGG_NUNIQUE || k == AGG_NTH_ELEMENT) return true;
    }
  return false;
}

void groupby_aggregate_sorted(const b2_groupby& gb, const std::vector<request_view>& reqs, cudaStream_t stream, table_ptr& keys_out,
                              table_ptr& res_out)
{
  const int64_t n_all = gb.keys.empty() ? 0 : gb.keys[0].size;
  for (auto& r : reqs) {
    validate_column(r.values);
    B2_EXPECTS(r.values.size == n_all, B2_ERR_LOGIC, "Size mismatch between request values and groupby keys.");
    B2_EXPECTS(!r.kinds.empty(), B2_ERR_LOGIC, "Empty aggregation request");
    for (int32_t raw : r.kinds) {
      const int32_t k = base_kind(raw);
      const bool ok = k == B2_AGG_SUM || k == B2_AGG_PRODUCT || k == B2_AGG_MIN || k == B2_AGG_MAX || k == B2_AGG_MEAN || k == B2_AGG_COUNT_VALID ||
                      k == B2_AGG_COUNT_ALL || needs_sumsq(k) || k == AGG_MEDIAN || k == AGG_NUNIQUE || k == AGG_NTH_ELEMENT;
      B2_EXPECTS(ok, B2_ERR_INVALID_ARGUMENT, "unsupported aggregation on the sort-based groupby path");
      if (k != B2_AGG_MIN && k != B2_AGG_MAX && k != B2_AGG_COUNT_VALID && k != B2_AGG_COUNT_ALL && k != AGG_NUNIQUE && k != AGG_NTH_ELEMENT)
        B2_EXPECTS(is_numeric(r.values.type_id), B2_ERR_LOGIC, "this aggregation needs a numeric values column");
    }
  }
  auto empty = [&] {
    keys_out = std::make_unique<b2_table>();
    for (auto& k : gb.keys) keys_out->cols.push_back(make_column(k.type_id, 0, false, stream));
    res_out = std::make_unique<b2_table>();
    for (auto& r : reqs)
      for (int32_t kind : r.kinds) res_out->cols.push_back(make_column(sorted_result_type(base_kind(kind), r.values.type_id), 0, false, stream));
  };
  if (n_all == 0) return empty();
  key_cols kc = make_key_cols(gb.keys, true);

  // order of the rows by key: ascending, nulls first (or the given order when the caller says the keys are sorted);
  // rows with a null key are dropped under EXCLUDE (single key column, as in groupby_scan)
  std::vector<uint8_t> asc(gb.keys.size(), B2_ASCENDING), before(gb.keys.size(), B2_NULL_BEFORE);
  column_ptr order_col;
  int64_t n = n_all;
  int64_t skip = 0;
  bool keys_nullable = false;
  for (auto& k : gb.keys) keys_nullable |= has_nulls(k);
  int32_t null_rows = 0;
  if (keys_nullable && gb.null_handling == B2_NULL_EXCLUDE) {
    dbuf m = bitmask_and(gb.keys, (int32_t)n_all, &null_rows, stream);
    if (null_rows > 0)
      B2_EXPECTS(gb.keys.size() == 1, B2_ERR_INVALID_ARGUMENT, "sort-based groupby with null keys under EXCLUDE supports a single key column on this path");
  }
  order_col = sorted_order(gb.keys, asc, before, true, stream);  // pre-sorted keys sort to the same grouping (stable), no shortcut needed for correctness
  skip = null_rows;
  n -= skip;
  const int32_t* order = order_col->data.as<int32_t>() + skip;
  if (n == 0) return empty();

  // group boundaries
  dbuf head(n, stream), head32(sizeof(int32_t) * n, stream);
  if (keys_are_wide(gb.keys)) B2_LAUNCH((group_heads_kernel<true>), grid_for(n), 256, 0, stream, kc, order, n, head.as<uint8_t>());
  else B2_LAUNCH((group_heads_kernel<false>), grid_for(n), 256, 0, stream, kc, order, n, head.as<uint8_t>());
  B2_LAUNCH(gb_head32_kernel, grid_for(n), 256, 0, stream, head.as<uint8_t>(), n, head32.as<int32_t>());
  b2_column_view hv{B2_INT32, (int32_t)n, head32.ptr, nullptr, 0, 0};
  auto gid = scan(hv, B2_AGG_SUM, B2_SCAN_INCLUSIVE, B2_NULL_EXCLUDE, stream);  // 1-based group number of every sorted row
  int32_t G = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&G, gid->data.as<int32_t>() + (n - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  dbuf offsets(sizeof(int32_t) * ((size_t)G + 1), stream);
  B2_LAUNCH(gb_offsets_kernel, grid_for(n), 256, 0, stream, head.as<uint8_t>(), gid->data.as<int32_t>(), n, G, offsets.as<int32_t>());
  const int32_t* off = offsets.as<int32_t>();
  const int ggrid = (G + 255) / 256;
  {
    dbuf rep(sizeof(int32_t) * (size_t)G, stream);
    B2_LAUNCH(gb_rep_rows_kernel, ggrid, 256, 0, stream, order, off, G, rep.as<int32_t>());
    keys_out = gather_table(gb.keys, rep.as<int32_t>(), G, false, stream);
  }
  res_out = std::make_unique<b2_table>();

  for (auto& r : reqs) {
    const auto& v = r.values;
    const int32_t st = storage_type(v.type_id);
    const bool nullable = has_nulls(v);
    auto vs = gather_column(v, order, (int32_t)n, false, stream);  // values in group order (input order inside a group)
    const b2_column_view vsv = vs->view();
    // valid count per group (shared by COUNT_VALID, M2 / VARIANCE / STD, MEDIAN)
    column_ptr vcnt;
    auto valid_counts = [&]() -> const int32_t* {
      if (!vcnt) {
        dbuf flags(sizeof(int32_t) * n, stream);
        B2_LAUNCH(gb_valid_flags_kernel, grid_for(n), 256, 0, stream, nullable ? vsv.null_mask : nullptr, n, flags.as<int32_t>());
        b2_column_view fv{B2_INT32, (int32_t)n, flags.ptr, nullptr, 0, 0};
        vcnt = segmented_reduce(fv, off, G + 1, B2_AGG_SUM, B2_INT32, B2_NULL_EXCLUDE, nullptr, stream);
        vcnt->mask.reset();
        vcnt->pending.reset();
        vcnt->null_count = 0;
      }
      return vcnt->data.as<int32_t>();
    };
    // the second order, by (keys, values): shares the group boundaries, sorts the values inside each group (nulls last)
    column_ptr vs2;
    auto values_sorted_in_group = [&]() -> const b2_column& {
      if (!vs2) {
        std::vector<b2_column_view> kv = gb.keys;
        kv.push_back(v);
        std::vector<uint8_t> a2(kv.size(), B2_ASCENDING), p2(kv.size(), B2_NULL_BEFORE);
        p2.back() = B2_NULL_AFTER;
        auto o2 = sorted_order(kv, a2, p2, true, stream);
        vs2 = gather_column(v, o2->data.as<int32_t>() + skip, (int32_t)n, false, stream);
      }
      return *vs2;
    };
    // MEAN (alone, and the first pass of M2 / VARIANCE / STD): for integral values the INT64 SUM over the valid count, so that a
    // sum above 2^53 or one that wraps gives the reference's result; float values are converted to double and summed in double
    auto group_mean = [&](const b2_column_view& xv) -> column_ptr {
      if (!is_integral_id(st)) return segmented_reduce(xv, off, G + 1, B2_AGG_MEAN, B2_FLOAT64, B2_NULL_EXCLUDE, nullptr, stream);
      b2_column_view sv = vsv;
      sv.type_id = st;
      auto col = segmented_reduce(sv, off, G + 1, B2_AGG_SUM, B2_INT64, B2_NULL_EXCLUDE, nullptr, stream);
      const int32_t* vc = valid_counts();
      B2_LAUNCH(gb_int_mean_kernel, ggrid, 256, 0, stream, col->data.as<long long>(), vc, G, col->data.as<double>());
      col->type_id = B2_FLOAT64;
      return col;
    };
    for (int32_t raw : r.kinds) {
      const int32_t kind = base_kind(raw);
      const int32_t rt = sorted_result_type(kind, v.type_id);
      column_ptr col;
      if (kind == B2_AGG_COUNT_ALL) {
        col = make_column(B2_INT32, G, false, stream);
        B2_LAUNCH(gb_sizes_kernel, ggrid, 256, 0, stream, off, G, col->data.as<int32_t>());
      } else if (kind == B2_AGG_COUNT_VALID) {
        col = make_column(B2_INT32, G, false, stream);
        B2_CUDA_TRY(cudaMemcpyAsync(col->data.ptr, valid_counts(), sizeof(int32_t) * (size_t)G, cudaMemcpyDeviceToDevice, stream));
      } else if (kind == B2_AGG_SUM || kind == B2_AGG_PRODUCT || kind == B2_AGG_MIN || kind == B2_AGG_MAX || kind == B2_AGG_MEAN) {
        b2_column_view sv = vsv;
        sv.type_id = (kind == B2_AGG_MIN || kind == B2_AGG_MAX) ? vsv.type_id : st;  // chrono sums go through their integer storage
        if (kind == B2_AGG_MEAN) col = group_mean(sv);
        else col = segmented_reduce(sv, off, G + 1, kind, (kind == B2_AGG_MIN || kind == B2_AGG_MAX) ? vsv.type_id : rt, B2_NULL_EXCLUDE, nullptr, stream);
        col->type_id = rt;
        if (!nullable) { col->pending.reset(); col->mask.reset(); col->null_count = 0; }  // a mask only when the input has nulls (output_utils.cu:67-86)
      } else if (needs_sumsq(kind)) {
        const bool sumsq = kind == B2_AGG_SUM_OF_SQUARES, want_int = sumsq && !is_float_id(st);
        dbuf x(sumsq ? 0 : sizeof(double) * n, stream), x2(sumsq && !want_int ? sizeof(double) * n : 0, stream), i2(want_int ? sizeof(long long) * n : 0, stream);
        B2_LAUNCH(gb_squares_kernel, grid_for(n), 256, 0, stream, vsv.data, st, n, x.as<double>(), x2.as<double>(), i2.as<long long>());
        if (kind == B2_AGG_SUM_OF_SQUARES) {
          b2_column_view qv{want_int ? B2_INT64 : B2_FLOAT64, (int32_t)n, want_int ? i2.ptr : x2.ptr, nullable ? vsv.null_mask : nullptr, nullable ? vsv.null_count : 0, 0};
          col = segmented_reduce(qv, off, G + 1, B2_AGG_SUM, rt, B2_NULL_EXCLUDE, nullptr, stream);
          if (!nullable) { col->pending.reset(); col->mask.reset(); col->null_count = 0; }
        } else {
          // two passes (gb_dev2_kernel): the group MEAN, then the sum of the squared deviations from it
          b2_column_view xv{B2_FLOAT64, (int32_t)n, x.ptr, nullable ? vsv.null_mask : nullptr, nullable ? vsv.null_count : 0, 0};
          auto mean = group_mean(xv);
          const bool var_std = kind != B2_AGG_M2;
          const int32_t ddof = kind_ddof(raw);
          const int32_t* vc = valid_counts();  // (evaluated here: launch arguments must not launch kernels themselves)
          dbuf terms(sizeof(double) * n, stream);
          B2_LAUNCH(gb_dev2_kernel, grid_for(n), 256, 0, stream, x.as<double>(), xv.null_mask, gid->data.as<int32_t>(), n, mean->data.as<double>(), vc,
                    var_std ? 1 : 0, ddof, terms.as<double>());
          b2_column_view tv{B2_FLOAT64, (int32_t)n, terms.ptr, nullptr, 0, 0};
          auto s = segmented_reduce(tv, off, G + 1, B2_AGG_SUM, B2_FLOAT64, B2_NULL_EXCLUDE, nullptr, stream);
          if (!var_std) {  // M2 has no null mask: an all-null group sums to 0
            col = std::move(s);
            col->pending.reset();
            col->mask.reset();
            col->null_count = 0;
          } else {
            col = make_column(B2_FLOAT64, G, true, stream);
            mark_pending_valid(*col, stream);
            B2_LAUNCH(gb_var_std_kernel, ggrid, 256, 0, stream, s->data.as<double>(), vc, G, ddof, kind == B2_AGG_STD ? 1 : 0, col->data.as<double>(),
                      col->mask.as<uint32_t>(), col->pending.as<unsigned long long>());
          }
        }
      } else if (kind == AGG_NTH_ELEMENT) {
        dbuf map(sizeof(int32_t) * (size_t)G, stream);
        B2_LAUNCH(gb_nth_map_kernel, ggrid, 256, 0, stream, off, G, kind_param_signed(raw), map.as<int32_t>());
        col = gather_column(vsv, map.as<int32_t>(), G, true, stream);
      } else if (kind == AGG_NUNIQUE) {
        const b2_column& s2c = values_sorted_in_group();
        const b2_column_view s2v = s2c.view();
        dbuf flags(sizeof(int32_t) * n, stream);
        dispatch_width(type_width(v.type_id), [&](auto tag) {
          using T = decltype(tag);
          B2_LAUNCH((gb_distinct_flags_kernel<T>), grid_for(n), 256, 0, stream, static_cast<const T*>(s2v.data), has_nulls(s2v) ? s2v.null_mask : nullptr,
                    gid->data.as<int32_t>(), n, is_float_id(st) ? 1 : 0, flags.as<int32_t>());
        });
        b2_column_view fv{B2_INT32, (int32_t)n, flags.ptr, nullptr, 0, 0};
        col = segmented_reduce(fv, off, G + 1, B2_AGG_SUM, B2_INT32, B2_NULL_EXCLUDE, nullptr, stream);
        col->pending.reset();
        col->mask.reset();
        col->null_count = 0;
      } else {  // MEDIAN
        const b2_column& s2c = values_sorted_in_group();
        const b2_column_view s2v = s2c.view();
        dbuf x(sizeof(double) * n, stream);
        B2_LAUNCH(gb_squares_kernel, grid_for(n), 256, 0, stream, s2v.data, st, n, x.as<double>(), (double*)nullptr, (long long*)nullptr);
        col = make_column(B2_FLOAT64, G, true, stream);
        mark_pending_valid(*col, stream);
        const int32_t* vc = valid_counts();
        B2_LAUNCH(gb_median_kernel, ggrid, 256, 0, stream, x.as<double>(), off, vc, G, col->data.as<double>(), col->mask.as<uint32_t>(),
                  col->pending.as<unsigned long long>());
      }
      res_out->cols.push_back(std::move(col));
    }
  }
}

}  // namespace b2

// ---- C ABI -----------------------------------------------------------------------------------------
extern "C" {

b2_status b2_groupby_create(const b2_table_view* keys, int32_t null_handling, int32_t keys_are_sorted, const uint8_t* column_order,
                            int32_t n_order, const uint8_t* null_precedence, int32_t n_null_prec, b2_groupby** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  auto gb = std::make_unique<b2_groupby>();
  validate_table(keys, gb->keys);
  gb->null_handling   = null_handling;
  gb->keys_are_sorted = keys_are_sorted != 0;
  if (column_order && n_order > 0) gb->order.assign(column_order, column_order + n_order);
  if (null_precedence && n_null_prec > 0) gb->nprec.assign(null_precedence, null_precedence + n_null_prec);
  (void)make_key_cols(gb->keys, true);  // validates the key shape early
  *out = gb.release();
  B2_TRY_END
}
void b2_groupby_destroy(b2_groupby* gb) { delete gb; }

static std::vector<request_view> to_requests(const b2_agg_request* requests, int32_t n)
{
  B2_EXPECTS(n >= 0 && (n == 0 || requests != nullptr), B2_ERR_INVALID_ARGUMENT, "invalid requests");
  std::vector<request_view> out;
  for (int32_t i = 0; i < n; ++i) {
    request_view r;
    r.values = requests[i].values;
    B2_EXPECTS(requests[i].num_kinds >= 0 && (requests[i].num_kinds == 0 || requests[i].kinds), B2_ERR_INVALID_ARGUMENT,
               "invalid aggregation list");
    r.kinds.assign(requests[i].kinds, requests[i].kinds + requests[i].num_kinds);
    out.push_back(std::move(r));
  }
  return out;
}

b2_status b2_groupby_aggregate(b2_groupby* gb, const b2_agg_request* requests, int32_t num_requests, b2_stream stream,
                               b2_table** out_keys, b2_table** out_results)
{
  B2_TRY_BEGIN
  B2_EXPECTS(gb && out_keys && out_results, B2_ERR_INVALID_ARGUMENT, "null argument");
  auto reqs = to_requests(requests, num_requests);
  table_ptr k, r;
  groupby_aggregate(*gb, reqs, static_cast<cudaStream_t>(stream), k, r);
  *out_keys    = k.release();
  *out_results = r.release();
  B2_TRY_END
}

b2_status b2_groupby_scan(b2_groupby* gb, const b2_agg_request* requests, int32_t num_requests, b2_stream stream, b2_table** out_keys,
                          b2_table** out_results)
{
  B2_TRY_BEGIN
  B2_EXPECTS(gb && out_keys && out_results, B2_ERR_INVALID_ARGUMENT, "null argument");
  auto reqs = to_requests(requests, num_requests);
  table_ptr k, r;
  groupby_scan(*gb, reqs, static_cast<cudaStream_t>(stream), k, r);
  *out_keys    = k.release();
  *out_results = r.release();
  B2_TRY_END
}

}  // extern "C"

// radix_join.cu — partitioned ("radix") inner join for large null-free key tables.
//
// Default for cudf::inner_join / left_join / full_join calls whose two sides both have at least 2^24 rows
// (B2_JOIN_RADIX_ROWS=<rows> moves the limit, 0 switches the path off).
//
// Same contract as the hash path it stands in for (cpp/src/join/join.cu:27-110 inner_join over
// cpp/src/join/hash_join/hash_join.cu:32-299): all (probe row, build row) pairs with equal keys, in unspecified
// order (join.hpp:130-136).  Why: the open-addressing table in HBM costs one 128-byte DRAM fetch per build row
// (CAS claim) and per probe row; at 1e9 x 1e9 rows build + count take several times what the ~80 GB of algorithmic
// traffic would.  Here every byte moves in streams:
//   1. both sides: h = mix64(packed key) (a bijection: h equality is key equality), computed on load inside two
//      one-sweep radix passes on the top 16 bits of h (radix_partition_top16_mix; a single 8-byte integer key column
//      is read in place) -> h and the original row ids grouped into 65536 partitions; bounds by binary search.
//   2. one CTA per partition: the build rows' h go to shared memory (16384 x 8 B) with an open-addressing table of
//      16-bit local row numbers (32768 slots, load factor <= 0.5, slot = bits 33..47 of h); the partition's probe
//      rows stream through it.  Larger partitions (skew, duplicates, > ~1e9 rows) are handled in chunks of 16384
//      build rows, re-streaming the probe rows per chunk.
//   3. ONE walk writes the pairs: per (work item, build chunk) count -> one global reservation -> revisit the matching
//      rows (rj_join_kernel).  A work item is (partition, piece of at most 65536 probe rows), so that a probe-side hot key
//      is spread over many CTAs (each re-builds the table).  The output buffers are sized by a guess and the walk is
//      repeated with the exact size when the guess was too small.
#include "common.cuh"
#include "device_utils.cuh"
#include "key_pack.cuh"

#include <algorithm>
#include <climits>
#include <cstdlib>

namespace b2 {
namespace {

constexpr int RJ_PARTS   = 1 << 16;
constexpr int RJ_THREADS = 1024;
constexpr int RJ_CAP     = 16384;  // build rows per shared-memory table (local row numbers fit 16 bits, 0xFFFF = empty)
constexpr int RJ_SLOTS   = 32768;
constexpr size_t RJ_SMEM = (size_t)RJ_CAP * sizeof(uint64_t) + (size_t)RJ_SLOTS * sizeof(uint16_t);
constexpr int RJ_PIECE   = 65536;  // probe rows per work item

// packed (normalised) key per row; the mixing happens inside the partition passes (radix_partition_top16_mix)
__global__ void __launch_bounds__(256) rj_pack_kernel(key_cols kc, int64_t n, uint64_t* __restrict__ packed)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint64_t key;
    uint32_t nb;
    pack_row(kc, r, key, nb);
    packed[r] = key;
  }
}

// off[p] = first row whose 16-bit prefix is >= p (p in [0, 65536]); rows are grouped by prefix in ascending order
__global__ void __launch_bounds__(256) rj_bounds_kernel(const uint64_t* __restrict__ h, int64_t n, int32_t* __restrict__ off)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > RJ_PARTS) return;
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    if ((h[mid] >> 48) < (uint64_t)p) lo = mid + 1;
    else hi = mid;
  }
  off[p] = (int32_t)lo;
}

// pieces[p] = number of work items of partition p (0 when either side is empty there; LEFT joins also visit probe rows
// whose partition has no build rows); pieces[RJ_PARTS] = 0
__global__ void __launch_bounds__(256) rj_pieces_kernel(const int32_t* __restrict__ boff, const int32_t* __restrict__ poff, bool left,
                                                        int32_t* __restrict__ pieces, int piece)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > RJ_PARTS) return;
  int32_t v = 0;
  if (p < RJ_PARTS) {
    const int64_t nb = (int64_t)boff[p + 1] - boff[p], np = (int64_t)poff[p + 1] - poff[p];
    if (np > 0 && (nb > 0 || left)) v = (int32_t)((np + piece - 1) / piece);
  }
  pieces[p] = v;
}

// item_part[i] = partition of work item i (items of partition p are item_first[p] .. item_first[p + 1] - 1): one load in the join
// kernel instead of a 17-step binary search by one thread while 1023 wait (33 % of the kernel's stall samples at 2^27 rows)
__global__ void __launch_bounds__(256) rj_item_part_kernel(const int32_t* __restrict__ item_first, int32_t* __restrict__ item_part)
{
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= RJ_PARTS) return;
  for (int i = item_first[p]; i < item_first[p + 1]; ++i) item_part[i] = p;
}

__device__ __forceinline__ uint32_t rj_slot(uint64_t h) { return (uint32_t)(h >> 33) & (uint32_t)(RJ_SLOTS - 1); }

// One CTA joins work item blockIdx.x = (partition, probe piece); item_first[p] is the first item of partition p
// (exclusive scan of rj_pieces_kernel's output, item_first[RJ_PARTS] = number of items).
// ONE walk produces the pairs: per (item, build chunk) the CTA first probes its rows counting matches (probe keys are
// fetched RJ_BATCH at a time per thread, so that their global-memory latency overlaps), reserves the output range of the
// whole chunk with one atomicAdd on the global cursor, and then revisits only the rows that matched to write their pairs —
// the structure of the reference's partitioned retrieve (cpp/src/join/hash_join/partitioned_retrieve_kernels.cuh:57-206:
// matches staged per block, one reservation per flush), with the table in shared memory. Pairs beyond `capacity` are counted
// but not written: the host reruns with the exact size (the cursor's final value) when its guess was too small.
// LEFT: a probe row without any match (over all build chunks) yields one pair (row, JoinNoMatch); a thread owns the same
// <= 64 probe rows in every chunk round, so one 64-bit register remembers which of them have matched.
constexpr int RJ_BATCH = 8;

__device__ __forceinline__ unsigned long long rj_block_reserve(unsigned long long mine, unsigned long long* cursor, unsigned long long* s_wsum,
                                                               unsigned long long* s_base)
{
  // exclusive scan of `mine` over the CTA + one global reservation; returns this thread's first output position
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long nb = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += nb;
  }
  if (lane == 31) s_wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    unsigned long long w = lane < RJ_THREADS / 32 ? s_wsum[lane] : 0ull;
    unsigned long long winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long nb = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += nb;
    }
    if (lane < RJ_THREADS / 32) s_wsum[lane] = winc - w;  // exclusive offset of each warp
    if (lane == 31) *s_base = winc ? atomicAdd(cursor, winc) : 0ull;
  }
  __syncthreads();
  const unsigned long long pos = *s_base + s_wsum[warp] + (inc - mine);
  __syncthreads();  // s_wsum / s_base are reused by the next reservation
  return pos;
}

template <bool LEFT = false>
__global__ void __launch_bounds__(RJ_THREADS, 1)
rj_join_kernel(const uint64_t* __restrict__ bh, const int32_t* __restrict__ bid, const int32_t* __restrict__ boff,
               const uint64_t* __restrict__ ph, const int32_t* __restrict__ pid, const int32_t* __restrict__ poff,
               const int32_t* __restrict__ item_first, const int32_t* __restrict__ item_part, unsigned long long* __restrict__ cursor,
               unsigned long long capacity, int32_t* __restrict__ out_probe, int32_t* __restrict__ out_build)
{
  B2_DYNAMIC_SMEM(rj_smem);
  uint64_t* bk  = reinterpret_cast<uint64_t*>(rj_smem);
  uint32_t* tab = reinterpret_cast<uint32_t*>(rj_smem + (size_t)RJ_CAP * sizeof(uint64_t));  // RJ_SLOTS / 2 words
  const uint16_t* tab16 = reinterpret_cast<const uint16_t*>(tab);
  __shared__ unsigned long long s_wsum[RJ_THREADS / 32];
  __shared__ unsigned long long s_base;

  const int item = blockIdx.x;
  const int tid  = threadIdx.x;
  if (item >= item_first[RJ_PARTS]) return;  // the grid is sized for the worst case; uniform over the CTA
  const int part = item_part[item];
  const int b0 = boff[part], b1 = boff[part + 1];
  const int64_t p0 = (int64_t)poff[part] + (int64_t)(item - item_first[part]) * RJ_PIECE;
  const int64_t p1 = min(p0 + RJ_PIECE, (int64_t)poff[part + 1]);
  constexpr int ROUNDS = RJ_PIECE / RJ_THREADS;  // probe rows per thread
  static_assert(ROUNDS <= 64 && ROUNDS % RJ_BATCH == 0, "one bit per probe row of a thread; whole batches");
  const int my_rounds = (int)((p1 - p0 - tid + RJ_THREADS - 1) / RJ_THREADS);  // rows p0 + tid + k * RJ_THREADS, k < my_rounds (may be <= 0)
  unsigned long long matched = 0;
  for (int64_t c0 = b0; c0 < b1; c0 += RJ_CAP) {  // 64-bit: row numbers go up to 2^31 - 1
    const int cn = (int)min((int64_t)RJ_CAP, (int64_t)b1 - c0);
    __syncthreads();  // the previous chunk's probes are done before the table is reset
    for (int i = tid; i < RJ_SLOTS / 2; i += RJ_THREADS) tab[i] = 0xFFFFFFFFu;
    for (int j = tid; j < cn; j += RJ_THREADS) bk[j] = ld_stream(bh + c0 + j);
    __syncthreads();
    // insert: claim a 16-bit slot with a 32-bit CAS on the word that holds it
    for (int j = tid; j < cn; j += RJ_THREADS) {
      uint32_t s = rj_slot(bk[j]);
      while (true) {
        uint32_t* w = &tab[s >> 1];
        const int sh = (int)(s & 1u) * 16;
        const uint32_t old = *reinterpret_cast<volatile uint32_t*>(w);
        if (((old >> sh) & 0xFFFFu) == 0xFFFFu) {
          const uint32_t neu = (old & ~(0xFFFFu << sh)) | ((uint32_t)j << sh);
          if (atomicCAS(w, old, neu) == old) break;
          // the word changed under us (either half): look at the same slot again
        } else {
          s = (s + 1) & (uint32_t)(RJ_SLOTS - 1);
        }
      }
    }
    __syncthreads();
    // ---- walk 1: count this chunk's matches, remember which of my rows matched ----
    unsigned long long hit = 0, local = 0;
    for (int kb = 0; kb < ROUNDS; kb += RJ_BATCH) {
      if (kb >= my_rounds) break;
      uint64_t h[RJ_BATCH];
#pragma unroll
      for (int u = 0; u < RJ_BATCH; ++u) h[u] = (kb + u < my_rounds) ? ld_stream(ph + p0 + tid + (int64_t)(kb + u) * RJ_THREADS) : 0ull;
#pragma unroll
      for (int u = 0; u < RJ_BATCH; ++u) {
        if (kb + u >= my_rounds) break;
        uint32_t s = rj_slot(h[u]);
        while (true) {
          const uint32_t e = tab16[s];
          if (e == 0xFFFFu) break;
          if (bk[e] == h[u]) {
            ++local;
            hit |= 1ull << (kb + u);
          }
          s = (s + 1) & (uint32_t)(RJ_SLOTS - 1);
        }
      }
    }
    if (LEFT) matched |= hit;
    // ---- one reservation for the chunk, then walk 2 over the rows that matched ----
    unsigned long long pos = rj_block_reserve(local, cursor, s_wsum, &s_base);
    while (hit) {
      const int k = (uint32_t)hit ? __ffs((int)(uint32_t)hit) - 1 : 32 + __ffs((int)(uint32_t)(hit >> 32)) - 1;
      hit &= hit - 1;
      const int64_t i = p0 + tid + (int64_t)k * RJ_THREADS;
      const uint64_t h = ph[i];
      const int32_t prow = pid[i];
      uint32_t s = rj_slot(h);
      while (true) {
        const uint32_t e = tab16[s];
        if (e == 0xFFFFu) break;
        if (bk[e] == h) {
          if (pos < capacity) {
            out_probe[pos] = prow;
            out_build[pos] = bid[c0 + e];
          }
          ++pos;
        }
        s = (s + 1) & (uint32_t)(RJ_SLOTS - 1);
      }
    }
  }
  if (LEFT) {
    unsigned long long un = 0;  // my rows that never matched
    for (int k = 0; k < my_rounds; ++k) un += ((matched >> k) & 1ull) ? 0ull : 1ull;
    unsigned long long pos = rj_block_reserve(un, cursor, s_wsum, &s_base);
    for (int k = 0; k < my_rounds; ++k) {
      if ((matched >> k) & 1ull) continue;
      if (pos < capacity) {
        out_probe[pos] = pid[p0 + tid + (int64_t)k * RJ_THREADS];
        out_build[pos] = B2_JOIN_NO_MATCH;
      }
      ++pos;
    }
  }
}

bool any_nulls(const std::vector<b2_column_view>& cols)
{
  for (auto& c : cols)
    if (has_nulls(c)) return true;
  return false;
}

struct rj_side {
  dbuf h, ids, off;
};

void rj_partition(const std::vector<b2_column_view>& cols, cudaStream_t stream, rj_side& s)
{
  const int64_t n = cols[0].size;
  const key_cols kc = make_key_cols(cols);
  s.h   = dbuf(sizeof(uint64_t) * n, stream);
  s.ids = dbuf(sizeof(int32_t) * n, stream);
  s.off = dbuf(sizeof(int32_t) * (RJ_PARTS + 1), stream);
  prof_scope ps("rjoin_partition", stream);
  // one 8-byte integer-like key column IS its packed form: the partition passes read it in place
  const bool in_place = cols.size() == 1 && type_width(cols[0].type_id) == 8 && !is_float_id(cols[0].type_id);
  dbuf packed;
  const uint64_t* src = static_cast<const uint64_t*>(cols[0].data) + cols[0].offset;
  if (!in_place) {
    packed = dbuf(sizeof(uint64_t) * n, stream);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, num_sms() * 16));
    B2_LAUNCH(rj_pack_kernel, grid, 256, 0, stream, kc, n, packed.as<uint64_t>());
    src = packed.as<uint64_t>();
  }
  radix_partition_top16_mix(src, n, s.h.as<uint64_t>(), s.ids.as<int32_t>(), stream);
  B2_LAUNCH(rj_bounds_kernel, (RJ_PARTS + 1 + 255) / 256, 256, 0, stream, s.h.as<uint64_t>(), n, s.off.as<int32_t>());
}

}  // namespace

// The partitioned join takes over when BOTH sides are large: a build side of 2^24 rows already needs a 512 MB table (beyond
// the L2), where every build / probe touch of the open-addressing path is a random DRAM fetch. Smaller build sides keep
// the hash table (L2 resident). B2_JOIN_RADIX_ROWS=<rows> moves the
// limit (0 = never).
bool radix_join_applicable(const std::vector<b2_column_view>& a, const std::vector<b2_column_view>& b)
{
  if (a.empty() || b.empty()) return false;
  const char* e = std::getenv("B2_JOIN_RADIX_ROWS");
  int64_t thr = int64_t(1) << 24;
  if (e) {
    thr = std::atoll(e);
    if (thr <= 0) return false;
  }
  return a[0].size >= thr && b[0].size >= thr && !any_nulls(a) && !any_nulls(b) && !keys_are_wide(a);
}

// pairs (probe row, build row) with equal keys; both tables null-free and non-empty. left: probe rows without a match
// are kept with JoinNoMatch as their build row (left join; the caller appends the unmatched build rows for a full join).
void radix_join(const std::vector<b2_column_view>& build, const std::vector<b2_column_view>& probe, bool left, cudaStream_t stream,
                column_ptr& out_probe, column_ptr& out_build)
{
  static std::atomic<uint64_t> attr_done{0};
  once_per_device(attr_done, [] {
    B2_CUDA_TRY(cudaFuncSetAttribute(rj_join_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RJ_SMEM));
    B2_CUDA_TRY(cudaFuncSetAttribute(rj_join_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RJ_SMEM));
  });
  rj_side bs, ps;
  rj_partition(build, stream, bs);
  rj_partition(probe, stream, ps);

  // work items: (partition, piece of <= RJ_PIECE probe rows); at most RJ_PARTS + n_probe / RJ_PIECE of them
  const int64_t n_probe = probe[0].size;
  const int32_t max_items = (int32_t)(RJ_PARTS + n_probe / RJ_PIECE + 1);
  dbuf pieces(sizeof(int32_t) * (RJ_PARTS + 1), stream);
  B2_LAUNCH(rj_pieces_kernel, (RJ_PARTS + 1 + 255) / 256, 256, 0, stream, bs.off.as<int32_t>(), ps.off.as<int32_t>(), left, pieces.as<int32_t>(),
            RJ_PIECE);
  b2_column_view pv{B2_INT32, (int32_t)(RJ_PARTS + 1), pieces.ptr, nullptr, 0, 0};
  auto item_first = scan(pv, B2_AGG_SUM, B2_SCAN_EXCLUSIVE, B2_NULL_EXCLUDE, stream);

  dbuf item_part(sizeof(int32_t) * (size_t)max_items, stream);
  B2_LAUNCH(rj_item_part_kernel, RJ_PARTS / 256, 256, 0, stream, item_first->data.as<int32_t>(), item_part.as<int32_t>());

  // The output size is only known after the walk (the reference walks twice: size_impl.cuh then retrieve_impl.cuh). Guess
  // one pair per probe row (left joins: a quarter more), write what fits, read the true size back, and repeat with the
  // exact size in the rare case the guess was too small.
  dbuf tot(sizeof(unsigned long long), stream);
  unsigned long long capacity = std::min<unsigned long long>((unsigned long long)INT32_MAX, (unsigned long long)n_probe + (left ? (unsigned long long)n_probe / 4 : 0ull));
  if (const char* e = std::getenv("B2_JOIN_RADIX_CAPACITY")) capacity = std::max<long long>(1, std::atoll(e));  // test hook: force the rerun
  for (int attempt = 0;; ++attempt) {
    auto op = make_column(B2_INT32, (int32_t)capacity, false, stream);
    auto ob = make_column(B2_INT32, (int32_t)capacity, false, stream);
    B2_CUDA_TRY(cudaMemsetAsync(tot.ptr, 0, sizeof(unsigned long long), stream));
    {
      prof_scope sc("rjoin_join", stream);
#define B2_RJ(L) B2_LAUNCH((rj_join_kernel<L>), max_items, RJ_THREADS, RJ_SMEM, stream, bs.h.as<uint64_t>(), bs.ids.as<int32_t>(),      \
                           bs.off.as<int32_t>(), ps.h.as<uint64_t>(), ps.ids.as<int32_t>(), ps.off.as<int32_t>(),                        \
                           item_first->data.as<int32_t>(), item_part.as<int32_t>(), tot.as<unsigned long long>(), capacity, op->data.as<int32_t>(),   \
                           ob->data.as<int32_t>())
      if (left) B2_RJ(true);
      else B2_RJ(false);
#undef B2_RJ
    }
    unsigned long long m = 0;
    B2_CUDA_TRY(cudaMemcpyAsync(&m, tot.ptr, sizeof(m), cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));  // the reference syncs for the output size too (size_impl.cuh:52-61)
    B2_EXPECTS(m <= (unsigned long long)INT32_MAX, B2_ERR_LOGIC /* std::overflow_error in libcudf */,
               "join output exceeds size_type (use hash_join::*_join_size and partition the probe side)");
    if (m > capacity) {
      B2_EXPECTS(attempt == 0, B2_ERR_LOGIC, "radix join: output size changed between walks");
      capacity = m;
      continue;
    }
    if (m == capacity) {
      out_probe = std::move(op);
      out_build = std::move(ob);
    } else {  // hand back right-sized columns (the guess may be ten times the result)
      out_probe = make_column(B2_INT32, (int32_t)m, false, stream);
      out_build = make_column(B2_INT32, (int32_t)m, false, stream);
      if (m) {
        B2_CUDA_TRY(cudaMemcpyAsync(out_probe->data.ptr, op->data.ptr, sizeof(int32_t) * m, cudaMemcpyDeviceToDevice, stream));
        B2_CUDA_TRY(cudaMemcpyAsync(out_build->data.ptr, ob->data.ptr, sizeof(int32_t) * m, cudaMemcpyDeviceToDevice, stream));
      }
    }
    return;
  }
}

}  // namespace b2

// compact.cuh — the stable compaction shared by stream compaction (stream_compaction.cu) and the semi / anti join
// (filtered_join.cu): compact_kernel evaluates a row predicate inline, ranks the kept rows of a warp with __ballot_sync /
// __popc, takes the tile base from a single-pass decoupled look-back (the 16-byte records of device_utils.cuh, as
// scan_kernel) and writes the kept row ids, INT32 and in input order. One host read-back per call, for the kept row count.
#pragma once
#include "common.cuh"
#include "device_utils.cuh"

namespace b2 {
namespace {

constexpr int CP_THREADS = 256;
constexpr int CP_K       = 32;  // warp steps of 32 rows per tile: 8192 rows per tile
constexpr int CP_NW      = CP_THREADS / 32;
constexpr int64_t CP_TILE = (int64_t)CP_THREADS * CP_K;

// workspace: ntiles look-back records, then {ticket (u32), pad, total kept rows (u64)} in one more 16-byte record
template <typename P>
__global__ void __launch_bounds__(CP_THREADS) compact_kernel(P pred, int64_t n, int32_t* __restrict__ out, scan_state st,
                                                             int64_t ntiles, unsigned long long* total)
{
  __shared__ uint32_t s_wtot[CP_NW];
  __shared__ unsigned long long s_prefix;
  __shared__ uint32_t s_tile;
  if (threadIdx.x == 0) s_tile = atomicAdd(st.ticket, 1u);  // tiles start in ticket order: the look-back cannot wait on a
  __syncthreads();                                           // tile that has not been scheduled
  const int64_t tile = s_tile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wbase = tile * CP_TILE + (int64_t)warp * 32 * CP_K;

  uint32_t ballot[CP_K];
  uint32_t cnt = 0;
#pragma unroll
  for (int k = 0; k < CP_K; ++k) {
    const int64_t r = wbase + k * 32 + lane;
    ballot[k] = __ballot_sync(0xffffffffu, r < n && pred(r));
    cnt += __popc(ballot[k]);
  }
  if (lane == 0) s_wtot[warp] = cnt;
  __syncthreads();
  if (warp == 0) {
    unsigned long long block_tot = 0;
#pragma unroll
    for (int w = 0; w < CP_NW; ++w) block_tot += s_wtot[w];
    unsigned long long excl = 0;
    if (tile == 0) {
      if (lane == 0) publish_rec<unsigned long long>(st.rec, 2u, block_tot);
    } else {
      if (lane == 0) publish_rec<unsigned long long>(st.rec + tile, 1u, block_tot);
      int64_t base = tile - 1;  // nearest predecessor not folded yet
      while (true) {
        // lane l reads the record at distance l from `base`; tiles before the first act as an inclusive zero
        const int64_t idx = base - lane;
        unsigned long long v = 0;
        const uint32_t f = idx >= 0 ? read_rec<unsigned long long>(st.rec + idx, v) : 2u;
        const unsigned incl_mask = __ballot_sync(0xffffffffu, f == 2u);
        const unsigned wait_mask = __ballot_sync(0xffffffffu, f == 0u);
        const int first_incl = incl_mask ? (__ffs(incl_mask) - 1) : 32;
        const int first_wait = wait_mask ? (__ffs(wait_mask) - 1) : 32;
        if (first_wait < first_incl) continue;  // a needed record is not published yet: poll again (volatile loads)
        excl += warp_sum(lane <= first_incl ? v : 0ull);
        if (incl_mask) break;
        base -= 32;
      }
      if (lane == 0) publish_rec<unsigned long long>(st.rec + tile, 2u, excl + block_tot);
    }
    if (lane == 0) {
      s_prefix = excl;
      if (tile == ntiles - 1) *total = excl + block_tot;
    }
  }
  __syncthreads();
  unsigned long long pos = s_prefix;
  for (int w = 0; w < warp; ++w) pos += s_wtot[w];
  const unsigned lt = lanemask_lt();
#pragma unroll
  for (int k = 0; k < CP_K; ++k) {
    if ((ballot[k] >> lane) & 1u) out[pos + __popc(ballot[k] & lt)] = (int32_t)(wbase + k * 32 + lane);
    pos += __popc(ballot[k]);
  }
}

// kept row ids of rows [0, n) in order; returns their count (one device -> host read-back)
template <typename P>
int32_t compact(const P& pred, int64_t n, dbuf& map, cudaStream_t stream)
{
  map = dbuf(sizeof(int32_t) * (size_t)n, stream);
  if (n == 0) return 0;
  const int64_t ntiles = (n + CP_TILE - 1) / CP_TILE;
  dbuf work(sizeof(uint4) * (size_t)(ntiles + 1), stream);
  B2_CUDA_TRY(cudaMemsetAsync(work.ptr, 0, work.bytes, stream));
  scan_state st;
  st.rec    = work.as<uint4>();
  st.ticket = reinterpret_cast<uint32_t*>(work.as<uint4>() + ntiles);
  auto* total = reinterpret_cast<unsigned long long*>(work.as<uint4>() + ntiles) + 1;
  {
    prof_scope ps("compact", stream);
    B2_LAUNCH((compact_kernel<P>), (unsigned)ntiles, CP_THREADS, 0, stream, pred, n, map.as<int32_t>(), st, ntiles, total);
  }
  unsigned long long h = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&h, total, sizeof(h), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  return (int32_t)h;
}

}  // namespace
}  // namespace b2

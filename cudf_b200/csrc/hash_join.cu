// hash_join.cu — hash join (inner / left / full) over an open-addressing table in HBM (no cuco).
//
// Replaces cpp/src/join/join.cu:27-124 (free functions, build on the smaller side for inner),
// cpp/src/join/hash_join/hash_join.cu:32-299 (cudf::hash_join: ctor validation, build, probe entry
// points, *_join_size), size_impl.cuh:26-62 (count pass), retrieve_impl.cuh:28-196 (retrieve pass),
// join_utils.cu (full-join complement) and the cuco::static_multiset they sit on.
//
// Table: S = pow2 >= rows / load_factor slots of 16 bytes {uint64 key, int32 row, uint32 nullbits};
// row == -1 marks an empty slot (the table is initialised with 0xFF bytes). Keys of all join columns
// are packed into 64 bits (sum of widths <= 8 bytes), floats normalised so that bit equality is the
// reference's row equality (-0 == +0, NaN == NaN: primitive_row_operators.cuh:121-143,
// common_utils.cuh:214-220); `nullbits` has bit c set when column c is null (value bits zeroed) so
// null == null under null_equality::EQUAL, and rows with nulls are skipped under UNEQUAL
// (hash_join.cu:77-84).  It is a multiset: every build row owns one slot (claimed with a 32-bit CAS
// on the row field, then the key is written; nobody compares keys during the build).
// Probe = count pass (per-row match counts + 64-bit total) -> exclusive scan -> retrieve pass that
// only re-walks rows that have matches; output pairs come out ordered by left row (a legal choice:
// the reference leaves the order unspecified, join.hpp:130-136).
#include "common.cuh"
#include "device_utils.cuh"
#include "key_pack.cuh"

#include <algorithm>
#include <cmath>

namespace b2 {
namespace {

__global__ void __launch_bounds__(256) build_kernel(key_cols kc, int64_t n, bool skip_nulls, slot_t* __restrict__ table,
                                                    uint32_t mask)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint64_t key;
    uint32_t nb;
    pack_row(kc, r, key, nb);
    if (skip_nulls && nb) continue;
    uint32_t i = slot_hash(key, nb, mask);
    while (true) {
      int old = atomicCAS(&table[i].row, -1, (int32_t)r);
      if (old == -1) {
        slot_t s{key, (int32_t)r, nb};
        int4 v;
        memcpy(&v, &s, 16);
        *reinterpret_cast<int4*>(&table[i]) = v;
        break;
      }
      i = (i + 1) & mask;
    }
  }
}

// counts[r] = number of build rows equal to probe row r; total += output rows
template <bool LEFT>
__global__ void __launch_bounds__(256) count_kernel(key_cols kc, int64_t n, bool skip_nulls, bool table_has_null_rows,
                                                    const slot_t* __restrict__ table, uint32_t mask, int32_t* __restrict__ counts,
                                                    unsigned long long* __restrict__ total)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long local = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint64_t key;
    uint32_t nb;
    pack_row(kc, r, key, nb);
    uint32_t c = 0;
    if (!(nb && (skip_nulls || !table_has_null_rows)) && table != nullptr) {
      uint32_t i = slot_hash(key, nb, mask);
      while (true) {
        const slot_t s = load_slot(&table[i]);
        if (s.row == -1) break;
        c += (s.key == key && s.nullbits == nb) ? 1u : 0u;
        i = (i + 1) & mask;
      }
    }
    // counts hold the TRUE match count (0 = no match) so that the retrieve pass can tell the
    // unmatched rows of a left join; the output size counts those rows once.
    if (counts) counts[r] = (int32_t)min(c, 0x7fffffffu);
    local += (LEFT && c == 0) ? 1ull : (unsigned long long)c;
  }
  local = warp_sum(local);
  if (lane_id() == 0 && local) atomicAdd(total, local);
}

// out offsets for LEFT joins: max(count,1) per row -> done by transforming counts in place
__global__ void left_adjust_kernel(const int32_t* __restrict__ counts, int64_t n, int32_t* __restrict__ adj)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) adj[r] = max(counts[r], 1);
}

template <bool LEFT>
__global__ void __launch_bounds__(256) retrieve_kernel(key_cols kc, int64_t n, const slot_t* __restrict__ table, uint32_t mask,
                                                       const int32_t* __restrict__ counts, const int32_t* __restrict__ offsets,
                                                       int32_t* __restrict__ out_left, int32_t* __restrict__ out_right)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    const int32_t c = counts[r];
    if (c == 0 && !LEFT) continue;
    uint64_t key;
    uint32_t nb;
    pack_row(kc, r, key, nb);
    int32_t o = offsets[r];
    if (c == 0) {
      out_left[o]  = (int32_t)r;
      out_right[o] = B2_JOIN_NO_MATCH;
      continue;
    }
    const int32_t end = o + c;
    uint32_t i = slot_hash(key, nb, mask);
    while (o < end) {
      const slot_t s = load_slot(&table[i]);
      if (s.row == -1) break;
      if (s.key == key && s.nullbits == nb) {
        out_left[o]  = (int32_t)r;
        out_right[o] = s.row;
        ++o;
      }
      i = (i + 1) & mask;
    }
  }
}

// ---- wide keys (sum of key widths > 8 bytes) ----------------------------------------------------------
// Same table and the same three passes, but the slot holds a 64-bit hash of the row (hash_row_wide) and a hash hit
// is confirmed by comparing the key columns of the probe row with those of the slot's build row (rows_equal_wide).
__global__ void __launch_bounds__(256) build_wide_kernel(key_cols kc, int64_t n, bool skip_nulls, slot_t* __restrict__ table,
                                                         uint32_t mask)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint64_t h;
    uint32_t nb;
    hash_row_wide(kc, r, h, nb);
    if (skip_nulls && nb) continue;
    uint32_t i = slot_hash(h, nb, mask);
    while (true) {
      int old = atomicCAS(&table[i].row, -1, (int32_t)r);
      if (old == -1) {
        slot_t s{h, (int32_t)r, nb};
        int4 v;
        memcpy(&v, &s, 16);
        *reinterpret_cast<int4*>(&table[i]) = v;
        break;
      }
      i = (i + 1) & mask;
    }
  }
}

template <bool LEFT>
__global__ void __launch_bounds__(256) count_wide_kernel(key_cols pk, key_cols bk, int64_t n, bool skip_nulls, bool table_has_null_rows,
                                                         const slot_t* __restrict__ table, uint32_t mask, int32_t* __restrict__ counts,
                                                         unsigned long long* __restrict__ total)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long local = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint64_t h;
    uint32_t nb;
    hash_row_wide(pk, r, h, nb);
    uint32_t c = 0;
    if (!(nb && (skip_nulls || !table_has_null_rows)) && table != nullptr) {
      uint32_t i = slot_hash(h, nb, mask);
      while (true) {
        const slot_t s = load_slot(&table[i]);
        if (s.row == -1) break;
        if (s.key == h && s.nullbits == nb && rows_equal_wide(pk, r, bk, s.row)) ++c;
        i = (i + 1) & mask;
      }
    }
    if (counts) counts[r] = (int32_t)min(c, 0x7fffffffu);
    local += (LEFT && c == 0) ? 1ull : (unsigned long long)c;
  }
  local = warp_sum(local);
  if (lane_id() == 0 && local) atomicAdd(total, local);
}

template <bool LEFT>
__global__ void __launch_bounds__(256) retrieve_wide_kernel(key_cols pk, key_cols bk, int64_t n, const slot_t* __restrict__ table,
                                                            uint32_t mask, const int32_t* __restrict__ counts,
                                                            const int32_t* __restrict__ offsets, int32_t* __restrict__ out_left,
                                                            int32_t* __restrict__ out_right)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    const int32_t c = counts[r];
    if (c == 0 && !LEFT) continue;
    int32_t o = offsets[r];
    if (c == 0) {
      out_left[o]  = (int32_t)r;
      out_right[o] = B2_JOIN_NO_MATCH;
      continue;
    }
    uint64_t h;
    uint32_t nb;
    hash_row_wide(pk, r, h, nb);
    const int32_t end = o + c;
    uint32_t i = slot_hash(h, nb, mask);
    while (o < end) {
      const slot_t s = load_slot(&table[i]);
      if (s.row == -1) break;
      if (s.key == h && s.nullbits == nb && rows_equal_wide(pk, r, bk, s.row)) {
        out_left[o]  = (int32_t)r;
        out_right[o] = s.row;
        ++o;
      }
      i = (i + 1) & mask;
    }
  }
}

// ---- partitioned probe (hash_join.hpp:331-411): retrieve rows [row_begin, row_begin + n) of the probe table from the
// match counts of a join_match_context. For LEFT the counts are >= 1 (an unmatched row owns one output slot), so an
// unmatched row is recognised by walking its chain without a hit. Offsets are local to the partition.
template <bool LEFT, bool WIDE>
__global__ void __launch_bounds__(256) retrieve_part_kernel(key_cols pk, key_cols bk, int64_t row_begin, int64_t n,
                                                            const slot_t* __restrict__ table, uint32_t mask,
                                                            const int32_t* __restrict__ counts, const int32_t* __restrict__ offsets,
                                                            int32_t* __restrict__ out_left, int32_t* __restrict__ out_right)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t r = row_begin + i;
    const int32_t c = counts[r];
    if (c == 0) continue;  // inner context: no match
    uint64_t key;
    uint32_t nb;
    if constexpr (WIDE) hash_row_wide(pk, r, key, nb);
    else pack_row(pk, r, key, nb);
    int32_t o = offsets[i];
    const int32_t end = o + c;
    bool any = false;
    if (table != nullptr) {
      uint32_t s0 = slot_hash(key, nb, mask);
      while (o < end) {
        const slot_t s = load_slot(&table[s0]);
        if (s.row == -1) break;
        bool hit = s.key == key && s.nullbits == nb;
        if constexpr (WIDE) hit = hit && rows_equal_wide(pk, r, bk, s.row);
        if (hit) {
          out_left[o]  = (int32_t)r;
          out_right[o] = s.row;
          ++o;
          any = true;
        }
        s0 = (s0 + 1) & mask;
      }
    }
    if (LEFT && !any) {
      out_left[o]  = (int32_t)r;
      out_right[o] = B2_JOIN_NO_MATCH;
    }
  }
}

__global__ void fill_i32_kernel(int32_t* p, int64_t n, int32_t v)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

// ---- full join complement (join_utils.cu finalize_full_join): build rows that never matched ----
__global__ void mark_kernel(const int32_t* __restrict__ right_idx, int64_t m, uint32_t* __restrict__ bitmap)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
    const int32_t r = right_idx[i];
    if (r >= 0) atomicOr(&bitmap[r >> 5], 1u << (r & 31));
  }
}
__global__ void unmatched_count_kernel(const uint32_t* __restrict__ bitmap, int64_t nrows, int32_t* __restrict__ word_counts)
{
  const int64_t nwords = (nrows + 31) / 32;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += stride) {
    uint32_t b = ~bitmap[w];
    int64_t rem = nrows - w * 32;
    if (rem < 32) b &= (1u << rem) - 1u;
    word_counts[w] = __popc(b);
  }
}
__global__ void unmatched_write_kernel(const uint32_t* __restrict__ bitmap, int64_t nrows, const int32_t* __restrict__ word_offsets,
                                       int64_t base, int32_t* __restrict__ out_left, int32_t* __restrict__ out_right)
{
  const int64_t nwords = (nrows + 31) / 32;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += stride) {
    uint32_t b = ~bitmap[w];
    int64_t rem = nrows - w * 32;
    if (rem < 32) b &= (1u << rem) - 1u;
    int64_t o = base + word_offsets[w];
    while (b) {
      int bit = __ffs(b) - 1;
      b &= b - 1;
      out_left[o]  = B2_JOIN_NO_MATCH;
      out_right[o] = (int32_t)(w * 32 + bit);
      ++o;
    }
  }
}

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, num_sms() * 16)); }

}  // namespace
}  // namespace b2

using namespace b2;

struct b2_hash_join {
  std::vector<int32_t> build_types;
  int32_t build_rows = 0;
  bool has_nulls     = false;  // nullable_join
  int32_t compare_nulls = B2_NULLS_EQUAL;
  uint32_t mask      = 0;
  bool table_has_null_rows = false;
  bool wide = false;           // keys wider than 8 bytes: hash in the slot + column comparison (build_cols must stay alive,
                               // like the reference's build table: hash_join.hpp "must outlive this object")
  std::vector<b2_column_view> build_cols;
  dbuf table;                  // empty when the build table has no rows
};

namespace b2 {

enum join_kind { JOIN_INNER = 0, JOIN_LEFT = 1, JOIN_FULL = 2 };

static bool table_has_nulls(const std::vector<b2_column_view>& cols)
{
  for (auto& c : cols)
    if (has_nulls(c)) return true;
  return false;
}

// cudf::hash_join ctor — hash_join.cu:112-148,189-198
b2_hash_join* hash_join_create(const std::vector<b2_column_view>& build, int has_nulls_arg, int compare_nulls,
                               double load_factor, cudaStream_t stream)
{
  B2_EXPECTS(!build.empty(), B2_ERR_INVALID_ARGUMENT, "Hash join build table is empty");
  B2_EXPECTS(load_factor > 0 && load_factor <= 1, B2_ERR_INVALID_ARGUMENT, "Invalid load factor: must be greater than 0 and at most 1.");
  auto hj = std::make_unique<b2_hash_join>();
  for (auto& c : build) hj->build_types.push_back(c.type_id);
  hj->build_rows    = build[0].size;
  hj->has_nulls     = has_nulls_arg < 0 ? true : has_nulls_arg != 0;  // ctor #1 = nullable_join::YES (hash_join.hpp)
  hj->compare_nulls = compare_nulls;
  hj->wide       = keys_are_wide(build);
  hj->build_cols = build;
  key_cols kc = make_key_cols(build, true);
  if (hj->build_rows == 0) return hj.release();
  const double want = std::ceil((double)hj->build_rows / load_factor);
  uint64_t slots = 16;
  // at least one slot must stay empty: every probe loop ends on an empty slot (load_factor 1.0 with a power-of-two row count)
  while ((double)slots < want || slots <= (uint64_t)hj->build_rows) slots <<= 1;
  B2_EXPECTS(slots <= (1ull << 31), B2_ERR_INVALID_ARGUMENT, "hash join: build table too large for this load factor");
  hj->mask  = (uint32_t)(slots - 1);
  hj->table = dbuf(slots * sizeof(slot_t), stream);
  B2_CUDA_TRY(cudaMemsetAsync(hj->table.ptr, 0xff, hj->table.bytes, stream));
  const bool skip_nulls = compare_nulls == B2_NULLS_UNEQUAL;
  const int64_t n = hj->build_rows;
  hj->table_has_null_rows = table_has_nulls(build) && !skip_nulls;
  {
    prof_scope ps("join_build", stream);
    if (hj->wide) B2_LAUNCH(build_wide_kernel, grid_for(n), 256, 0, stream, kc, n, skip_nulls, hj->table.as<slot_t>(), hj->mask);
    else B2_LAUNCH(build_kernel, grid_for(n), 256, 0, stream, kc, n, skip_nulls, hj->table.as<slot_t>(), hj->mask);
  }
  return hj.release();
}

// validate_hash_join_probe — hash_join.cu:47-59
static void validate_probe(const b2_hash_join& hj, const std::vector<b2_column_view>& probe)
{
  B2_EXPECTS(!probe.empty(), B2_ERR_INVALID_ARGUMENT, "Hash join probe table is empty");
  B2_EXPECTS(probe.size() == hj.build_types.size(), B2_ERR_INVALID_ARGUMENT, "Mismatch in number of columns to be joined on");
  B2_EXPECTS(hj.has_nulls || !table_has_nulls(probe), B2_ERR_INVALID_ARGUMENT,
             "Probe table has nulls while build table was not hashed with null check.");
  for (size_t i = 0; i < probe.size(); ++i)
    B2_EXPECTS(probe[i].type_id == hj.build_types[i], B2_ERR_DATA_TYPE, "Mismatch in joining column data types");
}

struct probe_counts {
  dbuf counts;  // int32 per probe row (true match counts)
  size_t total = 0;
};

static probe_counts run_count(const b2_hash_join& hj, const key_cols& kc, int64_t n, bool left, bool keep_counts,
                              cudaStream_t stream)
{
  probe_counts pc;
  if (n == 0) return pc;
  if (keep_counts) pc.counts = dbuf(sizeof(int32_t) * n, stream);
  dbuf tot(sizeof(unsigned long long), stream);
  B2_CUDA_TRY(cudaMemsetAsync(tot.ptr, 0, sizeof(unsigned long long), stream));
  const bool skip_nulls = hj.compare_nulls == B2_NULLS_UNEQUAL;
  const slot_t* table = hj.table.as<slot_t>();
  {
    prof_scope ps("join_count", stream);
    if (hj.wide) {
      const key_cols bk = make_key_cols(hj.build_cols, true);
      if (left)
        B2_LAUNCH((count_wide_kernel<true>), grid_for(n), 256, 0, stream, kc, bk, n, skip_nulls, hj.table_has_null_rows, table,
                  hj.mask, pc.counts.as<int32_t>(), tot.as<unsigned long long>());
      else
        B2_LAUNCH((count_wide_kernel<false>), grid_for(n), 256, 0, stream, kc, bk, n, skip_nulls, hj.table_has_null_rows, table,
                  hj.mask, pc.counts.as<int32_t>(), tot.as<unsigned long long>());
    } else if (left)
      B2_LAUNCH((count_kernel<true>), grid_for(n), 256, 0, stream, kc, n, skip_nulls, hj.table_has_null_rows, table, hj.mask,
                pc.counts.as<int32_t>(), tot.as<unsigned long long>());
    else
      B2_LAUNCH((count_kernel<false>), grid_for(n), 256, 0, stream, kc, n, skip_nulls, hj.table_has_null_rows, table, hj.mask,
                pc.counts.as<int32_t>(), tot.as<unsigned long long>());
  }
  unsigned long long h = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&h, tot.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));  // the reference syncs here too (size_impl.cuh:52-61)
  pc.total = (size_t)h;
  return pc;
}

void hash_join_probe(const b2_hash_join* hj, const std::vector<b2_column_view>& probe, int kind, bool has_size, size_t size_hint,
                     cudaStream_t stream, column_ptr& out_left, column_ptr& out_right);

size_t hash_join_size(const b2_hash_join* hj, const std::vector<b2_column_view>& probe, int kind, cudaStream_t stream)
{
  validate_probe(*hj, probe);
  const int64_t n = probe[0].size;
  const key_cols kc = make_key_cols(probe, hj->wide);
  if (kind == JOIN_INNER) {
    if (n == 0 || hj->build_rows == 0) return 0;
    return run_count(*hj, kc, n, false, false, stream).total;
  }
  size_t left_total = n == 0 ? 0 : run_count(*hj, kc, n, true, kind == JOIN_FULL, stream).total;
  if (kind == JOIN_LEFT) return left_total;
  // FULL: + build rows that no probe row matched. Needs the actual right indices -> run the join.
  column_ptr l, r;
  hash_join_probe(hj, probe, JOIN_FULL, false, 0, stream, l, r);
  return (size_t)l->size;
}

void hash_join_probe(const b2_hash_join* hj, const std::vector<b2_column_view>& probe, int kind, bool has_size, size_t size_hint,
                     cudaStream_t stream, column_ptr& out_left, column_ptr& out_right)
{
  (void)has_size; (void)size_hint;  // the size is always recomputed: the count pass also yields the offsets
  validate_probe(*hj, probe);
  const int64_t n = probe[0].size;
  const key_cols kc = make_key_cols(probe, hj->wide);
  const bool left = kind != JOIN_INNER;

  size_t m = 0;
  probe_counts pc;
  if (n > 0 && (left || hj->build_rows > 0)) {
    pc = run_count(*hj, kc, n, left, true, stream);
    m  = pc.total;
  }
  B2_EXPECTS(m <= (size_t)INT32_MAX, B2_ERR_LOGIC /* std::overflow_error in libcudf */,
             "join output exceeds size_type (use hash_join::*_join_size and partition the probe side)");

  // unmatched build rows (FULL) are appended after the left-join part
  dbuf bitmap, word_counts;
  column_ptr word_offsets;
  int64_t extra = 0;

  auto L = make_column(B2_INT32, (int32_t)m, false, stream);
  auto R = make_column(B2_INT32, (int32_t)m, false, stream);
  if (m > 0) {
    // offsets = exclusive scan of per-row output counts
    dbuf adj;
    const int32_t* cnt_for_scan = pc.counts.as<int32_t>();
    if (left) {
      adj = dbuf(sizeof(int32_t) * n, stream);
      B2_LAUNCH(left_adjust_kernel, grid_for(n), 256, 0, stream, pc.counts.as<int32_t>(), n, adj.as<int32_t>());
      cnt_for_scan = adj.as<int32_t>();
    }
    b2_column_view cv{B2_INT32, (int32_t)n, cnt_for_scan, nullptr, 0, 0};
    auto offs = scan(cv, B2_AGG_SUM, B2_SCAN_EXCLUSIVE, B2_NULL_EXCLUDE, stream);
    prof_scope ps("join_retrieve", stream);
    if (hj->wide) {
      const key_cols bk = make_key_cols(hj->build_cols, true);
      if (left)
        B2_LAUNCH((retrieve_wide_kernel<true>), grid_for(n), 256, 0, stream, kc, bk, n, hj->table.as<slot_t>(), hj->mask,
                  pc.counts.as<int32_t>(), offs->data.as<int32_t>(), L->data.as<int32_t>(), R->data.as<int32_t>());
      else
        B2_LAUNCH((retrieve_wide_kernel<false>), grid_for(n), 256, 0, stream, kc, bk, n, hj->table.as<slot_t>(), hj->mask,
                  pc.counts.as<int32_t>(), offs->data.as<int32_t>(), L->data.as<int32_t>(), R->data.as<int32_t>());
    } else if (left)
      B2_LAUNCH((retrieve_kernel<true>), grid_for(n), 256, 0, stream, kc, n, hj->table.as<slot_t>(), hj->mask,
                pc.counts.as<int32_t>(), offs->data.as<int32_t>(), L->data.as<int32_t>(), R->data.as<int32_t>());
    else
      B2_LAUNCH((retrieve_kernel<false>), grid_for(n), 256, 0, stream, kc, n, hj->table.as<slot_t>(), hj->mask,
                pc.counts.as<int32_t>(), offs->data.as<int32_t>(), L->data.as<int32_t>(), R->data.as<int32_t>());
  }
  if (kind == JOIN_FULL && hj->build_rows > 0) {
    const int64_t nb = hj->build_rows;
    const int64_t nwords = (nb + 31) / 32;
    bitmap = dbuf(sizeof(uint32_t) * nwords, stream);
    B2_CUDA_TRY(cudaMemsetAsync(bitmap.ptr, 0, bitmap.bytes, stream));
    if (m > 0) B2_LAUNCH(mark_kernel, grid_for((int64_t)m), 256, 0, stream, R->data.as<int32_t>(), (int64_t)m, bitmap.as<uint32_t>());
    word_counts = dbuf(sizeof(int32_t) * nwords, stream);
    B2_LAUNCH(unmatched_count_kernel, grid_for(nwords), 256, 0, stream, bitmap.as<uint32_t>(), nb, word_counts.as<int32_t>());
    b2_column_view wc{B2_INT32, (int32_t)nwords, word_counts.ptr, nullptr, 0, 0};
    word_offsets = scan(wc, B2_AGG_SUM, B2_SCAN_EXCLUSIVE, B2_NULL_EXCLUDE, stream);
    int32_t last_off = 0, last_cnt = 0;
    B2_CUDA_TRY(cudaMemcpyAsync(&last_off, word_offsets->data.as<int32_t>() + (nwords - 1), 4, cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaMemcpyAsync(&last_cnt, word_counts.as<int32_t>() + (nwords - 1), 4, cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    extra = (int64_t)last_off + last_cnt;
    if (extra > 0) {
      B2_EXPECTS(m + (size_t)extra <= (size_t)INT32_MAX, B2_ERR_LOGIC, "join output exceeds size_type");
      auto L2 = make_column(B2_INT32, (int32_t)(m + extra), false, stream);
      auto R2 = make_column(B2_INT32, (int32_t)(m + extra), false, stream);
      if (m > 0) {
        B2_CUDA_TRY(cudaMemcpyAsync(L2->data.ptr, L->data.ptr, m * 4, cudaMemcpyDeviceToDevice, stream));
        B2_CUDA_TRY(cudaMemcpyAsync(R2->data.ptr, R->data.ptr, m * 4, cudaMemcpyDeviceToDevice, stream));
      }
      B2_LAUNCH(unmatched_write_kernel, grid_for(nwords), 256, 0, stream, bitmap.as<uint32_t>(), nb, word_offsets->data.as<int32_t>(),
                (int64_t)m, L2->data.as<int32_t>(), R2->data.as<int32_t>());
      L = std::move(L2);
      R = std::move(R2);
    }
  }
  out_left  = std::move(L);
  out_right = std::move(R);
}

// cudf::hash_join::{inner,left,full}_join_match_context — hash_join.hpp:254-330, match_context.cu
column_ptr hash_join_match_counts(const b2_hash_join* hj, const std::vector<b2_column_view>& probe, int kind, cudaStream_t stream)
{
  validate_probe(*hj, probe);
  const int64_t n = probe[0].size;
  const bool left = kind != JOIN_INNER;
  auto out = make_column(B2_INT32, (int32_t)n, false, stream);
  if (n == 0) return out;
  const key_cols kc = make_key_cols(probe, hj->wide);
  int32_t* counts = out->data.as<int32_t>();
  if (hj->build_rows == 0 || hj->table.ptr == nullptr) {
    B2_LAUNCH(fill_i32_kernel, grid_for(n), 256, 0, stream, counts, n, left ? 1 : 0);
    return out;
  }
  dbuf tot(sizeof(unsigned long long), stream);
  B2_CUDA_TRY(cudaMemsetAsync(tot.ptr, 0, sizeof(unsigned long long), stream));
  const bool skip_nulls = hj->compare_nulls == B2_NULLS_UNEQUAL;
  const slot_t* table = hj->table.as<slot_t>();
  {
    prof_scope ps("join_count", stream);
    if (hj->wide) {
      const key_cols bk = make_key_cols(hj->build_cols, true);
      B2_LAUNCH((count_wide_kernel<false>), grid_for(n), 256, 0, stream, kc, bk, n, skip_nulls, hj->table_has_null_rows, table, hj->mask,
                counts, tot.as<unsigned long long>());
    } else {
      B2_LAUNCH((count_kernel<false>), grid_for(n), 256, 0, stream, kc, n, skip_nulls, hj->table_has_null_rows, table, hj->mask, counts,
                tot.as<unsigned long long>());
    }
  }
  if (left) B2_LAUNCH(left_adjust_kernel, grid_for(n), 256, 0, stream, counts, n, counts);  // in place: max(count, 1)
  return out;
}

// cudf::hash_join::partitioned_{inner,left,full}_join — hash_join.hpp:331-411, partitioned_*_join.cu
void hash_join_partitioned(const b2_hash_join* hj, const std::vector<b2_column_view>& probe, const b2_column_view& match_counts,
                           int32_t left_start, int32_t left_end, int kind, cudaStream_t stream, column_ptr& out_left,
                           column_ptr& out_right)
{
  validate_probe(*hj, probe);
  const int64_t n = probe[0].size;
  B2_EXPECTS(match_counts.data != nullptr || n == 0, B2_ERR_INVALID_ARGUMENT, "join_partition_context without match counts");
  B2_EXPECTS(match_counts.type_id == B2_INT32 && match_counts.size == n, B2_ERR_INVALID_ARGUMENT,
             "match counts must be an INT32 column with one entry per probe row");
  B2_EXPECTS(left_start >= 0 && left_start <= left_end && left_end <= n, B2_ERR_INVALID_ARGUMENT,
             "partition bounds are outside the left table");
  const bool left = kind != JOIN_INNER;
  const int64_t m = (int64_t)left_end - left_start;
  const int32_t* counts = static_cast<const int32_t*>(match_counts.data) + match_counts.offset;
  size_t total = 0;
  column_ptr offs;
  if (m > 0) {
    b2_column_view part{B2_INT32, (int32_t)m, counts, nullptr, 0, left_start};
    auto sum = reduce(part, B2_AGG_SUM, B2_INT64, nullptr, stream);
    long long h = 0;
    B2_CUDA_TRY(cudaMemcpyAsync(&h, sum->data.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    total = (size_t)h;
    B2_EXPECTS(total <= (size_t)INT32_MAX, B2_ERR_LOGIC, "join output of this partition exceeds size_type");
    offs = scan(part, B2_AGG_SUM, B2_SCAN_EXCLUSIVE, B2_NULL_EXCLUDE, stream);
  }
  out_left  = make_column(B2_INT32, (int32_t)total, false, stream);
  out_right = make_column(B2_INT32, (int32_t)total, false, stream);
  if (total == 0) return;
  const key_cols pk = make_key_cols(probe, hj->wide);
  const key_cols bk = hj->wide ? make_key_cols(hj->build_cols, true) : key_cols{};
  const slot_t* table = hj->build_rows > 0 ? hj->table.as<slot_t>() : nullptr;
  prof_scope ps("join_retrieve", stream);
#define B2_RP(L, W)                                                                                                              \
  B2_LAUNCH((retrieve_part_kernel<L, W>), grid_for(m), 256, 0, stream, pk, bk, (int64_t)left_start, m, table, hj->mask, counts, \
            offs->data.as<int32_t>(), out_left->data.as<int32_t>(), out_right->data.as<int32_t>())
  if (left) { if (hj->wide) B2_RP(true, true); else B2_RP(true, false); }
  else      { if (hj->wide) B2_RP(false, true); else B2_RP(false, false); }
#undef B2_RP
}

// cudf::hash_join::finalize_partitioned_full_join — hash_join.hpp:413-440, finalize_partitioned_full_join.cpp
void hash_join_finalize_full(const std::vector<b2_column_view>& lparts, const std::vector<b2_column_view>& rparts, int32_t left_rows,
                             int32_t right_rows, cudaStream_t stream, column_ptr& out_left, column_ptr& out_right)
{
  (void)left_rows;
  B2_EXPECTS(lparts.size() == rparts.size(), B2_ERR_INVALID_ARGUMENT, "left and right partials differ in number");
  B2_EXPECTS(right_rows >= 0, B2_ERR_INVALID_ARGUMENT, "negative table size");
  int64_t m = 0;
  for (size_t i = 0; i < lparts.size(); ++i) {
    B2_EXPECTS(lparts[i].size == rparts[i].size, B2_ERR_INVALID_ARGUMENT, "left and right partial of one partition differ in size");
    B2_EXPECTS(lparts[i].type_id == B2_INT32 && rparts[i].type_id == B2_INT32, B2_ERR_DATA_TYPE, "join indices are INT32");
    m += lparts[i].size;
  }
  const int64_t nwords = ((int64_t)right_rows + 31) / 32;
  dbuf bitmap(sizeof(uint32_t) * std::max<int64_t>(nwords, 1), stream), word_counts(sizeof(int32_t) * std::max<int64_t>(nwords, 1), stream);
  B2_CUDA_TRY(cudaMemsetAsync(bitmap.ptr, 0, bitmap.bytes, stream));
  for (auto& r : rparts)
    if (r.size > 0)
      B2_LAUNCH(mark_kernel, grid_for(r.size), 256, 0, stream, static_cast<const int32_t*>(r.data) + r.offset, (int64_t)r.size,
                bitmap.as<uint32_t>());
  int64_t extra = 0;
  column_ptr word_offsets;
  if (right_rows > 0) {
    B2_LAUNCH(unmatched_count_kernel, grid_for(nwords), 256, 0, stream, bitmap.as<uint32_t>(), (int64_t)right_rows, word_counts.as<int32_t>());
    b2_column_view wc{B2_INT32, (int32_t)nwords, word_counts.ptr, nullptr, 0, 0};
    word_offsets = scan(wc, B2_AGG_SUM, B2_SCAN_EXCLUSIVE, B2_NULL_EXCLUDE, stream);
    int32_t last_off = 0, last_cnt = 0;
    B2_CUDA_TRY(cudaMemcpyAsync(&last_off, word_offsets->data.as<int32_t>() + (nwords - 1), 4, cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaMemcpyAsync(&last_cnt, word_counts.as<int32_t>() + (nwords - 1), 4, cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    extra = (int64_t)last_off + last_cnt;
  }
  B2_EXPECTS(m + extra <= (int64_t)INT32_MAX, B2_ERR_LOGIC, "join output exceeds size_type");
  out_left  = make_column(B2_INT32, (int32_t)(m + extra), false, stream);
  out_right = make_column(B2_INT32, (int32_t)(m + extra), false, stream);
  int64_t at = 0;
  for (size_t i = 0; i < lparts.size(); ++i) {
    const int64_t k = lparts[i].size;
    if (k == 0) continue;
    B2_CUDA_TRY(cudaMemcpyAsync(out_left->data.as<int32_t>() + at, static_cast<const int32_t*>(lparts[i].data) + lparts[i].offset, k * 4,
                                cudaMemcpyDeviceToDevice, stream));
    B2_CUDA_TRY(cudaMemcpyAsync(out_right->data.as<int32_t>() + at, static_cast<const int32_t*>(rparts[i].data) + rparts[i].offset, k * 4,
                                cudaMemcpyDeviceToDevice, stream));
    at += k;
  }
  if (extra > 0)
    B2_LAUNCH(unmatched_write_kernel, grid_for(nwords), 256, 0, stream, bitmap.as<uint32_t>(), (int64_t)right_rows,
              word_offsets->data.as<int32_t>(), m, out_left->data.as<int32_t>(), out_right->data.as<int32_t>());
}

}  // namespace b2

// ---- C ABI -----------------------------------------------------------------------------------------
static cudaStream_t S(b2_stream s) { return static_cast<cudaStream_t>(s); }

// free functions: cpp/src/join/join.cu:27-110
static b2_status free_join(const b2_table_view* left, const b2_table_view* right, int32_t compare_nulls, int kind,
                           b2_stream stream, b2_column** out_left, b2_column** out_right)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out_left && out_right, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> l, r;
  validate_table(left, l);
  validate_table(right, r);
  B2_EXPECTS(l.size() == r.size(), B2_ERR_INVALID_ARGUMENT, "Mismatch in number of columns to be joined on");
  B2_EXPECTS(!l.empty(), B2_ERR_INVALID_ARGUMENT, "Join key tables are empty");
  for (size_t i = 0; i < l.size(); ++i) B2_EXPECTS(l[i].type_id == r[i].type_id, B2_ERR_DATA_TYPE, "Mismatch in joining column data types");
  const bool nulls = table_has_nulls(l) || table_has_nulls(r);
  column_ptr lo, ro;
  // inner join builds on the smaller table and swaps the outputs back (join.cu:52-59)
  if (radix_join_applicable(l, r)) {  // partitioned path (radix_join.cu): both sides >= 2^24 null-free rows, keys <= 8 bytes
    make_key_cols(l, true);  // same argument checks as the hash path
    if (kind == JOIN_INNER) {
      if (r[0].size > l[0].size) radix_join(l, r, false, S(stream), ro, lo);
      else radix_join(r, l, false, S(stream), lo, ro);
    } else {
      radix_join(r, l, true, S(stream), lo, ro);  // the left table is the probe side
      if (kind == JOIN_FULL) {
        const b2_column_view lv{B2_INT32, lo->size, lo->data.ptr, nullptr, 0, 0}, rv{B2_INT32, ro->size, ro->data.ptr, nullptr, 0, 0};
        column_ptr fl, fr;
        hash_join_finalize_full({lv}, {rv}, l[0].size, r[0].size, S(stream), fl, fr);
        lo = std::move(fl);
        ro = std::move(fr);
      }
    }
  } else if (kind == JOIN_INNER && r[0].size > l[0].size) {
    std::unique_ptr<b2_hash_join> hj(hash_join_create(l, nulls, compare_nulls, 0.5, S(stream)));
    hash_join_probe(hj.get(), r, JOIN_INNER, false, 0, S(stream), ro, lo);
  } else {
    std::unique_ptr<b2_hash_join> hj(hash_join_create(r, nulls, compare_nulls, 0.5, S(stream)));
    hash_join_probe(hj.get(), l, kind, false, 0, S(stream), lo, ro);
  }
  *out_left  = lo.release();
  *out_right = ro.release();
  B2_TRY_END
}

extern "C" {

b2_status b2_inner_join(const b2_table_view* l, const b2_table_view* r, int32_t cn, b2_stream s, b2_column** ol, b2_column** orr)
{
  return free_join(l, r, cn, JOIN_INNER, s, ol, orr);
}
b2_status b2_left_join(const b2_table_view* l, const b2_table_view* r, int32_t cn, b2_stream s, b2_column** ol, b2_column** orr)
{
  return free_join(l, r, cn, JOIN_LEFT, s, ol, orr);
}
b2_status b2_full_join(const b2_table_view* l, const b2_table_view* r, int32_t cn, b2_stream s, b2_column** ol, b2_column** orr)
{
  return free_join(l, r, cn, JOIN_FULL, s, ol, orr);
}

b2_status b2_hash_join_create(const b2_table_view* build, int32_t has_nulls, int32_t compare_nulls, double load_factor,
                              b2_stream stream, b2_hash_join** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(build, cols);
  *out = hash_join_create(cols, has_nulls, compare_nulls, load_factor, S(stream));
  B2_TRY_END
}
void b2_hash_join_destroy(b2_hash_join* hj) { delete hj; }

static b2_status obj_join(const b2_hash_join* hj, const b2_table_view* probe, int kind, int32_t has_size, size_t size, b2_stream stream,
                          b2_column** ol, b2_column** orr)
{
  B2_TRY_BEGIN
  B2_EXPECTS(hj && ol && orr, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(probe, cols);
  column_ptr l, r;
  hash_join_probe(hj, cols, kind, has_size != 0, size, S(stream), l, r);
  *ol  = l.release();
  *orr = r.release();
  B2_TRY_END
}
static b2_status obj_size(const b2_hash_join* hj, const b2_table_view* probe, int kind, b2_stream stream, size_t* out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(hj && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(probe, cols);
  *out = hash_join_size(hj, cols, kind, S(stream));
  B2_TRY_END
}
b2_status b2_hash_join_inner_join(const b2_hash_join* hj, const b2_table_view* p, int32_t hs, size_t sz, b2_stream s, b2_column** l, b2_column** r) { return obj_join(hj, p, JOIN_INNER, hs, sz, s, l, r); }
b2_status b2_hash_join_left_join(const b2_hash_join* hj, const b2_table_view* p, int32_t hs, size_t sz, b2_stream s, b2_column** l, b2_column** r) { return obj_join(hj, p, JOIN_LEFT, hs, sz, s, l, r); }
b2_status b2_hash_join_full_join(const b2_hash_join* hj, const b2_table_view* p, int32_t hs, size_t sz, b2_stream s, b2_column** l, b2_column** r) { return obj_join(hj, p, JOIN_FULL, hs, sz, s, l, r); }
b2_status b2_hash_join_match_counts(const b2_hash_join* hj, const b2_table_view* probe, int32_t join_kind, b2_stream stream,
                                    b2_column** out_counts)
{
  B2_TRY_BEGIN
  B2_EXPECTS(hj && out_counts, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_EXPECTS(join_kind >= JOIN_INNER && join_kind <= JOIN_FULL, B2_ERR_INVALID_ARGUMENT, "unknown join kind");
  std::vector<b2_column_view> p;
  validate_table(probe, p);
  *out_counts = hash_join_match_counts(hj, p, join_kind, S(stream)).release();
  B2_TRY_END
}

b2_status b2_hash_join_partitioned_join(const b2_hash_join* hj, const b2_table_view* probe, const b2_column_view* match_counts,
                                        int32_t left_start, int32_t left_end, int32_t join_kind, b2_stream stream, b2_column** out_left,
                                        b2_column** out_right)
{
  B2_TRY_BEGIN
  B2_EXPECTS(hj && out_left && out_right, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_EXPECTS(match_counts != nullptr, B2_ERR_INVALID_ARGUMENT, "join_partition_context without a match context");
  B2_EXPECTS(join_kind >= JOIN_INNER && join_kind <= JOIN_FULL, B2_ERR_INVALID_ARGUMENT, "unknown join kind");
  std::vector<b2_column_view> p;
  validate_table(probe, p);
  column_ptr l, r;
  hash_join_partitioned(hj, p, *match_counts, left_start, left_end, join_kind, S(stream), l, r);
  *out_left  = l.release();
  *out_right = r.release();
  B2_TRY_END
}

b2_status b2_hash_join_finalize_full_join(const b2_column_view* left_partials, const b2_column_view* right_partials, int32_t num_partials,
                                          int32_t left_table_num_rows, int32_t right_table_num_rows, b2_stream stream,
                                          b2_column** out_left, b2_column** out_right)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out_left && out_right && num_partials >= 0 && (num_partials == 0 || (left_partials && right_partials)),
             B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> lp(left_partials, left_partials + num_partials), rp(right_partials, right_partials + num_partials);
  column_ptr l, r;
  hash_join_finalize_full(lp, rp, left_table_num_rows, right_table_num_rows, S(stream), l, r);
  *out_left  = l.release();
  *out_right = r.release();
  B2_TRY_END
}

b2_status b2_hash_join_inner_join_size(const b2_hash_join* hj, const b2_table_view* p, b2_stream s, size_t* out) { return obj_size(hj, p, JOIN_INNER, s, out); }
b2_status b2_hash_join_left_join_size(const b2_hash_join* hj, const b2_table_view* p, b2_stream s, size_t* out) { return obj_size(hj, p, JOIN_LEFT, s, out); }
b2_status b2_hash_join_full_join_size(const b2_hash_join* hj, const b2_table_view* p, b2_stream s, size_t* out) { return obj_size(hj, p, JOIN_FULL, s, out); }

}  // extern "C"

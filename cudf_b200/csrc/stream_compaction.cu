// stream_compaction.cu — apply_boolean_mask / apply_deletion_mask, drop_nulls, drop_nans, unique, distinct,
// stable_distinct and distinct_indices for fixed-width tables (cpp/include/cudf/stream_compaction.hpp of the reference;
// cpp/src/stream_compaction/{apply_boolean_mask,drop_nulls,drop_nans,unique,distinct,stable_distinct}.cu).
//
// Every function ends in one stable compaction: compact_kernel (compact.cuh) evaluates a row predicate inline, ranks the
// kept rows of a warp with __ballot_sync / __popc, takes the tile base from a single-pass decoupled look-back (the 16-byte
// records of device_utils.cuh, as scan_kernel) and writes the kept row ids, INT32 and in input order. The columns are then
// gathered through that monotone map (gather.cu). One host read-back per call, for the output row count (the reference's
// copy_if also syncs for the size).
//   unique:   unique_flags_kernel marks row i kept by comparing its key with its neighbours (FIRST: i-1, LAST: i+1, NONE:
//             both), one byte per row; the flags are then compacted as a BOOL8 mask.
//   distinct: distinct_insert_kernel finds or claims each key row's slot {key, representative row, nullbits} in a linear-
//             probing table with one 128-bit CAS (the groupby's protocol, key_pack.cuh) and keeps an atomicMin (FIRST) /
//             atomicMax (LAST) of the row id or a count (NONE) per slot; rows whose key holds a null under nulls UNEQUAL,
//             or a NaN under nans UNEQUAL, are distinct by definition and are flagged directly. distinct_mark_kernel then
//             flags each slot's kept row. The flags compact in input order, so `distinct` returns the stable_distinct
//             result (a valid "unspecified" order). The table starts L2-sized and grows x8 after a device overflow signal.
#include "common.cuh"
#include "compact.cuh"
#include "device_utils.cuh"
#include "key_pack.cuh"

#include <algorithm>
#include <climits>

namespace b2 {
namespace {

// duplicate_keep_option (cpp/include/cudf/stream_compaction.hpp:68-73) and nan_equality (types.hpp)
enum { KEEP_ANY = 0, KEEP_FIRST = 1, KEEP_LAST = 2, KEEP_NONE = 3 };
enum { NULLS_EQUAL = 0, NULLS_UNEQUAL = 1 };
enum { NANS_ALL_EQUAL = 0, NANS_UNEQUAL = 1 };

// ---- row predicates ----------------------------------------------------------------------------------
// BOOL8 mask (data already offset; validity at bit `bit_offset + r`): keep when valid and (value != 0) != invert
struct mask_pred {
  const uint8_t* data;
  const uint32_t* valid;
  int64_t bit_offset;
  bool invert;
  __device__ __forceinline__ bool operator()(int64_t r) const
  {
    if (valid != nullptr && !bit_is_set(valid, bit_offset + r)) return false;
    return (__ldcs(data + r) != 0) != invert;
  }
};

// at least `threshold` of the key columns are valid at row r (kc.mask is null for columns without nulls)
struct valid_count_pred {
  key_cols kc;
  int32_t threshold;
  __device__ __forceinline__ bool operator()(int64_t r) const
  {
    int cnt = 0;
#pragma unroll 1
    for (int c = 0; c < kc.n; ++c) cnt += kc.mask[c] == nullptr || bit_is_set(kc.mask[c], r + kc.offset[c]);
    return cnt >= threshold;
  }
};

__device__ __forceinline__ bool key_is_nan(const key_cols& kc, int c, int64_t e)
{
  if (kc.width[c] == 4) return (static_cast<const uint32_t*>(kc.data[c])[e] & 0x7fffffffu) > 0x7f800000u;
  return (static_cast<const uint64_t*>(kc.data[c])[e] & 0x7fffffffffffffffull) > 0x7ff0000000000000ull;
}

// at least `threshold` of the (float) key columns are not NaN at row r; a null counts as not NaN (drop_nans.cu:24-38)
struct not_nan_count_pred {
  key_cols kc;
  int32_t threshold;
  __device__ __forceinline__ bool operator()(int64_t r) const
  {
    int cnt = 0;
#pragma unroll 1
    for (int c = 0; c < kc.n; ++c) {
      const int64_t e = r + kc.offset[c];
      cnt += (kc.mask[c] != nullptr && !bit_is_set(kc.mask[c], e)) || !key_is_nan(kc, c, e);
    }
    return cnt >= threshold;
  }
};

// ---- stable compaction (compact.cuh) + gather -------------------------------------------------------------
template <typename P>
table_ptr compact_table(const std::vector<b2_column_view>& cols, const P& pred, int64_t n, cudaStream_t stream)
{
  dbuf map;
  const int32_t m = compact(pred, n, map, stream);
  return gather_table(cols, map.as<int32_t>(), m, false, stream);
}

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)num_sms() * 16)); }

// ---- unique ----------------------------------------------------------------------------------------------
__device__ __forceinline__ bool any_null(const key_cols& kc, int64_t r)
{
#pragma unroll 1
  for (int c = 0; c < kc.n; ++c)
    if (kc.mask[c] != nullptr && !bit_is_set(kc.mask[c], r + kc.offset[c])) return true;
  return false;
}

// rows a and b have equal keys (NaN == NaN, -0 == +0); under nulls UNEQUAL a row with a null key equals no row
template <bool WIDE>
__device__ __forceinline__ bool keys_equal(const key_cols& kc, int64_t a, int64_t b, bool nulls_unequal)
{
  if constexpr (WIDE) {
    if (nulls_unequal && (any_null(kc, a) || any_null(kc, b))) return false;
    return rows_equal_wide(kc, a, kc, b);
  } else {
    uint64_t ka, kb;
    uint32_t na, nb;
    pack_row(kc, a, ka, na);
    pack_row(kc, b, kb, nb);
    if (nulls_unequal && (na | nb)) return false;
    return ka == kb && na == nb;
  }
}

template <bool WIDE>
__global__ void __launch_bounds__(256) unique_flags_kernel(key_cols kc, int64_t n, int keep, bool nulls_unequal,
                                                           uint8_t* __restrict__ flags)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    bool keep_row = true;
    if (keep != KEEP_LAST && r > 0) keep_row = !keys_equal<WIDE>(kc, r, r - 1, nulls_unequal);
    if (keep_row && keep != KEEP_FIRST && r + 1 < n) keep_row = !keys_equal<WIDE>(kc, r, r + 1, nulls_unequal);
    flags[r] = keep_row ? 1 : 0;
  }
}

// ---- distinct --------------------------------------------------------------------------------------------
struct dc_ctl {
  unsigned int nslots_used;
  unsigned int overflow;
};

__device__ __forceinline__ bool row_has_nan(const key_cols& kc, int64_t r)
{
#pragma unroll 1
  for (int c = 0; c < kc.n; ++c) {
    if (!kc.is_float[c]) continue;
    const int64_t e = r + kc.offset[c];
    if ((kc.mask[c] == nullptr || bit_is_set(kc.mask[c], e)) && key_is_nan(kc, c, e)) return true;
  }
  return false;
}

template <bool WIDE>
__global__ void __launch_bounds__(256) distinct_insert_kernel(key_cols kc, int64_t n, int keep, bool nulls_unequal,
                                                              bool nans_unequal, slot_t* __restrict__ table, uint32_t mask,
                                                              uint32_t cap, int32_t* __restrict__ aux, uint8_t* __restrict__ flags,
                                                              dc_ctl* ctl)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  slot_t empty;
  memset(&empty, 0xff, sizeof(empty));
  int iter = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride, ++iter) {
    // table too small -> the host grows it and reruns (polled rarely, as in groupby_kernel)
    if ((iter & 63) == 0 && *reinterpret_cast<volatile unsigned int*>(&ctl->overflow)) return;
    uint64_t key;
    uint32_t nb;
    if constexpr (WIDE) hash_row_wide(kc, r, key, nb);
    else pack_row(kc, r, key, nb);
    if ((nulls_unequal && nb) || (nans_unequal && row_has_nan(kc, r))) {  // equal to no other row
      flags[r] = 1;
      continue;
    }
    uint32_t i = slot_hash(key, nb, mask);
    int probes = 0;
    while (true) {
      if (((++probes) & 127) == 0 && *reinterpret_cast<volatile unsigned int*>(&ctl->overflow)) return;
      slot_t cur = load_slot_volatile(&table[i]);
      if (cur.row == -1) {
        const slot_t want{key, (int32_t)r, nb};
        cur = cas128(&table[i], empty, want);
        if (cur.row == -1) {  // this row claimed the slot
          if (atomicAdd(&ctl->nslots_used, 1u) >= cap) { atomicExch(&ctl->overflow, 1u); return; }
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
    if (keep == KEEP_FIRST) atomicMin(&aux[i], (int32_t)r);
    else if (keep == KEEP_LAST) atomicMax(&aux[i], (int32_t)r);
    else if (keep == KEEP_NONE) atomicAdd(&aux[i], 1);
  }
}

__global__ void __launch_bounds__(256) distinct_mark_kernel(const slot_t* __restrict__ table, int64_t slots, int keep,
                                                            const int32_t* __restrict__ aux, uint8_t* __restrict__ flags)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += stride) {
    const int32_t rep = table[i].row;
    if (rep < 0) continue;
    if (keep == KEEP_ANY) flags[rep] = 1;
    else if (keep == KEEP_NONE) { if (aux[i] == 1) flags[rep] = 1; }
    else flags[aux[i]] = 1;
  }
}

// one flag byte per key row: 1 = the row is kept
dbuf distinct_flags(const std::vector<b2_column_view>& keys, int keep, bool nulls_unequal, bool nans_unequal, cudaStream_t stream)
{
  const int64_t n = keys[0].size;
  const bool wide = keys_are_wide(keys);
  const key_cols kc = make_key_cols(keys, true);
  dbuf flags((size_t)n, stream);
  uint64_t max_slots = 16;
  while (max_slots < 2ull * (uint64_t)n) max_slots <<= 1;
  uint64_t slots = std::min<uint64_t>(max_slots, 1ull << 21);
  while (true) {
    const uint32_t cap = (uint32_t)std::min<uint64_t>((uint64_t)n, (uint64_t)(slots * 0.6));
    dbuf table(slots * sizeof(slot_t), stream), aux(slots * sizeof(int32_t), stream), ctl(sizeof(dc_ctl), stream);
    B2_CUDA_TRY(cudaMemsetAsync(table.ptr, 0xff, table.bytes, stream));
    // FIRST: min of row ids (0x7f7f7f7f exceeds every row id); LAST: max (-1); NONE: count (0)
    B2_CUDA_TRY(cudaMemsetAsync(aux.ptr, keep == KEEP_FIRST ? 0x7f : keep == KEEP_LAST ? 0xff : 0, aux.bytes, stream));
    B2_CUDA_TRY(cudaMemsetAsync(ctl.ptr, 0, sizeof(dc_ctl), stream));
    B2_CUDA_TRY(cudaMemsetAsync(flags.ptr, 0, flags.bytes, stream));
    {
      prof_scope ps("distinct_insert", stream);
      if (wide)
        B2_LAUNCH((distinct_insert_kernel<true>), grid_for(n), 256, 0, stream, kc, n, keep, nulls_unequal, nans_unequal,
                  table.as<slot_t>(), (uint32_t)(slots - 1), cap, aux.as<int32_t>(), flags.as<uint8_t>(), ctl.as<dc_ctl>());
      else
        B2_LAUNCH((distinct_insert_kernel<false>), grid_for(n), 256, 0, stream, kc, n, keep, nulls_unequal, nans_unequal,
                  table.as<slot_t>(), (uint32_t)(slots - 1), cap, aux.as<int32_t>(), flags.as<uint8_t>(), ctl.as<dc_ctl>());
    }
    dc_ctl h{};
    B2_CUDA_TRY(cudaMemcpyAsync(&h, ctl.ptr, sizeof(h), cudaMemcpyDeviceToHost, stream));
    B2_CUDA_TRY(cudaStreamSynchronize(stream));
    if (h.overflow) {
      B2_EXPECTS(slots < max_slots, B2_ERR_LOGIC, "distinct: hash table overflow at maximum size");
      slots = std::min<uint64_t>(max_slots, slots * 8);
      continue;  // buffers are released (stream-ordered) and rebuilt at the new size
    }
    prof_scope ps("distinct_mark", stream);
    B2_LAUNCH(distinct_mark_kernel, grid_for((int64_t)slots), 256, 0, stream, table.as<slot_t>(), (int64_t)slots, keep,
              aux.as<int32_t>(), flags.as<uint8_t>());
    return flags;
  }
}

// ---- host helpers ----------------------------------------------------------------------------------------
table_ptr empty_like(const std::vector<b2_column_view>& cols, cudaStream_t stream)
{
  auto t = std::make_unique<b2_table>();
  for (const auto& c : cols) t->cols.push_back(make_column(c.type_id, 0, false, stream));
  return t;
}

table_ptr copy_table(const std::vector<b2_column_view>& cols, cudaStream_t stream)
{
  auto t = std::make_unique<b2_table>();
  for (const auto& c : cols) {
    auto out = make_column(c.type_id, c.size, false, stream);
    const size_t w = type_width(c.type_id);
    if (c.size > 0)
      B2_CUDA_TRY(cudaMemcpyAsync(out->data.ptr, static_cast<const char*>(c.data) + w * (size_t)c.offset, w * (size_t)c.size,
                                  cudaMemcpyDeviceToDevice, stream));
    if (has_nulls(c)) {
      out->mask       = copy_bitmask(c.null_mask, c.offset, (int64_t)c.offset + c.size, stream);
      out->null_count = c.null_count;
    }
    t->cols.push_back(std::move(out));
  }
  return t;
}

// table_view::select: an index outside the table is std::out_of_range (std::vector::at)
std::vector<b2_column_view> select_keys(const std::vector<b2_column_view>& cols, const int32_t* keys, int32_t num_keys)
{
  B2_EXPECTS(num_keys >= 0 && (num_keys == 0 || keys != nullptr), B2_ERR_INVALID_ARGUMENT, "invalid key indices");
  std::vector<b2_column_view> out;
  for (int32_t i = 0; i < num_keys; ++i) {
    B2_EXPECTS(keys[i] >= 0 && keys[i] < (int32_t)cols.size(), B2_ERR_OUT_OF_RANGE, "key column index out of range");
    out.push_back(cols[keys[i]]);
  }
  return out;
}

void check_keep(int32_t keep, int32_t nulls_equal)
{
  B2_EXPECTS(keep >= KEEP_ANY && keep <= KEEP_NONE, B2_ERR_INVALID_ARGUMENT, "invalid duplicate_keep_option");
  B2_EXPECTS(nulls_equal == NULLS_EQUAL || nulls_equal == NULLS_UNEQUAL, B2_ERR_INVALID_ARGUMENT, "invalid null_equality");
}

// kept row ids of distinct (INT32, input order) in `map`; returns their count
int32_t distinct_map(const std::vector<b2_column_view>& keys, int32_t keep, int32_t nulls_equal, int32_t nans_equal, dbuf& map,
                     cudaStream_t stream)
{
  dbuf flags = distinct_flags(keys, keep, nulls_equal == NULLS_UNEQUAL, nans_equal == NANS_UNEQUAL, stream);
  return compact(mask_pred{flags.as<uint8_t>(), nullptr, 0, false}, keys[0].size, map, stream);
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_apply_boolean_mask(const b2_table_view* input, const b2_column_view* mask, int32_t deletion, b2_stream stream,
                                b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(mask && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto s = static_cast<cudaStream_t>(stream);
  if (mask->size == 0) { *out = empty_like(cols, s).release(); return B2_OK; }
  validate_column(*mask);
  B2_EXPECTS(mask->type_id == B2_BOOL8, B2_ERR_LOGIC, "Mask must be Boolean type");
  const int32_t rows = cols.empty() ? 0 : cols[0].size;
  B2_EXPECTS(rows == 0 || rows == mask->size, B2_ERR_LOGIC, "Column size mismatch");
  if (rows == 0) { *out = empty_like(cols, s).release(); return B2_OK; }
  const mask_pred p{static_cast<const uint8_t*>(mask->data) + mask->offset, has_nulls(*mask) ? mask->null_mask : nullptr,
                    (int64_t)mask->offset, deletion != 0};
  *out = compact_table(cols, p, rows, s).release();
  B2_TRY_END
}

b2_status b2_drop_nulls(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep_threshold,
                        b2_stream stream, b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto s = static_cast<cudaStream_t>(stream);
  const auto k = select_keys(cols, keys, num_keys);
  const bool any_nulls = std::any_of(k.begin(), k.end(), [](const b2_column_view& c) { return has_nulls(c); });
  if (k.empty() || k[0].size == 0 || !any_nulls) { *out = copy_table(cols, s).release(); return B2_OK; }
  *out = compact_table(cols, valid_count_pred{make_key_cols(k, true), keep_threshold}, k[0].size, s).release();
  B2_TRY_END
}

b2_status b2_drop_nans(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep_threshold,
                       b2_stream stream, b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto s = static_cast<cudaStream_t>(stream);
  const auto k = select_keys(cols, keys, num_keys);
  if (k.empty() || k[0].size == 0) { *out = copy_table(cols, s).release(); return B2_OK; }
  for (const auto& c : k) B2_EXPECTS(is_float_id(c.type_id), B2_ERR_LOGIC, "Key column is not of type floating-point");
  *out = compact_table(cols, not_nan_count_pred{make_key_cols(k, true), keep_threshold}, k[0].size, s).release();
  B2_TRY_END
}

b2_status b2_unique(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep, int32_t nulls_equal,
                    b2_stream stream, b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  check_keep(keep, nulls_equal);
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto s = static_cast<cudaStream_t>(stream);
  if (keep == KEEP_ANY) keep = KEEP_FIRST;
  const int32_t rows = cols.empty() ? 0 : cols[0].size;
  if (rows == 0 || cols.empty() || num_keys == 0) { *out = empty_like(cols, s).release(); return B2_OK; }
  const auto k = select_keys(cols, keys, num_keys);
  const key_cols kc = make_key_cols(k, true);
  dbuf flags((size_t)rows, s);
  if (keys_are_wide(k))
    B2_LAUNCH((unique_flags_kernel<true>), grid_for(rows), 256, 0, s, kc, (int64_t)rows, keep, nulls_equal == NULLS_UNEQUAL,
              flags.as<uint8_t>());
  else
    B2_LAUNCH((unique_flags_kernel<false>), grid_for(rows), 256, 0, s, kc, (int64_t)rows, keep, nulls_equal == NULLS_UNEQUAL,
              flags.as<uint8_t>());
  *out = compact_table(cols, mask_pred{flags.as<uint8_t>(), nullptr, 0, false}, rows, s).release();
  B2_TRY_END
}

b2_status b2_distinct(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep, int32_t nulls_equal,
                      int32_t nans_equal, int32_t stable, b2_stream stream, b2_table** out)
{
  (void)stable;  // both orders are produced by the same stable path
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  check_keep(keep, nulls_equal);
  B2_EXPECTS(nans_equal == NANS_ALL_EQUAL || nans_equal == NANS_UNEQUAL, B2_ERR_INVALID_ARGUMENT, "invalid nan_equality");
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto s = static_cast<cudaStream_t>(stream);
  const int32_t rows = cols.empty() ? 0 : cols[0].size;
  if (rows == 0 || cols.empty() || num_keys == 0) { *out = empty_like(cols, s).release(); return B2_OK; }
  const auto k   = select_keys(cols, keys, num_keys);
  dbuf map;
  const int32_t m = distinct_map(k, keep, nulls_equal, nans_equal, map, s);
  *out = gather_table(cols, map.as<int32_t>(), m, false, s).release();
  B2_TRY_END
}

b2_status b2_distinct_indices(const b2_table_view* input, int32_t keep, int32_t nulls_equal, int32_t nans_equal, b2_stream stream,
                              b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  check_keep(keep, nulls_equal);
  B2_EXPECTS(nans_equal == NANS_ALL_EQUAL || nans_equal == NANS_UNEQUAL, B2_ERR_INVALID_ARGUMENT, "invalid nan_equality");
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto s = static_cast<cudaStream_t>(stream);
  if (cols.empty() || cols[0].size == 0) { *out = make_column(B2_INT32, 0, false, s).release(); return B2_OK; }
  dbuf map;
  const int32_t m = distinct_map(cols, keep, nulls_equal, nans_equal, map, s);
  auto idx = make_column(B2_INT32, m, false, s);  // right-sized: the map has room for every input row
  if (m > 0) B2_CUDA_TRY(cudaMemcpyAsync(idx->data.ptr, map.ptr, sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToDevice, s));
  *out = idx.release();
  B2_TRY_END
}

}  // extern "C"

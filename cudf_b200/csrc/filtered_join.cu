// filtered_join.cu — left semi / anti join against a filter table built once (cudf::filtered_join:
// cpp/include/cudf/join/filtered_join.hpp, cpp/src/join/filtered_join/filtered_join.cu of the reference).
//
// Build: fj_build_kernel inserts every right key row into a DISTINCT set — a linear-probing table of 16-byte slots
// {packed key (or 64-bit row hash for keys wider than 8 bytes), representative right row, nullbits}, claimed with one
// 128-bit CAS (key_pack.cuh, the protocol of distinct_insert_kernel). A duplicate right key finds its slot and takes no
// second one, so probe chains stay short for duplicate-heavy filter tables. The table is sized up front from the right
// row count (more slots than rows: every chain ends on an empty slot), so construction needs no counters, no overflow
// signal and no read-back; it is fully stream-ordered.
// Probe: no kernel of its own. compact_kernel (compact.cuh) runs with contains_pred, which packs / hashes the left row,
// walks the slot chain with plain read-only loads until an empty slot or a hit, and keeps the row when found == semi. One
// kernel reads the left keys once, probes, ranks the kept rows and writes their ids in ascending order; one read-back per
// call, for the count. The ids are then copied into a right-sized INT32 column.
#include "common.cuh"
#include "compact.cuh"
#include "device_utils.cuh"
#include "key_pack.cuh"

#include <algorithm>
#include <cmath>

struct b2_filtered_join {
  std::vector<int32_t> right_types;
  int32_t right_rows = 0;
  bool nulls_unequal = false;
  bool wide          = false;  // keys wider than 8 bytes: a hit is confirmed against the right table's columns, which must
                               // outlive the object (the reference keeps a table_view of the right table too)
  b2::key_cols right_kc{};
  b2::dbuf right_kc_dev;       // a device copy of right_kc, read by the wide probe
  uint32_t mask = 0;
  b2::dbuf table;              // empty when the right table has no rows
};

namespace b2 {
namespace {

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)num_sms() * 16)); }

template <bool WIDE>
__device__ __forceinline__ void row_key(const key_cols& kc, int64_t r, uint64_t& key, uint32_t& nb)
{
  if constexpr (WIDE) hash_row_wide(kc, r, key, nb);
  else pack_row(kc, r, key, nb);
}

template <bool WIDE>
__global__ void __launch_bounds__(256) fj_build_kernel(key_cols kc, int64_t n, bool skip_nulls, slot_t* __restrict__ table,
                                                       uint32_t mask)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  slot_t empty;
  memset(&empty, 0xff, sizeof(empty));
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    uint64_t key;
    uint32_t nb;
    row_key<WIDE>(kc, r, key, nb);
    if (skip_nulls && nb) continue;  // nulls UNEQUAL: such a row matches no left row
    uint32_t i = slot_hash(key, nb, mask);
    while (true) {
      slot_t cur = load_slot_volatile(&table[i]);
      if (cur.row == -1) {
        cur = cas128(&table[i], empty, slot_t{key, (int32_t)r, nb});
        if (cur.row == -1) break;  // this row claimed the slot
      }
      if constexpr (WIDE) {
        if (cur.key == key && cur.nullbits == nb && rows_equal_wide(kc, r, kc, cur.row)) break;
      } else {
        if (cur.key == key && cur.nullbits == nb) break;
      }
      i = (i + 1) & mask;
    }
  }
}

// left row r has (semi) / has no (anti) equal row in the set
template <bool WIDE>
struct contains_pred {
  key_cols left;
  const key_cols* right;  // device memory, read only for wide keys (as a kernel parameter it made the probe spill)
  const slot_t* table;
  uint32_t mask;
  bool skip_nulls;
  bool semi;
  __device__ __forceinline__ bool operator()(int64_t r) const
  {
    uint64_t key;
    uint32_t nb;
    row_key<WIDE>(left, r, key, nb);
    bool found = false;
    if (!(skip_nulls && nb)) {
      uint32_t i = slot_hash(key, nb, mask);
      while (true) {
        const slot_t cur = load_slot(&table[i]);
        if (cur.row == -1) break;
        if (cur.key == key && cur.nullbits == nb) {
          if constexpr (WIDE) {
            if (rows_equal_wide(left, r, *right, cur.row)) { found = true; break; }
          } else {
            found = true;
            break;
          }
        }
        i = (i + 1) & mask;
      }
    }
    return found == semi;
  }
};

__global__ void __launch_bounds__(256) fj_sequence_kernel(int64_t n, int32_t* __restrict__ out)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (int32_t)i;
}

// Slots: the smallest power of two >= max(rows + 1, rows / load_factor), capped at 8x the smallest power of two above the
// row count and at 2^31 (slot indices are 32-bit). The cap bounds the memory a tiny load factor can ask for: 10M rows at
// 0.004 would otherwise take 2^32 slots (64 GB); 8x the rows keeps chains short while any cap > rows keeps a slot empty.
uint64_t set_slots(int64_t rows, double load_factor)
{
  uint64_t above = 1;
  while (above <= (uint64_t)rows) above <<= 1;
  const uint64_t cap = std::min<uint64_t>(above * 8, 1ull << 31);
  const double want  = std::max((double)rows + 1, std::ceil((double)rows / load_factor));
  uint64_t slots = 1;
  while (slots < cap && (double)slots < want) slots <<= 1;
  return slots;
}

b2_filtered_join* filtered_join_create(const std::vector<b2_column_view>& right, int32_t compare_nulls, double load_factor,
                                       cudaStream_t stream)
{
  B2_EXPECTS(load_factor > 0 && load_factor <= 1, B2_ERR_INVALID_ARGUMENT, "Invalid load factor: must be greater than 0 and at most 1.");
  B2_EXPECTS(compare_nulls == B2_NULLS_EQUAL || compare_nulls == B2_NULLS_UNEQUAL, B2_ERR_INVALID_ARGUMENT, "invalid null_equality");
  const key_cols kc = make_key_cols(right, true);
  auto fj = std::make_unique<b2_filtered_join>();
  for (const auto& c : right) fj->right_types.push_back(c.type_id);
  fj->right_rows    = right.empty() ? 0 : right[0].size;
  fj->nulls_unequal = compare_nulls == B2_NULLS_UNEQUAL;
  fj->wide          = keys_are_wide(right);
  fj->right_kc      = kc;
  if (fj->right_rows == 0) return fj.release();
  if (fj->wide) {
    fj->right_kc_dev = dbuf(sizeof(key_cols), stream);
    B2_CUDA_TRY(cudaMemcpyAsync(fj->right_kc_dev.ptr, &fj->right_kc, sizeof(key_cols), cudaMemcpyHostToDevice, stream));
  }
  const uint64_t slots = set_slots(fj->right_rows, load_factor);
  fj->mask  = (uint32_t)(slots - 1);
  fj->table = dbuf(slots * sizeof(slot_t), stream);
  B2_CUDA_TRY(cudaMemsetAsync(fj->table.ptr, 0xff, fj->table.bytes, stream));
  const int64_t n = fj->right_rows;
  prof_scope ps("filtered_join_build", stream);
  if (fj->wide)
    B2_LAUNCH((fj_build_kernel<true>), grid_for(n), 256, 0, stream, kc, n, fj->nulls_unequal, fj->table.as<slot_t>(), fj->mask);
  else
    B2_LAUNCH((fj_build_kernel<false>), grid_for(n), 256, 0, stream, kc, n, fj->nulls_unequal, fj->table.as<slot_t>(), fj->mask);
  return fj.release();
}

// filtered_join::semi_join / anti_join (filtered_join.cu:124-186): the early returns come before any check of the left
// table against the right one, as in the reference
column_ptr filtered_join_probe(const b2_filtered_join& fj, const std::vector<b2_column_view>& left, bool semi, cudaStream_t stream)
{
  const int32_t n = left.empty() ? 0 : left[0].size;
  if (n == 0 || (semi && fj.right_rows == 0)) return make_column(B2_INT32, 0, false, stream);
  if (fj.right_rows == 0) {  // anti join against an empty filter: every left row
    auto out = make_column(B2_INT32, n, false, stream);
    B2_LAUNCH(fj_sequence_kernel, grid_for(n), 256, 0, stream, (int64_t)n, out->data.as<int32_t>());
    return out;
  }
  // check_shape_compatibility of the reference: a column count or type mismatch is std::invalid_argument. (Its
  // numeric-only fast path raises cudf::logic_error for a count mismatch and checks no types; this one rule covers both.)
  B2_EXPECTS(left.size() == fj.right_types.size(), B2_ERR_INVALID_ARGUMENT, "Mismatch in number of columns to be joined on");
  for (size_t c = 0; c < left.size(); ++c)
    B2_EXPECTS(left[c].type_id == fj.right_types[c], B2_ERR_INVALID_ARGUMENT, "Mismatch in joining column data types");
  const key_cols lk = make_key_cols(left, true);
  dbuf map;
  int32_t m;
  if (fj.wide)
    m = compact(contains_pred<true>{lk, fj.right_kc_dev.as<key_cols>(), fj.table.as<slot_t>(), fj.mask, fj.nulls_unequal, semi},
                n, map, stream);
  else
    m = compact(contains_pred<false>{lk, nullptr, fj.table.as<slot_t>(), fj.mask, fj.nulls_unequal, semi}, n, map, stream);
  auto out = make_column(B2_INT32, m, false, stream);  // right-sized: the map has room for every left row
  if (m > 0) B2_CUDA_TRY(cudaMemcpyAsync(out->data.ptr, map.ptr, sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToDevice, stream));
  return out;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_filtered_join_create(const b2_table_view* right, int32_t compare_nulls, double load_factor, b2_stream stream,
                                  b2_filtered_join** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(right, cols);
  *out = filtered_join_create(cols, compare_nulls, load_factor, static_cast<cudaStream_t>(stream));
  B2_TRY_END
}

void b2_filtered_join_destroy(b2_filtered_join* fj) { delete fj; }

static b2_status filtered_join_call(const b2_filtered_join* fj, const b2_table_view* left, bool semi, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(fj && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(left, cols);
  *out = filtered_join_probe(*fj, cols, semi, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_filtered_join_semi_join(const b2_filtered_join* fj, const b2_table_view* left, b2_stream stream, b2_column** out)
{
  return filtered_join_call(fj, left, true, stream, out);
}

b2_status b2_filtered_join_anti_join(const b2_filtered_join* fj, const b2_table_view* left, b2_stream stream, b2_column** out)
{
  return filtered_join_call(fj, left, false, stream, out);
}

}  // extern "C"

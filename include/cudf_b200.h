/*
 * cudf_b200.h — flat C ABI of the H100-native hot path (sort / hash join / hash groupby /
 * scan / reduce / segmented reduce / gather / null-mask utilities).
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++ types, no torch types.
 * The reference (rapidsai/cudf) has no C ABI of its own; its boundary is the libcudf C++ API that
 * pylibcudf's .pxd files bind.  Every entry point below names the reference interface it replaces
 * (paths relative to the reference tree).  `include/cudf/ *.hpp` re-creates that C++ surface as
 * header-only wrappers over these functions; `cudf_b200/pylibcudf` is the Python twin.
 *
 * Conventions
 *  - All pointers inside views are DEVICE pointers (Arrow layout, fixed-width types only).
 *  - `b2_column_view` mirrors cudf::column_view (cpp/include/cudf/column/column_view.hpp:237-244):
 *    element i lives at data[(offset+i)], validity bit at bit (offset+i) of null_mask (LSB first,
 *    32-bit words, 1 = valid); null_mask may be NULL (all valid); null_count must be exact.
 *  - Every call is ordered on `stream` (a cudaStream_t passed as void*) and may return before the
 *    device work finishes, except where a size has to be read back (join size, groupby growth).
 *  - Outputs are library-owned handles released with the matching *_free function.
 *  - Return value: b2_status; on failure b2_last_error() holds a thread-local message.  The status
 *    maps 1:1 on the reference exception taxonomy (cpp/include/cudf/utilities/error.hpp:35-118):
 *      LOGIC -> cudf::logic_error, INVALID_ARGUMENT -> std::invalid_argument,
 *      DATA_TYPE -> cudf::data_type_error, OUT_OF_RANGE -> std::out_of_range,
 *      BAD_ALLOC -> std::bad_alloc, CUDA -> cudf::cuda_error.
 */
#ifndef CUDF_B200_H
#define CUDF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_API __attribute__((visibility("default")))

typedef void* b2_stream; /* cudaStream_t */

typedef enum b2_status {
  B2_OK                   = 0,
  B2_ERR_LOGIC            = 1,
  B2_ERR_INVALID_ARGUMENT = 2,
  B2_ERR_DATA_TYPE        = 3,
  B2_ERR_OUT_OF_RANGE     = 4,
  B2_ERR_BAD_ALLOC        = 5,
  B2_ERR_CUDA             = 6
} b2_status;

/* cudf::type_id values (cpp/include/cudf/types.hpp:183-216). Only fixed-width ids are accepted. */
enum {
  B2_EMPTY = 0, B2_INT8 = 1, B2_INT16 = 2, B2_INT32 = 3, B2_INT64 = 4,
  B2_UINT8 = 5, B2_UINT16 = 6, B2_UINT32 = 7, B2_UINT64 = 8,
  B2_FLOAT32 = 9, B2_FLOAT64 = 10, B2_BOOL8 = 11,
  B2_TIMESTAMP_DAYS = 12, B2_TIMESTAMP_SECONDS = 13, B2_TIMESTAMP_MILLISECONDS = 14,
  B2_TIMESTAMP_MICROSECONDS = 15, B2_TIMESTAMP_NANOSECONDS = 16,
  B2_DURATION_DAYS = 17, B2_DURATION_SECONDS = 18, B2_DURATION_MILLISECONDS = 19,
  B2_DURATION_MICROSECONDS = 20, B2_DURATION_NANOSECONDS = 21
};

/* cudf::order / null_order / null_policy / null_equality (types.hpp:99-150): bool enums. */
enum { B2_ASCENDING = 0, B2_DESCENDING = 1 };
enum { B2_NULL_AFTER = 0, B2_NULL_BEFORE = 1 };
enum { B2_NULL_EXCLUDE = 0, B2_NULL_INCLUDE = 1 };
enum { B2_NULLS_EQUAL = 0, B2_NULLS_UNEQUAL = 1 };
/* cudf::out_of_bounds_policy (cpp/include/cudf/copying.hpp:37-40) */
enum { B2_OOB_NULLIFY = 0, B2_OOB_DONT_CHECK = 1 };
/* cudf::mask_state (types.hpp:172-177) */
enum { B2_MASK_UNALLOCATED = 0, B2_MASK_UNINITIALIZED = 1, B2_MASK_ALL_VALID = 2, B2_MASK_ALL_NULL = 3 };
/* cudf::aggregation::Kind subset (cpp/include/cudf/aggregation.hpp:78-121), same numeric values. */
enum {
  B2_AGG_SUM = 0, B2_AGG_PRODUCT = 2, B2_AGG_MIN = 3, B2_AGG_MAX = 4,
  B2_AGG_COUNT_VALID = 5, B2_AGG_COUNT_ALL = 6, B2_AGG_SUM_OF_SQUARES = 9, B2_AGG_MEAN = 10, B2_AGG_M2 = 11,
  B2_AGG_VARIANCE = 12, B2_AGG_STD = 13, /* groupby only; ddof = 1 unless given with B2_AGG_WITH_DDOF */
  B2_AGG_ARGMAX = 16, B2_AGG_ARGMIN = 17 /* groupby only: INT32 row index of the extreme value (first row among ties) */
};
/* make_variance_aggregation(ddof) / make_std_aggregation(ddof) (aggregation.hpp:231-260): the kind word carries ddof */
#define B2_AGG_WITH_DDOF(kind, ddof) ((int32_t)(kind) | (1 << 30) | (((int32_t)(ddof) & 0xFFFF) << 8))
/* cudf::scan_type (cpp/include/cudf/reduction.hpp) */
enum { B2_SCAN_INCLUSIVE = 0, B2_SCAN_EXCLUSIVE = 1 };
/* JoinNoMatch sentinel (cpp/include/cudf/join/join.hpp:72) */
#define B2_JOIN_NO_MATCH INT32_MIN

typedef struct b2_column_view {
  int32_t         type_id;
  int32_t         size;
  const void*     data;
  const uint32_t* null_mask;
  int32_t         null_count;
  int32_t         offset;
} b2_column_view;

typedef struct b2_table_view {
  const b2_column_view* columns;
  int32_t               num_columns;
} b2_table_view;

typedef struct b2_column    b2_column;    /* owning cudf::column     (column.hpp:36-334)  */
typedef struct b2_table     b2_table;     /* owning cudf::table      (table.hpp:31-215)   */
typedef struct b2_scalar    b2_scalar;    /* owning numeric_scalar<T> (scalar/scalar.hpp) */
typedef struct b2_buffer    b2_buffer;    /* owning rmm::device_buffer                    */
typedef struct b2_hash_join b2_hash_join; /* cudf::hash_join         (join/hash_join.hpp) */
typedef struct b2_filtered_join b2_filtered_join;   /* cudf::filtered_join (join/filtered_join.hpp) */
typedef struct b2_groupby   b2_groupby;   /* cudf::groupby::groupby  (groupby.hpp)        */

/* cudf::groupby::aggregation_request (cpp/include/cudf/groupby.hpp:60-64) */
typedef struct b2_agg_request {
  b2_column_view values;
  const int32_t* kinds;     /* B2_AGG_* */
  int32_t        num_kinds;
} b2_agg_request;

/* ---- errors / runtime ------------------------------------------------------------------- */
B2_API const char* b2_last_error(void);
B2_API const char* b2_version(void);
/* Number of kernels this library has launched in this process (bench.py gpu_launches). */
B2_API uint64_t b2_kernel_launch_count(void);
/* Optional per-kernel-family timing with CUDA events on the caller's stream (off by default; the
 * NVTX-range analogue of CUDF_FUNC_RANGE, used by bench.py for the live roofline figure).
 * b2_profile_get synchronises the device and returns accumulated milliseconds and launch count. */
B2_API void      b2_profile_enable(int32_t on);
B2_API void      b2_profile_reset(void);
B2_API b2_status b2_profile_get(const char* name, double* total_ms, int64_t* launches);
/* same, restricted to the scopes that took at least `min_ms` (separates executed radix passes from skipped ones) */
B2_API b2_status b2_profile_get_over(const char* name, double min_ms, double* total_ms, int64_t* launches);
/* Trim the stream-ordered pool back to the driver (rmm pool release analogue). */
B2_API b2_status b2_trim_pool(void);

/* ---- owning handles --------------------------------------------------------------------- */
B2_API b2_status b2_column_view_of(const b2_column* col, b2_column_view* out);
B2_API void      b2_column_free(b2_column* col);
B2_API int32_t   b2_table_num_columns(const b2_table* tbl);
B2_API int32_t   b2_table_num_rows(const b2_table* tbl);
/* borrowed pointer, valid while the table lives */
B2_API const b2_column* b2_table_column(const b2_table* tbl, int32_t i);
/* cudf::table::release(): moves the columns out (caller frees each), table becomes empty */
B2_API b2_status b2_table_release(b2_table* tbl, b2_column** out_cols, int32_t capacity);
B2_API void      b2_table_free(b2_table* tbl);
B2_API void*     b2_buffer_data(const b2_buffer* buf);
B2_API size_t    b2_buffer_size(const b2_buffer* buf);
B2_API void      b2_buffer_free(b2_buffer* buf);
/* numeric_scalar<T>: value bytes are the native representation of type_id (<= 8 bytes). */
B2_API b2_status b2_scalar_create(int32_t type_id, const void* host_value, int32_t is_valid,
                                  b2_stream stream, b2_scalar** out);
B2_API int32_t     b2_scalar_type(const b2_scalar* s);
B2_API const void* b2_scalar_device_data(const b2_scalar* s);
/* synchronises `stream`; copies the value (<= 8 bytes) and validity to the host */
B2_API b2_status b2_scalar_get(const b2_scalar* s, b2_stream stream, void* host_value, int32_t* is_valid);
B2_API void      b2_scalar_free(b2_scalar* s);

/* ---- null masks: cpp/include/cudf/null_mask.hpp, cpp/src/bitmask/null_mask.cu ------------ */
B2_API size_t    b2_bitmask_allocation_size_bytes(int32_t number_of_bits);             /* null_mask.hpp:55 */
B2_API b2_status b2_create_null_mask(int32_t size, int32_t mask_state, b2_stream stream,
                                     b2_buffer** out);                                  /* null_mask.cu:48-86 */
B2_API b2_status b2_set_null_mask(uint32_t* bitmask, int32_t begin_bit, int32_t end_bit, int32_t valid,
                                  b2_stream stream);                                    /* null_mask.cu:339-404 */
B2_API b2_status b2_copy_bitmask(const uint32_t* mask, int32_t begin_bit, int32_t end_bit, b2_stream stream,
                                 b2_buffer** out);                                      /* null_mask.cu:409-560 */
B2_API b2_status b2_count_set_bits(const uint32_t* bitmask, int32_t start, int32_t stop, b2_stream stream,
                                   int32_t* out);                                       /* cudf::detail::count_set_bits */
B2_API b2_status b2_null_count(const uint32_t* bitmask, int32_t start, int32_t stop, b2_stream stream,
                                   int32_t* out);                                       /* cudf::null_count */
/* AND of the masks of all columns -> (mask, null_count); mask NULL when no column is nullable */
B2_API b2_status b2_bitmask_and(const b2_table_view* view, b2_stream stream, b2_buffer** out_mask,
                                int32_t* out_null_count);                               /* null_mask.cu:608-735 */

/* ---- gather: cpp/include/cudf/copying.hpp:81-86, cpp/include/cudf/detail/gather.cuh:627-675 */
B2_API b2_status b2_gather(const b2_table_view* source, const b2_column_view* gather_map, int32_t oob_policy,
                           b2_stream stream, b2_table** out);

/* ---- sort: cpp/include/cudf/sorting.hpp:44-163, cpp/src/sort/{sort,stable_sort}.cu -------- */
/* column_order / null_precedence: arrays of B2_ASCENDING.. / B2_NULL_AFTER.. of length n_order /
 * n_null_prec; 0 length = defaults (ASCENDING, BEFORE: sort_impl.cuh:56-57). */
B2_API b2_status b2_sorted_order(const b2_table_view* keys, const uint8_t* column_order, int32_t n_order,
                                 const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable,
                                 b2_stream stream, b2_column** out);
B2_API b2_status b2_sort(const b2_table_view* input, const uint8_t* column_order, int32_t n_order,
                         const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable,
                         b2_stream stream, b2_table** out);
B2_API b2_status b2_sort_by_key(const b2_table_view* values, const b2_table_view* keys,
                                const uint8_t* column_order, int32_t n_order,
                                const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable,
                                b2_stream stream, b2_table** out);

/* cudf::{stable_,}segmented_sorted_order / segmented_sort_by_key (sorting.hpp:232-366): segment_offsets is an INT32
 * column of start offsets (the last entry ends the last segment); rows outside [offsets[0], offsets[last]) keep their
 * place; fewer than two offsets sort nothing; a non-INT32 offsets column -> LOGIC error. */
B2_API b2_status b2_segmented_sorted_order(const b2_table_view* keys, const b2_column_view* segment_offsets,
                                           const uint8_t* column_order, int32_t n_order,
                                           const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable,
                                           b2_stream stream, b2_column** out);
B2_API b2_status b2_segmented_sort_by_key(const b2_table_view* values, const b2_table_view* keys,
                                          const b2_column_view* segment_offsets, const uint8_t* column_order,
                                          int32_t n_order, const uint8_t* null_precedence, int32_t n_null_prec,
                                          int32_t stable, b2_stream stream, b2_table** out);
/* cudf::top_k / top_k_order (sorting.hpp:370-416, top_k.cu:100-170): the k first rows of the stable sorted order
 * (nulls last for ASCENDING, first for DESCENDING); k >= size returns all rows; k < 0 -> INVALID_ARGUMENT. */
B2_API b2_status b2_top_k(const b2_column_view* col, int32_t k, int32_t topk_order, b2_stream stream, b2_column** out);
B2_API b2_status b2_top_k_order(const b2_column_view* col, int32_t k, int32_t topk_order, b2_stream stream,
                                b2_column** out);
/* cudf::rank (sorting.hpp:165-230, cpp/src/sort/rank.cu:236-356). method = cudf::rank_method (0 FIRST, 1 AVERAGE,
 * 2 MIN, 3 MAX, 4 DENSE); the result is FLOAT64 for AVERAGE or percentage, INT32 otherwise; under
 * null_handling = EXCLUDE the result carries the input's validity; percentage divides by the row count (DENSE: by
 * the number of distinct values). */
B2_API b2_status b2_rank(const b2_column_view* input, int32_t method, int32_t column_order, int32_t null_handling,
                         int32_t null_precedence, int32_t percentage, b2_stream stream, b2_column** out);

/* ---- hash join: cpp/include/cudf/join/join.hpp:127-249, join/hash_join.hpp ---------------- */
/* Results are two INT32 columns of equal length (cudf returns device_uvector<size_type>), row
 * order unspecified (join.hpp:130-136). */
B2_API b2_status b2_inner_join(const b2_table_view* left_keys, const b2_table_view* right_keys,
                               int32_t compare_nulls, b2_stream stream, b2_column** out_left,
                               b2_column** out_right);
B2_API b2_status b2_left_join(const b2_table_view* left_keys, const b2_table_view* right_keys,
                              int32_t compare_nulls, b2_stream stream, b2_column** out_left,
                              b2_column** out_right);
B2_API b2_status b2_full_join(const b2_table_view* left_keys, const b2_table_view* right_keys,
                              int32_t compare_nulls, b2_stream stream, b2_column** out_left,
                              b2_column** out_right);
/* hash_join(build, has_nulls, compare_nulls, load_factor, stream): hash_join.hpp ctor #2.
 * has_nulls < 0 = derive from the build table (ctor #1). load_factor outside (0,1] ->
 * INVALID_ARGUMENT (cpp/tests/join/join_tests.cpp:346-366). */
B2_API b2_status b2_hash_join_create(const b2_table_view* build, int32_t has_nulls, int32_t compare_nulls,
                                     double load_factor, b2_stream stream, b2_hash_join** out);
B2_API void      b2_hash_join_destroy(b2_hash_join* hj);
/* has_output_size = 0 -> the size is computed (std::optional<size_t> output_size = nullopt) */
B2_API b2_status b2_hash_join_inner_join(const b2_hash_join* hj, const b2_table_view* probe,
                                         int32_t has_output_size, size_t output_size, b2_stream stream,
                                         b2_column** out_left, b2_column** out_right);
B2_API b2_status b2_hash_join_left_join(const b2_hash_join* hj, const b2_table_view* probe,
                                        int32_t has_output_size, size_t output_size, b2_stream stream,
                                        b2_column** out_left, b2_column** out_right);
B2_API b2_status b2_hash_join_full_join(const b2_hash_join* hj, const b2_table_view* probe,
                                        int32_t has_output_size, size_t output_size, b2_stream stream,
                                        b2_column** out_left, b2_column** out_right);
B2_API b2_status b2_hash_join_inner_join_size(const b2_hash_join* hj, const b2_table_view* probe,
                                              b2_stream stream, size_t* out);
B2_API b2_status b2_hash_join_left_join_size(const b2_hash_join* hj, const b2_table_view* probe,
                                             b2_stream stream, size_t* out);
B2_API b2_status b2_hash_join_full_join_size(const b2_hash_join* hj, const b2_table_view* probe,
                                             b2_stream stream, size_t* out);

/* hash_join::{inner,left,full}_join_match_context (hash_join.hpp:254-330, join.hpp:81-125): per probe row, the
 * number of matching build rows as an INT32 column of probe.num_rows (join_kind: 0 inner, 1 left, 2 full; for
 * left / full a row without a match counts 1 — its null-placeholder output row). Golden: join_tests.cpp:2339-2527. */
B2_API b2_status b2_hash_join_match_counts(const b2_hash_join* hj, const b2_table_view* probe, int32_t join_kind,
                                           b2_stream stream, b2_column** out_counts);
/* hash_join::partitioned_{inner,left,full}_join (hash_join.hpp:331-411): join rows [left_start, left_end) of the
 * probe table given the match counts of the WHOLE probe table (from b2_hash_join_match_counts with the same
 * join_kind). Left indices are relative to the whole probe table. join_kind 2 does not append the unmatched build
 * rows: b2_hash_join_finalize_full_join does. Bounds outside [0, num_rows] -> INVALID_ARGUMENT. */
B2_API b2_status b2_hash_join_partitioned_join(const b2_hash_join* hj, const b2_table_view* probe,
                                               const b2_column_view* match_counts, int32_t left_start,
                                               int32_t left_end, int32_t join_kind, b2_stream stream,
                                               b2_column** out_left, b2_column** out_right);
/* hash_join::finalize_partitioned_full_join (hash_join.hpp:413-440): concatenates the per-partition index pairs and
 * appends (JoinNoMatch, r) for every build row r that no partition matched. */
B2_API b2_status b2_hash_join_finalize_full_join(const b2_column_view* left_partials,
                                                 const b2_column_view* right_partials, int32_t num_partials,
                                                 int32_t left_table_num_rows, int32_t right_table_num_rows,
                                                 b2_stream stream, b2_column** out_left, b2_column** out_right);

/* ---- semi / anti join: cpp/include/cudf/join/filtered_join.hpp, cpp/src/join/filtered_join/filtered_join.cu ---------------
 * The right (filter) table's key rows form a distinct set built once; semi_join returns the INT32 indices of the left rows
 * equal to some right row, anti_join those equal to none, both strictly ascending.  Row equality is the hash join's (NaN ==
 * NaN, -0 == +0); compare_nulls = null_equality (0 EQUAL: null == null; 1 UNEQUAL: a row with a null key matches nothing,
 * so it is in the anti result).  semi_join of an empty side is empty; anti_join of an empty left side is empty and against
 * an empty right side is 0..n-1.  load_factor outside (0, 1] -> INVALID_ARGUMENT (the reference's default is 0.5); the set
 * has the smallest power of two >= max(rows + 1, rows / load_factor) slots of 16 bytes, at most 8x the smallest power of
 * two above the row count and at most 2^31.  Key column count or type differing from the right table's ->
 * INVALID_ARGUMENT; more than 8 key columns -> INVALID_ARGUMENT; a non-fixed-width column -> DATA_TYPE.  The object is
 * immutable: probes may run concurrently from several threads / streams once construction has completed on its stream.
 * With keys wider than 8 bytes the right table's memory must outlive the object. */
B2_API b2_status b2_filtered_join_create(const b2_table_view* right, int32_t compare_nulls, double load_factor,
                                         b2_stream stream, b2_filtered_join** out);
B2_API void      b2_filtered_join_destroy(b2_filtered_join* fj);
B2_API b2_status b2_filtered_join_semi_join(const b2_filtered_join* fj, const b2_table_view* left, b2_stream stream,
                                            b2_column** out);
B2_API b2_status b2_filtered_join_anti_join(const b2_filtered_join* fj, const b2_table_view* left, b2_stream stream,
                                            b2_column** out);

/* ---- groupby: cpp/include/cudf/groupby.hpp:121-125,181-184, cpp/src/groupby/groupby.cu ----- */
B2_API b2_status b2_groupby_create(const b2_table_view* keys, int32_t null_handling, int32_t keys_are_sorted,
                                   const uint8_t* column_order, int32_t n_order,
                                   const uint8_t* null_precedence, int32_t n_null_prec, b2_groupby** out);
B2_API void      b2_groupby_destroy(b2_groupby* gb);
/* aggregate(): out_keys = distinct key rows; out_results = one column per (request, kind) in
 * request-major order (aggregation_result::results flattened). Row order arbitrary (groupby.hpp:148). */
B2_API b2_status b2_groupby_aggregate(b2_groupby* gb, const b2_agg_request* requests, int32_t num_requests,
                                      b2_stream stream, b2_table** out_keys, b2_table** out_results);
/* scan(): rows in sorted key order (cpp/src/groupby/sort/scan.cpp) */
B2_API b2_status b2_groupby_scan(b2_groupby* gb, const b2_agg_request* requests, int32_t num_requests,
                                 b2_stream stream, b2_table** out_keys, b2_table** out_results);

/* ---- reduce / scan / segmented reduce: cpp/include/cudf/reduction.hpp ---------------------- */
/* init may be NULL (std::nullopt). */
B2_API b2_status b2_reduce(const b2_column_view* col, int32_t agg_kind, int32_t output_type_id,
                           const b2_scalar* init, b2_stream stream, b2_scalar** out);
B2_API b2_status b2_segmented_reduce(const b2_column_view* values, const int32_t* offsets, int32_t num_offsets,
                                     int32_t agg_kind, int32_t output_type_id, int32_t null_handling,
                                     const b2_scalar* init, b2_stream stream, b2_column** out);
B2_API b2_status b2_scan(const b2_column_view* col, int32_t agg_kind, int32_t scan_type, int32_t null_handling,
                         b2_stream stream, b2_column** out);

/* ---- sharded path helpers (no libcudf equivalent on one GPU; role of cudf::hash_partition,
 *      cpp/include/cudf/partitioning.hpp:103-145, and of cudf_polars' sort splitters) ----------- */
/* Stable partition of `input` rows into num_partitions buckets. out_offsets (host int32[P+1]).
 * mode 0: bucket = number of splitters <= key (range partition on the single key column `keys`,
 *         splitters = device array of P-1 ascending keys of the same type)
 * mode 1: bucket = mix64(key bits) % P (hash partition)                                          */
B2_API b2_status b2_partition(const b2_table_view* input, const b2_column_view* keys, int32_t mode,
                              const void* splitters, int32_t num_partitions, b2_stream stream,
                              b2_table** out, int32_t* out_offsets);

/* cudf::hash_partition(input, keys, num_partitions, hash_function, seed) — cpp/include/cudf/partitioning.hpp:103-145,
 * cpp/src/partitioning/partitioning.cu:875-945.  Row hash as in libcudf (hash_function 1 = HASH_MURMUR3: MurmurHash3_x86_32
 * per column with `seed`, floats normalised, null = UINT32_MAX, columns folded with hash_combine; 0 = HASH_IDENTITY on
 * integral keys), partition = hash % num_partitions: a row lands in the same partition as under libcudf, so the output
 * interoperates with dask_cudf / rapidsmpf style shuffles.  out_offsets: host int32[num_partitions + 1].  Rows keep their
 * input order inside a partition.  Up to 256 partitions take the tile-based partition kernels, more go through a stable
 * radix order of the 32-bit partition ids; zero key columns / rows give an empty result. */
B2_API b2_status b2_hash_partition(const b2_table_view* input, const b2_table_view* keys, int32_t num_partitions,
                                   int32_t hash_function, uint32_t seed, b2_stream stream, b2_table** out, int32_t* out_offsets);

/* cudf::partition(t, partition_map, num_partitions) for any partition count (cpp/include/cudf/partitioning.hpp:58-101): the
 * integer map names each row's partition; stable order of the map values + fused gather. out_offsets: int32[P + 1]. */
B2_API b2_status b2_partition_by_map(const b2_table_view* input, const b2_column_view* partition_map, int32_t num_partitions,
                                     b2_stream stream, b2_table** out, int32_t* out_offsets);

/* ---- stream compaction: cpp/include/cudf/stream_compaction.hpp, cpp/src/stream_compaction/*.  Fixed-width keys, at most
 *      8 key columns.  keep = cudf::duplicate_keep_option (0 ANY, 1 FIRST, 2 LAST, 3 NONE); nulls_equal = null_equality
 *      (0 EQUAL, 1 UNEQUAL); nans_equal = cudf::nan_equality (0 ALL_EQUAL, 1 UNEQUAL).  A key index outside the table is
 *      OUT_OF_RANGE (table_view::select). -------------------------------------------------------------------------------- */
enum { B2_KEEP_ANY = 0, B2_KEEP_FIRST = 1, B2_KEEP_LAST = 2, B2_KEEP_NONE = 3 };
enum { B2_NANS_ALL_EQUAL = 0, B2_NANS_UNEQUAL = 1 };
/* cudf::apply_boolean_mask (deletion = 0; apply_boolean_mask.cu:22-117) / cudf::apply_deletion_mask (deletion = 1): keeps
 * row i when mask[i] is valid and true (false), in input order.  The mask must be BOOL8 (LOGIC) and, when the table has
 * rows, have as many rows (LOGIC); an empty mask gives an empty table of the input's types. */
B2_API b2_status b2_apply_boolean_mask(const b2_table_view* input, const b2_column_view* mask, int32_t deletion, b2_stream stream,
                                       b2_table** out);
/* cudf::drop_nulls (drop_nulls.cu:57-66): keeps the rows with at least keep_threshold valid key columns.  No keys, no rows
 * or no nulls in the keys: a copy of the input. */
B2_API b2_status b2_drop_nulls(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep_threshold,
                               b2_stream stream, b2_table** out);
/* cudf::drop_nans (drop_nans.cu:78-100): keeps the rows with at least keep_threshold non-NaN key columns (a null is not
 * NaN).  A non-float key column is LOGIC. */
B2_API b2_status b2_drop_nans(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep_threshold,
                              b2_stream stream, b2_table** out);
/* cudf::unique (unique.cu:42-121): drops consecutive duplicate key rows (ANY = FIRST; NONE drops every row with an equal
 * neighbour); NaN == NaN, -0 == +0. */
B2_API b2_status b2_unique(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep, int32_t nulls_equal,
                           b2_stream stream, b2_table** out);
/* cudf::distinct / cudf::stable_distinct (distinct.cu:76-200, stable_distinct.cu): one row per set of equal key rows (NONE:
 * only the rows whose key occurs once).  Both return the rows in input order; `stable` is accepted for symmetry. */
B2_API b2_status b2_distinct(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep, int32_t nulls_equal,
                             int32_t nans_equal, int32_t stable, b2_stream stream, b2_table** out);
/* cudf::distinct_indices (distinct.cu:76-200, 185-200): INT32 indices of the kept rows over all columns, ascending. */
B2_API b2_status b2_distinct_indices(const b2_table_view* input, int32_t keep, int32_t nulls_equal, int32_t nans_equal,
                                     b2_stream stream, b2_column** out);

/* ---- binary operations: cpp/include/cudf/binaryop.hpp, cpp/src/binaryop/binaryop.cpp, cpp/src/binaryop/compiled/* -----------
 * out[i] = op(lhs[i], rhs[i]) over fixed-width columns, or a column and a scalar (a scalar operand is the same value in every
 * row).  The operator values are cudf::binary_operator's.  Types: INT8..UINT64, FLOAT32, FLOAT64 and BOOL8 in any combination
 * of lhs, rhs and output; a timestamp or duration operand only against the same type id, for the six comparisons,
 * NULL_EQUALS / NULL_NOT_EQUALS (output BOOL8) and NULL_MAX / NULL_MIN (output of the operands' type), on the storage integers.
 *  - Compute type C = std::common_type<out, lhs, rhs> (for a chrono comparison: the operands' storage type).  The value is
 *    Out(op(C(x), C(y))) with C++ semantics: integers narrower than 32 bits are computed as int and wrap on the cast to Out,
 *    signed overflow wraps; TRUE_DIV, POW, LOG_BASE, ATAN2 and PYMOD on floats compute in double; FLOOR_DIV rounds toward
 *    -inf for integers and is floor(x / y) for floats; MOD on floats is fmod; INT_POW is exponentiation by squaring in C and 0
 *    for a negative exponent; comparisons and logical operators write BOOL8.
 *  - Validity: the AND of the operands' (a null scalar makes every row null), except for the null-aware operators, whose
 *    output always has a mask: NULL_EQUALS(null, null) = true, NULL_EQUALS(null, x) = false, NULL_NOT_EQUALS its negation,
 *    all valid; NULL_MAX / NULL_MIN take the valid operand, null when both are; NULL_LOGICAL_AND(null, false) = false,
 *    NULL_LOGICAL_OR(null, true) = true, otherwise null when an operand is.  The output has a mask when a row can be null;
 *    null_count is exact.  An empty column gives an empty column of the output type.
 *  - Undefined values (as in the reference; no result depends on them): integer division or modulo by zero and INT_MIN / -1
 *    (DIV, FLOOR_DIV, MOD, PMOD, PYMOD), shifts by a negative amount or at / beyond the width of the promoted left operand,
 *    float-to-integer conversions of NaN or of values whose integer part the output type cannot hold, integer-only operators
 *    (INT_POW, shifts, bitwise) whose C is a float because the output is (here computed in std::common_type<lhs, rhs>), and
 *    values under null bits.
 *  - Errors: column sizes differ -> INVALID_ARGUMENT; a type id outside cudf::type_id -> LOGIC; GENERIC_BINARY, an operator
 *    outside the enum, decimal / string / nested types and every other unsupported combination -> DATA_TYPE.
 *  - The scalar forms read the scalar's validity back (one synchronisation of `stream`), as the reference does; the column
 *    form does not synchronise. */
enum {
  B2_BINOP_ADD = 0, B2_BINOP_SUB = 1, B2_BINOP_MUL = 2, B2_BINOP_DIV = 3, B2_BINOP_TRUE_DIV = 4, B2_BINOP_FLOOR_DIV = 5,
  B2_BINOP_MOD = 6, B2_BINOP_PMOD = 7, B2_BINOP_PYMOD = 8, B2_BINOP_POW = 9, B2_BINOP_INT_POW = 10, B2_BINOP_LOG_BASE = 11,
  B2_BINOP_ATAN2 = 12, B2_BINOP_SHIFT_LEFT = 13, B2_BINOP_SHIFT_RIGHT = 14, B2_BINOP_SHIFT_RIGHT_UNSIGNED = 15,
  B2_BINOP_BITWISE_AND = 16, B2_BINOP_BITWISE_OR = 17, B2_BINOP_BITWISE_XOR = 18, B2_BINOP_LOGICAL_AND = 19,
  B2_BINOP_LOGICAL_OR = 20, B2_BINOP_EQUAL = 21, B2_BINOP_NOT_EQUAL = 22, B2_BINOP_LESS = 23, B2_BINOP_GREATER = 24,
  B2_BINOP_LESS_EQUAL = 25, B2_BINOP_GREATER_EQUAL = 26, B2_BINOP_NULL_EQUALS = 27, B2_BINOP_NULL_NOT_EQUALS = 28,
  B2_BINOP_NULL_MAX = 29, B2_BINOP_NULL_MIN = 30, B2_BINOP_GENERIC_BINARY = 31, B2_BINOP_NULL_LOGICAL_AND = 32,
  B2_BINOP_NULL_LOGICAL_OR = 33, B2_BINOP_INVALID_BINARY = 34
};
B2_API b2_status b2_binary_operation(const b2_column_view* lhs, const b2_column_view* rhs, int32_t op, int32_t out_type,
                                     b2_stream stream, b2_column** out);
B2_API b2_status b2_binary_operation_cs(const b2_column_view* lhs, const b2_scalar* rhs, int32_t op, int32_t out_type,
                                        b2_stream stream, b2_column** out);
B2_API b2_status b2_binary_operation_sc(const b2_scalar* lhs, const b2_column_view* rhs, int32_t op, int32_t out_type,
                                        b2_stream stream, b2_column** out);
/* cudf::binops::is_supported_operation: *result = 1 when the call above accepts (out, lhs, rhs, op); type ids outside
 * cudf::type_id -> LOGIC. */
B2_API b2_status b2_binary_is_supported_operation(int32_t out_type, int32_t lhs_type, int32_t rhs_type, int32_t op,
                                                  int32_t* result);

/* ---- unary operations and casts: cpp/include/cudf/unary.hpp, cpp/src/unary/{math_ops,cast_ops,nan_ops,null_ops}.cu -----------
 * One elementwise pass over a fixed-width column.  The operator values are cudf::unary_operator's.  T is the input's type.
 * b2_unary_operation:
 *  - SIN .. ARCTANH, EXP, LOG, SQRT, CBRT, CEIL, FLOOR, ABS: INT8..UINT64, FLOAT32, FLOAT64, BOOL8 -> T.  FLOAT32 computes in
 *    float, FLOAT64 in double, every integer type and BOOL8 in double and converts back to T (BOOL8: nonzero -> true).  No
 *    fast-math: SQRT is correctly rounded, subnormals are kept.  ABS: signed integers abs() after integral promotion (INT8 -128
 *    stays -128), unsigned integers and BOOL8 unchanged, floats fabs().
 *  - RINT: FLOAT32, FLOAT64 -> T, half to even.
 *  - BIT_COUNT: integer types and BOOL8 -> INT32, the popcount of the same-width unsigned value (BOOL8: 0 / 1).
 *  - BIT_INVERT: integer types and BOOL8 -> T, ~x after promotion (BOOL8: every valid row true).
 *  - NOT: INT8..BOOL8 -> BOOL8, x == 0 (NaN -> false, -0.0 -> true).
 *  - NEGATE: signed integers, floats and every DURATION -> T, -x after promotion (floats flip the sign of +-0 and NaN).
 * b2_cast (out_type any fixed-width id):
 *  - numeric <-> numeric, BOOL8 included: static_cast (float -> integer truncates toward zero; -> BOOL8 is x != 0, NaN -> true);
 *  - timestamp / duration <-> timestamp / duration: cuda::std::chrono::floor, ticks converted toward -inf in int64 and then
 *    narrowed to the target's rep (int32 for DAYS, int64 otherwise);
 *  - numeric -> duration: rep(x), a tick count with no unit scaling; duration -> numeric: To(count);
 *  - a same-type cast is a copy.
 * Null rows: the output has a mask exactly when the input has one (a copy of it, at offset 0), and the input's null_count.
 * An empty input gives an empty column of the output type; b2_unary_operation then checks no type (RINT of an empty INT32
 * column is an empty INT32 column).  No call synchronises.
 * Undefined values (as in the reference; no result depends on them): float -> integer conversions of NaN or of a value whose
 * truncation the target cannot hold (b2_cast, and the integer-typed results of the math operators: EXP of INT8 10, CEIL of
 * INT64 near 2^63); ABS / NEGATE of INT32_MIN, INT64_MIN and the minimum duration; chrono up-casts that overflow int64 and
 * down-casts whose result the int32 DAYS rep cannot hold; values under null bits.
 * Errors: an unsupported (op, type) pair or an op outside the enum -> LOGIC; decimal, dictionary, string and nested inputs ->
 * DATA_TYPE (the reference computes decimal ABS / CEIL / FLOOR / NEGATE; this library holds no decimal column).  b2_cast:
 * timestamp <-> numeric -> LOGIC, even on an empty column; a decimal source or target -> DATA_TYPE; any other target that is
 * not fixed-width -> LOGIC. */
enum {
  B2_UNARY_SIN = 0, B2_UNARY_COS = 1, B2_UNARY_TAN = 2, B2_UNARY_ARCSIN = 3, B2_UNARY_ARCCOS = 4, B2_UNARY_ARCTAN = 5,
  B2_UNARY_SINH = 6, B2_UNARY_COSH = 7, B2_UNARY_TANH = 8, B2_UNARY_ARCSINH = 9, B2_UNARY_ARCCOSH = 10, B2_UNARY_ARCTANH = 11,
  B2_UNARY_EXP = 12, B2_UNARY_LOG = 13, B2_UNARY_SQRT = 14, B2_UNARY_CBRT = 15, B2_UNARY_CEIL = 16, B2_UNARY_FLOOR = 17,
  B2_UNARY_ABS = 18, B2_UNARY_RINT = 19, B2_UNARY_BIT_COUNT = 20, B2_UNARY_BIT_INVERT = 21, B2_UNARY_NOT = 22,
  B2_UNARY_NEGATE = 23
};
B2_API b2_status b2_unary_operation(const b2_column_view* input, int32_t op, b2_stream stream, b2_column** out);
B2_API b2_status b2_cast(const b2_column_view* input, int32_t out_type, b2_stream stream, b2_column** out);
/* cudf::is_supported_cast: *result = 1 exactly when b2_cast accepts (from, to).  It equals the reference's answer on every pair
 * of INT8..DURATION_NANOSECONDS; a decimal pair is 0 here (the reference supports decimal casts).  Type ids outside
 * cudf::type_id -> LOGIC. */
B2_API b2_status b2_is_supported_cast(int32_t from_type, int32_t to_type, int32_t* result);
/* cudf::is_null / is_valid: a BOOL8 column without a mask, from the input's validity alone (any fixed-width type). */
B2_API b2_status b2_is_null(const b2_column_view* input, b2_stream stream, b2_column** out);
B2_API b2_status b2_is_valid(const b2_column_view* input, b2_stream stream, b2_column** out);
/* cudf::is_nan / is_not_nan: FLOAT32 / FLOAT64 only (any other type -> LOGIC, even empty); a BOOL8 column without a mask, a
 * null row is_nan = false and is_not_nan = true. */
B2_API b2_status b2_is_nan(const b2_column_view* input, b2_stream stream, b2_column** out);
B2_API b2_status b2_is_not_nan(const b2_column_view* input, b2_stream stream, b2_column** out);

/* ---- replacement: cpp/include/cudf/replace.hpp, cpp/src/replace/{nulls,nans,replace,clamp}.cu -------------------------------
 * One pass over a fixed-width column (INT8..DURATION_NANOSECONDS).  "A copy" is a new column with the input view's values, its
 * mask (realigned to offset 0) when it has one, and its null count.  An empty input gives an empty column (find_and_replace_all,
 * clamp, normalize: a copy) after the checks listed below.  Where the output's mask is computed, its null count is counted on
 * the device (the column resolves it on first use); only the scalar forms of replace_nulls and clamp synchronise, to read the
 * scalars' validity.
 * b2_replace_nulls: out[i] = valid(in[i]) ? in[i] : replacement[i].  The output has a mask exactly when the replacement has
 *   nulls.  An input without nulls gives a copy.  Errors: types differ -> DATA_TYPE; sizes differ -> LOGIC.
 * b2_replace_nulls_scalar: null rows take the scalar; the output has no mask.  An input without nulls or a null scalar gives a
 *   copy (with no type check, as in the reference); otherwise types differ -> DATA_TYPE.
 * b2_replace_nulls_policy: PRECEDING: a null row takes the nearest valid value before it; FOLLOWING: after it.  A leading
 *   (PRECEDING) or trailing (FOLLOWING) null run stays null.  An input with nulls gives an output with a mask whose null count
 *   is that run's length; an input without nulls gives a copy.  A policy outside the enum -> LOGIC.
 * b2_replace_nans / _scalar: FLOAT32 / FLOAT64 (any other type -> LOGIC, also empty).  A NaN row (valid) takes the
 *   replacement's value and validity; a null row stays null.  The output has a mask when the input has nulls or the replacement
 *   has a mask (the scalar form: always).  Sizes or types differ -> LOGIC.
 * b2_find_and_replace_all: rows equal (C++ ==: -0.0 == +0.0, NaN equals nothing) to values_to_replace[j] take
 *   replacement_values[j], the first such j among duplicates; a null replacement nulls the row; null rows stay null.  The output
 *   has a mask exactly when the input or replacement_values has nulls.  Errors: sizes of the two value columns differ -> LOGIC;
 *   any type differs -> DATA_TYPE; values_to_replace has nulls -> LOGIC.  An empty argument gives a copy.
 * b2_clamp: x < lo -> lo_replace, x > hi -> hi_replace (C++ < and >: NaN is never clamped, -0.0 is not below +0.0); a null lo
 *   or hi bound is not applied.  The output's mask is a copy of the input's.  Errors, in order: lo / hi, lo_replace /
 *   hi_replace or lo / lo_replace types differ -> DATA_TYPE; both bounds null or an empty input -> a copy; a valid bound with a
 *   null replacement -> LOGIC; input and lo types differ -> DATA_TYPE.  cudf::clamp(input, lo, hi) passes lo and hi as their
 *   own replacements.
 * b2_normalize_nans_and_zeros (/_inplace: over the view's own data): every NaN becomes quiet_NaN()'s bit pattern and -0.0
 *   becomes +0.0; the mask and null count are the input's.  FLOAT32 / FLOAT64 only, else LOGIC (an empty input: a copy / no-op).
 * Undefined values (as in the reference; no result depends on them): values under null bits.
 * Decimal, dictionary, string and nested inputs -> DATA_TYPE (this library holds no such column). */
enum { B2_REPLACE_PRECEDING = 0, B2_REPLACE_FOLLOWING = 1 };
B2_API b2_status b2_replace_nulls(const b2_column_view* input, const b2_column_view* replacement, b2_stream stream, b2_column** out);
B2_API b2_status b2_replace_nulls_scalar(const b2_column_view* input, const b2_scalar* replacement, b2_stream stream, b2_column** out);
B2_API b2_status b2_replace_nulls_policy(const b2_column_view* input, int32_t policy, b2_stream stream, b2_column** out);
B2_API b2_status b2_replace_nans(const b2_column_view* input, const b2_column_view* replacement, b2_stream stream, b2_column** out);
B2_API b2_status b2_replace_nans_scalar(const b2_column_view* input, const b2_scalar* replacement, b2_stream stream, b2_column** out);
B2_API b2_status b2_find_and_replace_all(const b2_column_view* input, const b2_column_view* values_to_replace,
                                         const b2_column_view* replacement_values, b2_stream stream, b2_column** out);
B2_API b2_status b2_clamp(const b2_column_view* input, const b2_scalar* lo, const b2_scalar* lo_replace, const b2_scalar* hi,
                          const b2_scalar* hi_replace, b2_stream stream, b2_column** out);
B2_API b2_status b2_normalize_nans_and_zeros(const b2_column_view* input, b2_stream stream, b2_column** out);
B2_API b2_status b2_normalize_nans_and_zeros_inplace(const b2_column_view* in_out, b2_stream stream);

/* Two-phase form of b2_partition for the fused partition + exchange: the plan holds the bucket id and the
 * stable in-bucket rank of every row; out_counts[b] = rows of bucket b.  b2_partition_scatter then writes one
 * fixed-width column straight to P destination base addresses — local buffers or PEER device memory mapped with
 * b2_ipc_open — so that the all-to-all exchange happens inside the scatter kernel over NVLink
 * (dest_ptrs[b] = address of bucket b's first row; host array of P device pointers). */
typedef struct b2_partition_plan b2_partition_plan;
B2_API b2_status b2_partition_plan_create(const b2_column_view* keys, int32_t mode, const void* splitters,
                                          int32_t num_partitions, b2_stream stream, b2_partition_plan** out,
                                          int64_t* out_counts);
B2_API b2_status b2_partition_scatter(const b2_partition_plan* plan, const b2_column_view* column,
                                      void* const* dest_ptrs, b2_stream stream);
/* EXPERIMENTAL variant of b2_partition_scatter: stages per-destination runs of a 4096-row tile in shared memory
 * before the (remote) stores; compiled in round 1 but not yet validated on hardware and not used by default. */
B2_API b2_status b2_partition_scatter_staged(const b2_partition_plan* plan, const b2_column_view* column,
                                             void* const* dest_ptrs, b2_stream stream);
B2_API void      b2_partition_plan_free(b2_partition_plan* plan);
/* Range partition fused into ONE one-sweep pass whose digit is the bucket (number of splitters <= key): first the bucket counts of
 * this rank's rows, then — after the ranks exchanged their counts — a stable pass that writes bucket b's keys (and optionally one
 * 4- / 8-byte payload column) to key_dst[b] / val_dst[b], local or peer memory (host arrays of num_partitions device pointers: the
 * address of THIS rank's first row of bucket b). One null-free 8-byte integer-like key column; splitters = device array of P - 1
 * ascending keys of the column's type. The sharded sort's partition + exchange (SURVEY §8e: "fuse with the first radix pass").
 * splitters == NULL selects a HASH partition instead (bucket = high-multiply of a 64-bit mix of the key by num_partitions; the
 * same function in both calls and on every rank): the sharded join's shuffle. */
B2_API b2_status b2_range_partition_counts(const b2_column_view* keys, const void* splitters, int32_t num_partitions, b2_stream stream,
                                           int64_t* out_counts);
B2_API b2_status b2_range_partition_scatter(const b2_column_view* keys, const b2_column_view* values, const void* splitters,
                                            int32_t num_partitions, void* const* key_dst, void* const* val_dst, b2_stream stream);
/* CUDA-IPC exchange buffers (cudaMalloc + cudaIpcGetMemHandle / cudaIpcOpenMemHandle); handle = 64 bytes */
B2_API b2_status b2_ipc_alloc(size_t bytes, void** out_ptr, uint8_t* out_handle64);
B2_API b2_status b2_ipc_open(const uint8_t* handle64, void** out_ptr);
B2_API b2_status b2_ipc_close(void* ptr);
B2_API b2_status b2_ipc_free(void* ptr);
/* Copy `bytes` (any alignment) from local device memory to `dst`, which may be PEER memory mapped with b2_ipc_open: a
 * plain copy kernel whose stores travel over NVLink (the bucket exchange after b2_partition: one contiguous run per
 * destination rank). Stream-ordered. */
B2_API b2_status b2_peer_copy(void* dst, const void* src, size_t bytes, b2_stream stream);

/* ---- cudf::pack / packed_size / pack_metadata / unpack (cpp/include/cudf/contiguous_split.hpp:233-317, cpp/src/copying/pack.cpp):
 *      libcudf's contiguous wire format for tables of fixed-width columns. metadata = host bytes (16-byte table header +
 *      40 bytes per column), gpu_data = one device buffer (validity then data per column, 64-byte padded). -------------- */
B2_API b2_status b2_packed_size(const b2_table_view* input, size_t* out_bytes);
B2_API b2_status b2_pack(const b2_table_view* input, b2_stream stream, uint8_t* metadata, size_t metadata_capacity,
                         size_t* metadata_size, b2_buffer** gpu_data);
B2_API b2_status b2_pack_metadata(const b2_table_view* input, const uint8_t* contiguous_buffer, size_t buffer_size,
                                  uint8_t* metadata, size_t metadata_capacity, size_t* metadata_size);
/* No allocation: out_columns[i] point into gpu_data (the caller keeps it alive). */
B2_API b2_status b2_unpack(const uint8_t* metadata, size_t metadata_size, const void* gpu_data, b2_column_view* out_columns,
                           int32_t capacity, int32_t* num_columns, int32_t* num_rows);

/* ---- Arrow C Data / C Device Data interface (cpp/include/cudf/interop.hpp to_arrow_schema / to_arrow_device / to_arrow_host /
 *      from_arrow_device_column / from_arrow; cpp/src/interop/*).  The structs are the published Arrow ABI: a pointer to
 *      b2_arrow_schema / b2_arrow_array / b2_arrow_device_array IS a pointer to ArrowSchema / ArrowArray / ArrowDeviceArray.
 *      Fixed-width types only (BOOL8 is bit-packed on the Arrow side and converted). --------------------------------------- */
typedef struct b2_arrow_schema {
  const char* format; const char* name; const char* metadata; int64_t flags; int64_t n_children;
  struct b2_arrow_schema** children; struct b2_arrow_schema* dictionary;
  void (*release)(struct b2_arrow_schema*); void* private_data;
} b2_arrow_schema;
typedef struct b2_arrow_array {
  int64_t length; int64_t null_count; int64_t offset; int64_t n_buffers; int64_t n_children;
  const void** buffers; struct b2_arrow_array** children; struct b2_arrow_array* dictionary;
  void (*release)(struct b2_arrow_array*); void* private_data;
} b2_arrow_array;
typedef struct b2_arrow_device_array {
  b2_arrow_array array; int64_t device_id; int32_t device_type; void* sync_event; int64_t reserved[3];
} b2_arrow_device_array;
B2_API b2_status b2_to_arrow_schema(const b2_column_view* col, const char* name, b2_arrow_schema* out);
/* zero copy: the caller keeps the column alive until out->array.release is called; sync_event is recorded on `stream` */
B2_API b2_status b2_to_arrow_device(const b2_column_view* col, b2_stream stream, b2_arrow_device_array* out);
B2_API b2_status b2_to_arrow_host(const b2_column_view* col, b2_stream stream, b2_arrow_array* out);
/* out_view points into the producer's buffers (which must outlive it); BOOL8 input is converted: *out_owner owns the copy */
B2_API b2_status b2_from_arrow_device(const b2_arrow_schema* schema, const b2_arrow_device_array* in, b2_stream stream,
                                      b2_column_view* out_view, b2_column** out_owner);
B2_API b2_status b2_from_arrow_host(const b2_arrow_schema* schema, const b2_arrow_array* in, b2_stream stream, b2_column** out);
B2_API void      b2_arrow_schema_release(b2_arrow_schema* schema);
B2_API void      b2_arrow_array_release(b2_arrow_array* array);

/* ---- synthetic data (SURVEY §8d generator): x_i = splitmix64(seed + first + i) -------------- */
/* kind 0: raw uint64 -> int64 ; 1: float64 uniform [0,1) ; 2: x mod modulus as int64 ;
 * 3: int32 low bits ; 4: validity bitmask words with P(valid)=0.5 (n = number of bits) */
B2_API b2_status b2_fill_splitmix64(void* dst, int64_t n, uint64_t seed, int64_t first, int32_t kind,
                                    uint64_t modulus, b2_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* CUDF_B200_H */

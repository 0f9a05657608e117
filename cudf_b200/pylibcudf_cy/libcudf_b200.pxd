# cython: language_level=3
# Declarations of the C ABI (include/cudf_b200.h) for Cython callers — the role python/pylibcudf/pylibcudf/libcudf/*.pxd
# play for libcudf's C++ API (e.g. libcudf/sorting.pxd:24-90, libcudf/join.pxd, libcudf/groupby.pxd, libcudf/reduce.pxd).
# Cython checks every call in _core.pyx against these prototypes, and the C compiler checks the prototypes against the header.
from libc.stdint cimport int32_t, int64_t, uint8_t, uint32_t, uint64_t

cdef extern from "cudf_b200.h" nogil:
    ctypedef void* b2_stream

    ctypedef enum b2_status:
        B2_SUCCESS

    ctypedef struct b2_column_view:
        int32_t type_id
        int32_t size
        const void* data
        const uint32_t* null_mask
        int32_t null_count
        int32_t offset

    ctypedef struct b2_table_view:
        const b2_column_view* columns
        int32_t num_columns

    ctypedef struct b2_column
    ctypedef struct b2_table
    ctypedef struct b2_scalar
    ctypedef struct b2_groupby
    ctypedef struct b2_hash_join
    ctypedef struct b2_filtered_join

    ctypedef struct b2_agg_request:
        b2_column_view values
        const int32_t* kinds
        int32_t num_kinds

    const char* b2_last_error()
    const char* b2_version()
    uint64_t b2_kernel_launch_count()

    # owning handles
    b2_status b2_column_view_of(const b2_column* col, b2_column_view* out)
    void b2_column_free(b2_column* col)
    int32_t b2_table_num_columns(const b2_table* tbl)
    b2_status b2_table_release(b2_table* tbl, b2_column** out_cols, int32_t capacity)
    void b2_table_free(b2_table* tbl)
    int32_t b2_scalar_type(const b2_scalar* s)
    b2_status b2_scalar_get(const b2_scalar* s, b2_stream stream, void* host_value, int32_t* is_valid)
    void b2_scalar_free(b2_scalar* s)

    # null masks
    b2_status b2_null_count(const uint32_t* bitmask, int32_t start, int32_t stop, b2_stream stream, int32_t* out)

    # copying
    b2_status b2_gather(const b2_table_view* source, const b2_column_view* gather_map, int32_t oob_policy, b2_stream stream,
                        b2_table** out)

    # sorting (cpp/include/cudf/sorting.hpp:44-163)
    b2_status b2_sorted_order(const b2_table_view* keys, const uint8_t* column_order, int32_t n_order,
                              const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable, b2_stream stream, b2_column** out)
    b2_status b2_sort(const b2_table_view* input, const uint8_t* column_order, int32_t n_order, const uint8_t* null_precedence,
                      int32_t n_null_prec, int32_t stable, b2_stream stream, b2_table** out)
    b2_status b2_sort_by_key(const b2_table_view* values, const b2_table_view* keys, const uint8_t* column_order, int32_t n_order,
                             const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable, b2_stream stream, b2_table** out)

    # joins (cpp/include/cudf/join/join.hpp:127-249, join/hash_join.hpp)
    b2_status b2_inner_join(const b2_table_view* left_keys, const b2_table_view* right_keys, int32_t compare_nulls, b2_stream stream,
                            b2_column** out_left, b2_column** out_right)
    b2_status b2_left_join(const b2_table_view* left_keys, const b2_table_view* right_keys, int32_t compare_nulls, b2_stream stream,
                           b2_column** out_left, b2_column** out_right)
    b2_status b2_full_join(const b2_table_view* left_keys, const b2_table_view* right_keys, int32_t compare_nulls, b2_stream stream,
                           b2_column** out_left, b2_column** out_right)
    b2_status b2_hash_join_create(const b2_table_view* build, int32_t has_nulls, int32_t compare_nulls, double load_factor,
                                  b2_stream stream, b2_hash_join** out)
    void b2_hash_join_destroy(b2_hash_join* hj)
    b2_status b2_hash_join_inner_join(const b2_hash_join* hj, const b2_table_view* probe, int32_t has_output_size, size_t output_size,
                                      b2_stream stream, b2_column** out_left, b2_column** out_right)
    b2_status b2_hash_join_left_join(const b2_hash_join* hj, const b2_table_view* probe, int32_t has_output_size, size_t output_size,
                                     b2_stream stream, b2_column** out_left, b2_column** out_right)
    b2_status b2_hash_join_full_join(const b2_hash_join* hj, const b2_table_view* probe, int32_t has_output_size, size_t output_size,
                                     b2_stream stream, b2_column** out_left, b2_column** out_right)
    b2_status b2_hash_join_inner_join_size(const b2_hash_join* hj, const b2_table_view* probe, b2_stream stream, size_t* out)
    b2_status b2_hash_join_left_join_size(const b2_hash_join* hj, const b2_table_view* probe, b2_stream stream, size_t* out)
    b2_status b2_hash_join_full_join_size(const b2_hash_join* hj, const b2_table_view* probe, b2_stream stream, size_t* out)

    # semi / anti joins (cpp/include/cudf/join/filtered_join.hpp)
    b2_status b2_filtered_join_create(const b2_table_view* right, int32_t compare_nulls, double load_factor, b2_stream stream,
                                      b2_filtered_join** out)
    void b2_filtered_join_destroy(b2_filtered_join* fj)
    b2_status b2_filtered_join_semi_join(const b2_filtered_join* fj, const b2_table_view* left, b2_stream stream, b2_column** out)
    b2_status b2_filtered_join_anti_join(const b2_filtered_join* fj, const b2_table_view* left, b2_stream stream, b2_column** out)

    # groupby (cpp/include/cudf/groupby.hpp:54-184)
    b2_status b2_groupby_create(const b2_table_view* keys, int32_t null_handling, int32_t keys_are_sorted, const uint8_t* column_order,
                                int32_t n_order, const uint8_t* null_precedence, int32_t n_null_prec, b2_groupby** out)
    void b2_groupby_destroy(b2_groupby* gb)
    b2_status b2_groupby_aggregate(b2_groupby* gb, const b2_agg_request* requests, int32_t num_requests, b2_stream stream,
                                   b2_table** out_keys, b2_table** out_results)
    b2_status b2_groupby_scan(b2_groupby* gb, const b2_agg_request* requests, int32_t num_requests, b2_stream stream,
                              b2_table** out_keys, b2_table** out_results)

    # reductions (cpp/include/cudf/reduction.hpp)
    b2_status b2_reduce(const b2_column_view* col, int32_t agg_kind, int32_t output_type_id, const b2_scalar* init, b2_stream stream,
                        b2_scalar** out)
    b2_status b2_segmented_reduce(const b2_column_view* values, const int32_t* offsets, int32_t num_offsets, int32_t agg_kind,
                                  int32_t output_type_id, int32_t null_handling, const b2_scalar* init, b2_stream stream,
                                  b2_column** out)
    b2_status b2_scan(const b2_column_view* col, int32_t agg_kind, int32_t scan_type, int32_t null_handling, b2_stream stream,
                      b2_column** out)

    # ---- the rest of the path's modules ----
    ctypedef struct b2_buffer
    size_t b2_bitmask_allocation_size_bytes(int32_t number_of_bits)
    b2_status b2_create_null_mask(int32_t size, int32_t mask_state, b2_stream stream, b2_buffer** out)
    b2_status b2_set_null_mask(uint32_t* bitmask, int32_t begin_bit, int32_t end_bit, int32_t valid, b2_stream stream)
    b2_status b2_copy_bitmask(const uint32_t* mask, int32_t begin_bit, int32_t end_bit, b2_stream stream, b2_buffer** out)
    b2_status b2_count_set_bits(const uint32_t* bitmask, int32_t start, int32_t stop, b2_stream stream, int32_t* out)
    b2_status b2_bitmask_and(const b2_table_view* view, b2_stream stream, b2_buffer** out_mask, int32_t* out_null_count)

    b2_status b2_segmented_sorted_order(const b2_table_view* keys, const b2_column_view* segment_offsets, const uint8_t* column_order,
                                        int32_t n_order, const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable,
                                        b2_stream stream, b2_column** out)
    b2_status b2_segmented_sort_by_key(const b2_table_view* values, const b2_table_view* keys, const b2_column_view* segment_offsets,
                                       const uint8_t* column_order, int32_t n_order, const uint8_t* null_precedence, int32_t n_null_prec,
                                       int32_t stable, b2_stream stream, b2_table** out)
    b2_status b2_top_k(const b2_column_view* col, int32_t k, int32_t topk_order, b2_stream stream, b2_column** out)
    b2_status b2_top_k_order(const b2_column_view* col, int32_t k, int32_t topk_order, b2_stream stream, b2_column** out)
    b2_status b2_rank(const b2_column_view* input, int32_t method, int32_t column_order, int32_t null_handling, int32_t null_precedence,
                      int32_t percentage, b2_stream stream, b2_column** out)

    b2_status b2_hash_join_match_counts(const b2_hash_join* hj, const b2_table_view* probe, int32_t join_kind, b2_stream stream,
                                        b2_column** out_counts)
    b2_status b2_hash_join_partitioned_join(const b2_hash_join* hj, const b2_table_view* probe, const b2_column_view* match_counts,
                                            int32_t left_start, int32_t left_end, int32_t join_kind, b2_stream stream,
                                            b2_column** out_left, b2_column** out_right)
    b2_status b2_hash_join_finalize_full_join(const b2_column_view* left_partials, const b2_column_view* right_partials,
                                              int32_t num_partials, int32_t left_table_num_rows, int32_t right_table_num_rows,
                                              b2_stream stream, b2_column** out_left, b2_column** out_right)

    b2_status b2_hash_partition(const b2_table_view* input, const b2_table_view* keys, int32_t num_partitions, int32_t hash_function,
                                uint32_t seed, b2_stream stream, b2_table** out, int32_t* out_offsets)
    b2_status b2_partition_by_map(const b2_table_view* input, const b2_column_view* partition_map, int32_t num_partitions,
                                  b2_stream stream, b2_table** out, int32_t* out_offsets)

    # stream compaction (cpp/include/cudf/stream_compaction.hpp)
    b2_status b2_apply_boolean_mask(const b2_table_view* input, const b2_column_view* mask, int32_t deletion, b2_stream stream,
                                    b2_table** out)
    b2_status b2_drop_nulls(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep_threshold,
                            b2_stream stream, b2_table** out)
    b2_status b2_drop_nans(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep_threshold,
                           b2_stream stream, b2_table** out)
    b2_status b2_unique(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep, int32_t nulls_equal,
                        b2_stream stream, b2_table** out)
    b2_status b2_distinct(const b2_table_view* input, const int32_t* keys, int32_t num_keys, int32_t keep, int32_t nulls_equal,
                          int32_t nans_equal, int32_t stable, b2_stream stream, b2_table** out)
    b2_status b2_distinct_indices(const b2_table_view* input, int32_t keep, int32_t nulls_equal, int32_t nans_equal,
                                  b2_stream stream, b2_column** out)

    # binary operations (cpp/include/cudf/binaryop.hpp)
    b2_status b2_binary_operation(const b2_column_view* lhs, const b2_column_view* rhs, int32_t op, int32_t out_type, b2_stream stream,
                                  b2_column** out)
    b2_status b2_binary_operation_cs(const b2_column_view* lhs, const b2_scalar* rhs, int32_t op, int32_t out_type, b2_stream stream,
                                     b2_column** out)
    b2_status b2_binary_operation_sc(const b2_scalar* lhs, const b2_column_view* rhs, int32_t op, int32_t out_type, b2_stream stream,
                                     b2_column** out)
    b2_status b2_binary_is_supported_operation(int32_t out_type, int32_t lhs_type, int32_t rhs_type, int32_t op, int32_t* result)

    # unary operations and casts (cpp/include/cudf/unary.hpp)
    b2_status b2_unary_operation(const b2_column_view* input, int32_t op, b2_stream stream, b2_column** out)
    b2_status b2_cast(const b2_column_view* input, int32_t out_type, b2_stream stream, b2_column** out)
    b2_status b2_is_supported_cast(int32_t from_type, int32_t to_type, int32_t* result)
    b2_status b2_is_null(const b2_column_view* input, b2_stream stream, b2_column** out)
    b2_status b2_is_valid(const b2_column_view* input, b2_stream stream, b2_column** out)
    b2_status b2_is_nan(const b2_column_view* input, b2_stream stream, b2_column** out)
    b2_status b2_is_not_nan(const b2_column_view* input, b2_stream stream, b2_column** out)

    # replacement (cpp/include/cudf/replace.hpp)
    b2_status b2_replace_nulls(const b2_column_view* input, const b2_column_view* replacement, b2_stream stream, b2_column** out)
    b2_status b2_replace_nulls_scalar(const b2_column_view* input, const b2_scalar* replacement, b2_stream stream, b2_column** out)
    b2_status b2_replace_nulls_policy(const b2_column_view* input, int32_t policy, b2_stream stream, b2_column** out)
    b2_status b2_find_and_replace_all(const b2_column_view* input, const b2_column_view* values_to_replace,
                                      const b2_column_view* replacement_values, b2_stream stream, b2_column** out)
    b2_status b2_clamp(const b2_column_view* input, const b2_scalar* lo, const b2_scalar* lo_replace, const b2_scalar* hi,
                       const b2_scalar* hi_replace, b2_stream stream, b2_column** out)
    b2_status b2_normalize_nans_and_zeros(const b2_column_view* input, b2_stream stream, b2_column** out)
    b2_status b2_normalize_nans_and_zeros_inplace(const b2_column_view* in_out, b2_stream stream)

    # cudf::pack / unpack (cpp/include/cudf/contiguous_split.hpp:233-317)
    void* b2_buffer_data(const b2_buffer* buf)
    size_t b2_buffer_size(const b2_buffer* buf)
    b2_status b2_packed_size(const b2_table_view* input, size_t* out_bytes)
    b2_status b2_pack(const b2_table_view* input, b2_stream stream, uint8_t* metadata, size_t metadata_capacity, size_t* metadata_size,
                      b2_buffer** gpu_data)
    b2_status b2_pack_metadata(const b2_table_view* input, const uint8_t* contiguous_buffer, size_t buffer_size, uint8_t* metadata,
                               size_t metadata_capacity, size_t* metadata_size)
    b2_status b2_unpack(const uint8_t* metadata, size_t metadata_size, const void* gpu_data, b2_column_view* out_columns, int32_t capacity,
                        int32_t* num_columns, int32_t* num_rows)

"""ctypes binding of include/cudf_b200.h. No fallback: a missing library is an ImportError."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libcudf_b200.so"


class Cudf_b200Error(RuntimeError):
    pass


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        if os.environ.get("CUDF_B200_AUTOBUILD", "0") == "1":
            from .build import build

            build()
        else:
            raise ImportError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback for this package)"
            )
    return C.CDLL(str(LIB_PATH), mode=C.RTLD_GLOBAL)


lib = _load()

b2_stream = C.c_void_p


class ColumnView(C.Structure):
    _fields_ = [
        ("type_id", C.c_int32),
        ("size", C.c_int32),
        ("data", C.c_void_p),
        ("null_mask", C.c_void_p),
        ("null_count", C.c_int32),
        ("offset", C.c_int32),
    ]


class TableView(C.Structure):
    _fields_ = [("columns", C.POINTER(ColumnView)), ("num_columns", C.c_int32)]


class AggRequest(C.Structure):
    _fields_ = [("values", ColumnView), ("kinds", C.POINTER(C.c_int32)), ("num_kinds", C.c_int32)]


# logic_error -> RuntimeError etc.: python/pylibcudf/pylibcudf/exception_handler.pxd:29-66
_STATUS_EXC = {
    1: RuntimeError,   # cudf::logic_error
    2: ValueError,     # std::invalid_argument
    3: TypeError,      # cudf::data_type_error
    4: IndexError,     # std::out_of_range
    5: MemoryError,    # std::bad_alloc
    6: RuntimeError,   # cudf::cuda_error
}

lib.b2_last_error.restype = C.c_char_p
lib.b2_version.restype = C.c_char_p
lib.b2_kernel_launch_count.restype = C.c_uint64


def check(status: int) -> None:
    if status != 0:
        msg = lib.b2_last_error().decode("utf-8", "replace")
        raise _STATUS_EXC.get(status, RuntimeError)(msg)


MISSING: list[str] = []


def _sig(name, argtypes, restype=C.c_int):
    try:
        fn = getattr(lib, name)
    except AttributeError:  # reported by tests/test_capi_symbols.py; calling it raises AttributeError
        MISSING.append(name)
        return None
    fn.argtypes = argtypes
    fn.restype = restype
    return fn


P = C.POINTER
vp = C.c_void_p
i32 = C.c_int32
u8p = P(C.c_uint8)

_sig("b2_column_view_of", [vp, P(ColumnView)])
_sig("b2_column_free", [vp], None)
_sig("b2_table_num_columns", [vp], i32)
_sig("b2_table_num_rows", [vp], i32)
_sig("b2_table_column", [vp, i32], vp)
_sig("b2_table_release", [vp, P(vp), i32])
_sig("b2_table_free", [vp], None)
_sig("b2_buffer_data", [vp], vp)
_sig("b2_buffer_size", [vp], C.c_size_t)
_sig("b2_buffer_free", [vp], None)
_sig("b2_scalar_create", [i32, vp, i32, b2_stream, P(vp)])
_sig("b2_scalar_type", [vp], i32)
_sig("b2_scalar_device_data", [vp], vp)
_sig("b2_scalar_get", [vp, b2_stream, vp, P(i32)])
_sig("b2_scalar_free", [vp], None)
_sig("b2_trim_pool", [])
_sig("b2_profile_enable", [i32], None)
_sig("b2_profile_reset", [], None)
_sig("b2_profile_get", [C.c_char_p, P(C.c_double), P(C.c_int64)])
_sig("b2_profile_get_over", [C.c_char_p, C.c_double, P(C.c_double), P(C.c_int64)])
_sig("b2_bitmask_allocation_size_bytes", [i32], C.c_size_t)
_sig("b2_create_null_mask", [i32, i32, b2_stream, P(vp)])
_sig("b2_set_null_mask", [vp, i32, i32, i32, b2_stream])
_sig("b2_copy_bitmask", [vp, i32, i32, b2_stream, P(vp)])
_sig("b2_count_set_bits", [vp, i32, i32, b2_stream, P(i32)])
_sig("b2_null_count", [vp, i32, i32, b2_stream, P(i32)])
_sig("b2_bitmask_and", [P(TableView), b2_stream, P(vp), P(i32)])
_sig("b2_gather", [P(TableView), P(ColumnView), i32, b2_stream, P(vp)])
_sig("b2_sorted_order", [P(TableView), u8p, i32, u8p, i32, i32, b2_stream, P(vp)])
_sig("b2_sort", [P(TableView), u8p, i32, u8p, i32, i32, b2_stream, P(vp)])
_sig("b2_sort_by_key", [P(TableView), P(TableView), u8p, i32, u8p, i32, i32, b2_stream, P(vp)])
_sig("b2_segmented_sorted_order", [P(TableView), P(ColumnView), u8p, i32, u8p, i32, i32, b2_stream, P(vp)])
_sig("b2_segmented_sort_by_key", [P(TableView), P(TableView), P(ColumnView), u8p, i32, u8p, i32, i32, b2_stream, P(vp)])
_sig("b2_top_k", [P(ColumnView), i32, i32, b2_stream, P(vp)])
_sig("b2_top_k_order", [P(ColumnView), i32, i32, b2_stream, P(vp)])
_sig("b2_rank", [P(ColumnView), i32, i32, i32, i32, i32, b2_stream, P(vp)])
for _j in ("inner", "left", "full"):
    _sig(f"b2_{_j}_join", [P(TableView), P(TableView), i32, b2_stream, P(vp), P(vp)])
    _sig(f"b2_hash_join_{_j}_join", [vp, P(TableView), i32, C.c_size_t, b2_stream, P(vp), P(vp)])
    _sig(f"b2_hash_join_{_j}_join_size", [vp, P(TableView), b2_stream, P(C.c_size_t)])
_sig("b2_hash_join_match_counts", [vp, P(TableView), i32, b2_stream, P(vp)])
_sig("b2_hash_join_partitioned_join", [vp, P(TableView), P(ColumnView), i32, i32, i32, b2_stream, P(vp), P(vp)])
_sig("b2_hash_join_finalize_full_join", [P(ColumnView), P(ColumnView), i32, i32, i32, b2_stream, P(vp), P(vp)])
_sig("b2_hash_join_create", [P(TableView), i32, i32, C.c_double, b2_stream, P(vp)])
_sig("b2_hash_join_destroy", [vp], None)
_sig("b2_filtered_join_create", [P(TableView), i32, C.c_double, b2_stream, P(vp)])
_sig("b2_filtered_join_destroy", [vp], None)
_sig("b2_filtered_join_semi_join", [vp, P(TableView), b2_stream, P(vp)])
_sig("b2_filtered_join_anti_join", [vp, P(TableView), b2_stream, P(vp)])
_sig("b2_binary_operation", [P(ColumnView), P(ColumnView), i32, i32, b2_stream, P(vp)])
_sig("b2_binary_operation_cs", [P(ColumnView), vp, i32, i32, b2_stream, P(vp)])
_sig("b2_binary_operation_sc", [vp, P(ColumnView), i32, i32, b2_stream, P(vp)])
_sig("b2_binary_is_supported_operation", [i32, i32, i32, i32, P(i32)])
_sig("b2_unary_operation", [P(ColumnView), i32, b2_stream, P(vp)])
_sig("b2_cast", [P(ColumnView), i32, b2_stream, P(vp)])
_sig("b2_is_supported_cast", [i32, i32, P(i32)])
_sig("b2_is_null", [P(ColumnView), b2_stream, P(vp)])
_sig("b2_is_valid", [P(ColumnView), b2_stream, P(vp)])
_sig("b2_is_nan", [P(ColumnView), b2_stream, P(vp)])
_sig("b2_is_not_nan", [P(ColumnView), b2_stream, P(vp)])
_sig("b2_replace_nulls", [P(ColumnView), P(ColumnView), b2_stream, P(vp)])
_sig("b2_replace_nulls_scalar", [P(ColumnView), vp, b2_stream, P(vp)])
_sig("b2_replace_nulls_policy", [P(ColumnView), i32, b2_stream, P(vp)])
_sig("b2_replace_nans", [P(ColumnView), P(ColumnView), b2_stream, P(vp)])
_sig("b2_replace_nans_scalar", [P(ColumnView), vp, b2_stream, P(vp)])
_sig("b2_find_and_replace_all", [P(ColumnView), P(ColumnView), P(ColumnView), b2_stream, P(vp)])
_sig("b2_clamp", [P(ColumnView), vp, vp, vp, vp, b2_stream, P(vp)])
_sig("b2_normalize_nans_and_zeros", [P(ColumnView), b2_stream, P(vp)])
_sig("b2_normalize_nans_and_zeros_inplace", [P(ColumnView), b2_stream])
_sig("b2_groupby_create", [P(TableView), i32, i32, u8p, i32, u8p, i32, P(vp)])
_sig("b2_groupby_destroy", [vp], None)
_sig("b2_groupby_aggregate", [vp, P(AggRequest), i32, b2_stream, P(vp), P(vp)])
_sig("b2_groupby_scan", [vp, P(AggRequest), i32, b2_stream, P(vp), P(vp)])
_sig("b2_reduce", [P(ColumnView), i32, i32, vp, b2_stream, P(vp)])
_sig("b2_segmented_reduce", [P(ColumnView), vp, i32, i32, i32, i32, vp, b2_stream, P(vp)])
_sig("b2_scan", [P(ColumnView), i32, i32, i32, b2_stream, P(vp)])
_sig("b2_partition", [P(TableView), P(ColumnView), i32, vp, i32, b2_stream, P(vp), P(i32)])
_sig("b2_hash_partition", [P(TableView), P(TableView), i32, i32, C.c_uint32, b2_stream, P(vp), P(i32)])
_sig("b2_partition_by_map", [P(TableView), P(ColumnView), i32, b2_stream, P(vp), P(i32)])
_sig("b2_partition_plan_create", [P(ColumnView), i32, vp, i32, b2_stream, P(vp), P(C.c_int64)])
_sig("b2_partition_scatter", [vp, P(ColumnView), P(vp), b2_stream])
_sig("b2_partition_scatter_staged", [vp, P(ColumnView), P(vp), b2_stream])
_sig("b2_partition_plan_free", [vp], None)
_sig("b2_range_partition_counts", [P(ColumnView), vp, i32, b2_stream, P(C.c_int64)])
_sig("b2_range_partition_scatter", [P(ColumnView), P(ColumnView), vp, i32, P(vp), P(vp), b2_stream])
_sig("b2_ipc_alloc", [C.c_size_t, P(vp), u8p])
_sig("b2_ipc_open", [u8p, P(vp)])
_sig("b2_ipc_close", [vp])
_sig("b2_ipc_free", [vp])
_sig("b2_peer_copy", [vp, vp, C.c_size_t, b2_stream])
_sig("b2_packed_size", [P(TableView), P(C.c_size_t)])
_sig("b2_pack", [P(TableView), b2_stream, u8p, C.c_size_t, P(C.c_size_t), P(vp)])
_sig("b2_pack_metadata", [P(TableView), vp, C.c_size_t, u8p, C.c_size_t, P(C.c_size_t)])
_sig("b2_unpack", [u8p, C.c_size_t, vp, P(ColumnView), i32, P(i32), P(i32)])
_sig("b2_apply_boolean_mask", [P(TableView), P(ColumnView), i32, b2_stream, P(vp)])
_sig("b2_drop_nulls", [P(TableView), P(i32), i32, i32, b2_stream, P(vp)])
_sig("b2_drop_nans", [P(TableView), P(i32), i32, i32, b2_stream, P(vp)])
_sig("b2_unique", [P(TableView), P(i32), i32, i32, i32, b2_stream, P(vp)])
_sig("b2_distinct", [P(TableView), P(i32), i32, i32, i32, i32, i32, b2_stream, P(vp)])
_sig("b2_distinct_indices", [P(TableView), i32, i32, i32, b2_stream, P(vp)])
_sig("b2_fill_splitmix64", [vp, C.c_int64, C.c_uint64, C.c_int64, i32, C.c_uint64, b2_stream])

# every symbol the header declares, for the loader test
DECLARED_SYMBOLS = [
    "b2_last_error", "b2_version", "b2_kernel_launch_count", "b2_trim_pool", "b2_profile_enable", "b2_profile_reset",
    "b2_profile_get", "b2_column_view_of", "b2_column_free",
    "b2_table_num_columns", "b2_table_num_rows", "b2_table_column", "b2_table_release", "b2_table_free",
    "b2_buffer_data", "b2_buffer_size", "b2_buffer_free", "b2_scalar_create", "b2_scalar_type",
    "b2_scalar_device_data", "b2_scalar_get", "b2_scalar_free", "b2_bitmask_allocation_size_bytes",
    "b2_create_null_mask", "b2_set_null_mask", "b2_copy_bitmask", "b2_count_set_bits", "b2_null_count",
    "b2_bitmask_and", "b2_gather", "b2_sorted_order", "b2_sort", "b2_sort_by_key", "b2_segmented_sorted_order",
    "b2_segmented_sort_by_key", "b2_top_k", "b2_top_k_order", "b2_rank", "b2_inner_join", "b2_left_join",
    "b2_full_join", "b2_hash_join_create", "b2_hash_join_destroy", "b2_hash_join_inner_join",
    "b2_hash_join_left_join", "b2_hash_join_full_join", "b2_hash_join_inner_join_size",
    "b2_hash_join_left_join_size", "b2_hash_join_full_join_size", "b2_hash_join_match_counts",
    "b2_hash_join_partitioned_join", "b2_hash_join_finalize_full_join", "b2_groupby_create", "b2_groupby_destroy",
    "b2_groupby_aggregate", "b2_groupby_scan", "b2_reduce", "b2_segmented_reduce", "b2_scan", "b2_partition",
    "b2_partition_plan_create", "b2_partition_scatter", "b2_partition_scatter_staged", "b2_partition_plan_free", "b2_ipc_alloc", "b2_ipc_open", "b2_ipc_close",
    "b2_ipc_free", "b2_peer_copy", "b2_profile_get_over", "b2_hash_partition", "b2_partition_by_map", "b2_range_partition_counts", "b2_range_partition_scatter", "b2_packed_size", "b2_pack", "b2_pack_metadata", "b2_unpack", "b2_to_arrow_schema", "b2_to_arrow_device", "b2_to_arrow_host", "b2_from_arrow_device",
    "b2_from_arrow_host", "b2_arrow_schema_release", "b2_arrow_array_release",
    "b2_fill_splitmix64", "b2_apply_boolean_mask", "b2_drop_nulls", "b2_drop_nans", "b2_unique", "b2_distinct",
    "b2_distinct_indices", "b2_filtered_join_create", "b2_filtered_join_destroy", "b2_filtered_join_semi_join",
    "b2_filtered_join_anti_join", "b2_binary_operation", "b2_binary_operation_cs", "b2_binary_operation_sc",
    "b2_binary_is_supported_operation", "b2_unary_operation", "b2_cast", "b2_is_supported_cast", "b2_is_null", "b2_is_valid",
    "b2_is_nan", "b2_is_not_nan", "b2_replace_nulls", "b2_replace_nulls_scalar", "b2_replace_nulls_policy", "b2_replace_nans",
    "b2_replace_nans_scalar", "b2_find_and_replace_all", "b2_clamp", "b2_normalize_nans_and_zeros",
    "b2_normalize_nans_and_zeros_inplace",
]


def current_stream() -> int:
    """cudaStream_t of torch's current stream when torch is imported and CUDA is up, else the legacy stream."""
    import sys

    torch = sys.modules.get("torch")
    if torch is not None and torch.cuda.is_available():
        return int(torch.cuda.current_stream().cuda_stream)
    return 0


def stream_arg(stream) -> C.c_void_p:
    if stream is None:
        return C.c_void_p(current_stream())
    if hasattr(stream, "cuda_stream"):
        return C.c_void_p(int(stream.cuda_stream))
    return C.c_void_p(int(stream))


def kernel_launch_count() -> int:
    return int(lib.b2_kernel_launch_count())


def profile_get(name: str):
    ms, cnt = C.c_double(0), C.c_int64(0)
    check(lib.b2_profile_get(name.encode(), C.byref(ms), C.byref(cnt)))
    return ms.value, cnt.value


def profile_get_over(name: str, min_ms: float):
    """(total ms, count) of the profiled scopes `name` that lasted at least min_ms."""
    ms, cnt = C.c_double(0), C.c_int64(0)
    check(lib.b2_profile_get_over(name.encode(), float(min_ms), C.byref(ms), C.byref(cnt)))
    return ms.value, cnt.value

"""pylibcudf.stream_compaction twin (python/pylibcudf/pylibcudf/stream_compaction.pyx; cpp/include/cudf/stream_compaction.hpp)
over b2_apply_boolean_mask / b2_drop_nulls / b2_drop_nans / b2_unique / b2_distinct / b2_distinct_indices
(cudf_b200/csrc/stream_compaction.cu: one stable compaction kernel + gather).

Fixed-width columns, at most 8 key columns. `distinct` returns its rows in input order, which is one valid order of the
reference's unspecified one."""
from __future__ import annotations

import ctypes as C
import enum

from .. import _lib
from .._lib import check, lib
from .column import Column, Table
from .types import NanEquality, NullEquality


class DuplicateKeepOption(enum.IntEnum):  # cudf::duplicate_keep_option (stream_compaction.hpp)
    KEEP_ANY = 0
    KEEP_FIRST = 1
    KEEP_LAST = 2
    KEEP_NONE = 3


def _keys(keys):
    keys = [int(k) for k in keys]
    return (C.c_int32 * max(len(keys), 1))(*keys), len(keys)


def _mask(source_table: Table, mask: Column, deletion: int, stream) -> Table:
    out = C.c_void_p()
    tv, mv = source_table._view(), mask._view()
    check(lib.b2_apply_boolean_mask(C.byref(tv), C.byref(mv), deletion, _lib.stream_arg(stream), C.byref(out)))
    return Table._from_handle(out.value)


def apply_boolean_mask(source_table: Table, boolean_mask: Column, stream=None, mr=None) -> Table:
    """Rows where `boolean_mask` (BOOL8) is valid and true, in input order."""
    return _mask(source_table, boolean_mask, 0, stream)


def apply_deletion_mask(input: Table, deletion_mask: Column, stream=None, mr=None) -> Table:  # noqa: A002
    """Rows where `deletion_mask` (BOOL8) is valid and false, in input order."""
    return _mask(input, deletion_mask, 1, stream)


def _threshold_call(fn, source_table: Table, keys, keep_threshold, stream) -> Table:
    arr, nk = _keys(keys)
    thr = nk if keep_threshold is None else int(keep_threshold)
    out = C.c_void_p()
    tv = source_table._view()
    check(fn(C.byref(tv), arr, nk, thr, _lib.stream_arg(stream), C.byref(out)))
    return Table._from_handle(out.value)


def drop_nulls(source_table: Table, keys, keep_threshold: int | None = None, stream=None, mr=None) -> Table:
    """Rows with at least `keep_threshold` (default: all) valid columns among `keys`."""
    return _threshold_call(lib.b2_drop_nulls, source_table, keys, keep_threshold, stream)


def drop_nans(source_table: Table, keys, keep_threshold: int | None = None, stream=None, mr=None) -> Table:
    """Rows with at least `keep_threshold` (default: all) non-NaN columns among the float `keys`; a null is not NaN."""
    return _threshold_call(lib.b2_drop_nans, source_table, keys, keep_threshold, stream)


def unique(input: Table, keys, keep: DuplicateKeepOption, nulls_equal: NullEquality, stream=None, mr=None) -> Table:  # noqa: A002
    """Drops consecutive duplicate rows of the `keys` columns."""
    arr, nk = _keys(keys)
    out = C.c_void_p()
    tv = input._view()
    check(lib.b2_unique(C.byref(tv), arr, nk, int(keep), int(nulls_equal), _lib.stream_arg(stream), C.byref(out)))
    return Table._from_handle(out.value)


def _distinct(input: Table, keys, keep, nulls_equal, nans_equal, stable, stream) -> Table:  # noqa: A002
    arr, nk = _keys(keys)
    out = C.c_void_p()
    tv = input._view()
    check(lib.b2_distinct(C.byref(tv), arr, nk, int(keep), int(nulls_equal), int(nans_equal), stable, _lib.stream_arg(stream),
                          C.byref(out)))
    return Table._from_handle(out.value)


def distinct(input: Table, keys, keep: DuplicateKeepOption, nulls_equal: NullEquality, nans_equal: NanEquality,  # noqa: A002
             stream=None, mr=None) -> Table:
    """One row per set of equal `keys` rows; the order is unspecified (here: input order)."""
    return _distinct(input, keys, keep, nulls_equal, nans_equal, 0, stream)


def stable_distinct(input: Table, keys, keep: DuplicateKeepOption, nulls_equal: NullEquality, nans_equal: NanEquality,  # noqa: A002
                    stream=None, mr=None) -> Table:
    """The rows of `distinct`, in input order."""
    return _distinct(input, keys, keep, nulls_equal, nans_equal, 1, stream)


def distinct_indices(input: Table, keep: DuplicateKeepOption, nulls_equal: NullEquality, nans_equal: NanEquality,  # noqa: A002
                     stream=None, mr=None) -> Column:
    """INT32 indices of the rows `distinct` keeps over all columns of `input`, ascending."""
    out = C.c_void_p()
    tv = input._view()
    check(lib.b2_distinct_indices(C.byref(tv), int(keep), int(nulls_equal), int(nans_equal), _lib.stream_arg(stream), C.byref(out)))
    return Column._from_handle(out.value)

"""pylibcudf.join twin (python/pylibcudf/pylibcudf/join.pyx:63-306) + the cudf::hash_join and cudf::filtered_join objects."""
from __future__ import annotations

import ctypes as C

from .. import _lib
from .._lib import check, lib
from .column import Column, Table
from .types import NullEquality


def _free_join(name, left_keys, right_keys, nulls_equal, stream):
    lo, ro = C.c_void_p(), C.c_void_p()
    lv, rv = left_keys._view(), right_keys._view()
    check(getattr(lib, name)(C.byref(lv), C.byref(rv), int(nulls_equal), _lib.stream_arg(stream), C.byref(lo), C.byref(ro)))
    return Column._from_handle(lo.value), Column._from_handle(ro.value)


def inner_join(left_keys: Table, right_keys: Table, nulls_equal: NullEquality, stream=None, mr=None):
    return _free_join("b2_inner_join", left_keys, right_keys, nulls_equal, stream)


def left_join(left_keys: Table, right_keys: Table, nulls_equal: NullEquality, stream=None, mr=None):
    return _free_join("b2_left_join", left_keys, right_keys, nulls_equal, stream)


def full_join(left_keys: Table, right_keys: Table, nulls_equal: NullEquality, stream=None, mr=None):
    return _free_join("b2_full_join", left_keys, right_keys, nulls_equal, stream)


def left_semi_join(left_keys: Table, right_keys: Table, nulls_equal: NullEquality, stream=None, mr=None) -> Column:
    """INT32 indices of the left rows equal to some right row, ascending (join.pyx:207-256: a FilteredJoin probed once)."""
    return FilteredJoin(right_keys, nulls_equal, stream=stream).semi_join(left_keys, stream)


def left_anti_join(left_keys: Table, right_keys: Table, nulls_equal: NullEquality, stream=None, mr=None) -> Column:
    """INT32 indices of the left rows equal to no right row, ascending (join.pyx:259-306)."""
    return FilteredJoin(right_keys, nulls_equal, stream=stream).anti_join(left_keys, stream)


class FilteredJoin:
    """cudf::filtered_join (cpp/include/cudf/join/filtered_join.hpp): the right (filter) table's keys become a distinct set
    once; semi_join / anti_join probe it with any number of left tables. Keeps `right` alive: keys wider than 8 bytes are
    compared against its columns."""

    def __init__(self, right: Table, compare_nulls: NullEquality, load_factor: float = 0.5, stream=None):
        self._right = right
        out = C.c_void_p()
        rv = right._view()
        check(lib.b2_filtered_join_create(C.byref(rv), int(compare_nulls), float(load_factor), _lib.stream_arg(stream), C.byref(out)))
        self._handle = out.value

    def _probe(self, name, left, stream):
        out = C.c_void_p()
        lv = left._view()
        check(getattr(lib, name)(C.c_void_p(self._handle), C.byref(lv), _lib.stream_arg(stream), C.byref(out)))
        return Column._from_handle(out.value)

    def semi_join(self, left: Table, stream=None, mr=None) -> Column:
        return self._probe("b2_filtered_join_semi_join", left, stream)

    def anti_join(self, left: Table, stream=None, mr=None) -> Column:
        return self._probe("b2_filtered_join_anti_join", left, stream)

    def __del__(self):
        if getattr(self, "_handle", 0):
            lib.b2_filtered_join_destroy(C.c_void_p(self._handle))
            self._handle = 0


class HashJoin:
    """cudf::hash_join (cpp/include/cudf/join/hash_join.hpp): build once, probe many."""

    def __init__(self, build: Table, compare_nulls: NullEquality = NullEquality.EQUAL, has_nulls: bool | None = None,
                 load_factor: float = 0.5, stream=None):
        self._build = build
        out = C.c_void_p()
        bv = build._view()
        hn = -1 if has_nulls is None else int(bool(has_nulls))
        check(lib.b2_hash_join_create(C.byref(bv), hn, int(compare_nulls), float(load_factor), _lib.stream_arg(stream), C.byref(out)))
        self._handle = out.value

    def _probe(self, name, probe, output_size, stream):
        lo, ro = C.c_void_p(), C.c_void_p()
        pv = probe._view()
        check(getattr(lib, name)(C.c_void_p(self._handle), C.byref(pv), 0 if output_size is None else 1, int(output_size or 0),
                                 _lib.stream_arg(stream), C.byref(lo), C.byref(ro)))
        return Column._from_handle(lo.value), Column._from_handle(ro.value)

    def _size(self, name, probe, stream):
        out = C.c_size_t(0)
        pv = probe._view()
        check(getattr(lib, name)(C.c_void_p(self._handle), C.byref(pv), _lib.stream_arg(stream), C.byref(out)))
        return out.value

    def inner_join(self, probe: Table, output_size: int | None = None, stream=None):
        return self._probe("b2_hash_join_inner_join", probe, output_size, stream)

    def left_join(self, probe: Table, output_size: int | None = None, stream=None):
        return self._probe("b2_hash_join_left_join", probe, output_size, stream)

    def full_join(self, probe: Table, output_size: int | None = None, stream=None):
        return self._probe("b2_hash_join_full_join", probe, output_size, stream)

    def inner_join_size(self, probe: Table, stream=None) -> int:
        return self._size("b2_hash_join_inner_join_size", probe, stream)

    def left_join_size(self, probe: Table, stream=None) -> int:
        return self._size("b2_hash_join_left_join_size", probe, stream)

    def full_join_size(self, probe: Table, stream=None) -> int:
        return self._size("b2_hash_join_full_join_size", probe, stream)

    # ---- match context / partitioned probes (hash_join.hpp:254-440) ---------------------------------
    def _match_context(self, kind: int, probe: Table, stream) -> "JoinMatchContext":
        out = C.c_void_p()
        pv = probe._view()
        check(lib.b2_hash_join_match_counts(C.c_void_p(self._handle), C.byref(pv), kind, _lib.stream_arg(stream), C.byref(out)))
        return JoinMatchContext(probe, Column._from_handle(out.value), kind)

    def inner_join_match_context(self, probe: Table, stream=None) -> "JoinMatchContext":
        return self._match_context(0, probe, stream)

    def left_join_match_context(self, probe: Table, stream=None) -> "JoinMatchContext":
        return self._match_context(1, probe, stream)

    def full_join_match_context(self, probe: Table, stream=None) -> "JoinMatchContext":
        return self._match_context(2, probe, stream)

    def _partitioned(self, kind: int, context: "JoinPartitionContext", stream):
        ctx = context.left_table_context
        if ctx is None or ctx._match_counts is None:
            raise ValueError("join_partition_context without a match context")
        lo, ro = C.c_void_p(), C.c_void_p()
        pv, cv = ctx._left_table._view(), ctx._match_counts._view()
        check(lib.b2_hash_join_partitioned_join(C.c_void_p(self._handle), C.byref(pv), C.byref(cv), int(context.left_start_idx),
                                                int(context.left_end_idx), kind, _lib.stream_arg(stream), C.byref(lo), C.byref(ro)))
        return Column._from_handle(lo.value), Column._from_handle(ro.value)

    def partitioned_inner_join(self, context: "JoinPartitionContext", stream=None):
        return self._partitioned(0, context, stream)

    def partitioned_left_join(self, context: "JoinPartitionContext", stream=None):
        return self._partitioned(1, context, stream)

    def partitioned_full_join(self, context: "JoinPartitionContext", stream=None):
        """Probe side only; finalize_partitioned_full_join appends the unmatched build rows."""
        return self._partitioned(2, context, stream)

    @staticmethod
    def finalize_partitioned_full_join(left_partials, right_partials, left_table_num_rows: int, right_table_num_rows: int, stream=None):
        n = len(left_partials)
        lv = (_lib.ColumnView * max(n, 1))(*[c._view() for c in left_partials])
        rv = (_lib.ColumnView * max(n, 1))(*[c._view() for c in right_partials])
        lo, ro = C.c_void_p(), C.c_void_p()
        check(lib.b2_hash_join_finalize_full_join(lv, rv, n, int(left_table_num_rows), int(right_table_num_rows), _lib.stream_arg(stream),
                                                  C.byref(lo), C.byref(ro)))
        return Column._from_handle(lo.value), Column._from_handle(ro.value)

    def __del__(self):
        if getattr(self, "_handle", 0):
            lib.b2_hash_join_destroy(C.c_void_p(self._handle))
            self._handle = 0


class JoinMatchContext:
    """cudf::join_match_context (join.hpp:81-107): the left table and its per-row match counts (INT32 column)."""

    def __init__(self, left_table: Table, match_counts: Column, kind: int = 0):
        self._left_table = left_table
        self._match_counts = match_counts
        self._kind = kind


class JoinPartitionContext:
    """cudf::join_partition_context (join.hpp:120-125)."""

    def __init__(self, left_table_context: JoinMatchContext, left_start_idx: int, left_end_idx: int):
        self.left_table_context = left_table_context
        self.left_start_idx = left_start_idx
        self.left_end_idx = left_end_idx

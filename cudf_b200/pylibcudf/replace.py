"""pylibcudf.replace twin (python/pylibcudf/pylibcudf/replace.pyx; cpp/include/cudf/replace.hpp) over b2_replace_nulls /
_scalar / _policy, b2_find_and_replace_all, b2_clamp and b2_normalize_nans_and_zeros / _inplace (cudf_b200/csrc/replace.cu: one
kernel per call).

Fixed-width columns only; decimal, dictionary, string and nested types are not held here. Semantics, undefined values and errors:
include/cudf_b200.h."""
from __future__ import annotations

import ctypes as C
import enum

from .. import _lib
from .._lib import check, lib
from .column import Column, Scalar


class ReplacePolicy(enum.IntEnum):  # cudf::replace_policy (cpp/include/cudf/replace.hpp:32): values are ABI
    PRECEDING = 0
    FOLLOWING = 1


def _new(fn, *args) -> Column:
    out = C.c_void_p()
    check(fn(*args, C.byref(out)))
    return Column._from_handle(out.value)


def replace_nulls(source_column: Column, replacement, stream=None, mr=None) -> Column:
    """Nulls of source_column replaced: by replacement[i] (a Column), by one value (a Scalar; the output has no mask), or by the
    nearest valid value before / after the row (a ReplacePolicy; a leading / trailing null run stays null)."""
    v = source_column._view()
    s = _lib.stream_arg(stream)
    if isinstance(replacement, Column):
        r = replacement._view()
        return _new(lib.b2_replace_nulls, C.byref(v), C.byref(r), s)
    if isinstance(replacement, Scalar):
        return _new(lib.b2_replace_nulls_scalar, C.byref(v), C.c_void_p(replacement._handle), s)
    if isinstance(replacement, ReplacePolicy):
        return _new(lib.b2_replace_nulls_policy, C.byref(v), int(replacement), s)
    raise TypeError("replacement must be a Column, Scalar, or replace_policy")


def find_and_replace_all(source_column: Column, values_to_replace: Column, replacement_values: Column, stream=None,
                         mr=None) -> Column:
    """Rows equal to values_to_replace[j] take replacement_values[j] (the first j among duplicates; -0.0 == +0.0, NaN matches
    nothing)."""
    v, o, r = source_column._view(), values_to_replace._view(), replacement_values._view()
    return _new(lib.b2_find_and_replace_all, C.byref(v), C.byref(o), C.byref(r), _lib.stream_arg(stream))


def clamp(source_column: Column, lo: Scalar, hi: Scalar, lo_replace: Scalar | None = None, hi_replace: Scalar | None = None,
          stream=None, mr=None) -> Column:
    """x < lo -> lo_replace (default lo), x > hi -> hi_replace (default hi); a null bound is not applied."""
    if (lo_replace is None) != (hi_replace is None):
        raise ValueError("lo_replace and hi_replace must be specified together")
    if lo_replace is None:
        lo_replace, hi_replace = lo, hi
    v = source_column._view()
    h = [C.c_void_p(x._handle) for x in (lo, lo_replace, hi, hi_replace)]
    return _new(lib.b2_clamp, C.byref(v), *h, _lib.stream_arg(stream))


def normalize_nans_and_zeros(source_column: Column, inplace: bool = False, stream=None, mr=None) -> Column | None:
    """Every NaN as quiet_NaN() and -0.0 as +0.0 (FLOAT32 / FLOAT64). inplace=True rewrites source_column's data and returns
    None."""
    v = source_column._view()
    if inplace:
        check(lib.b2_normalize_nans_and_zeros_inplace(C.byref(v), _lib.stream_arg(stream)))
        return None
    return _new(lib.b2_normalize_nans_and_zeros, C.byref(v), _lib.stream_arg(stream))


__all__ = ["ReplacePolicy", "clamp", "find_and_replace_all", "normalize_nans_and_zeros", "replace_nulls"]

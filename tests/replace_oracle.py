"""numpy restatement of cudf::replace_nulls, replace_nans, find_and_replace_all, clamp and normalize_nans_and_zeros over
fixed-width columns (cpp/src/replace/{nulls,nans,replace,clamp}.cu of the reference), as include/cudf_b200.h states them,
checks included: cudf::data_type_error is TypeError and cudf::logic_error RuntimeError, in the reference's order.

A column is (values, valid, type_id): valid None means no mask. A scalar is Scalar(value, valid, type_id). Every function
returns (values, valid) of the output, valid None when the output has no mask; values under null bits are not part of the
answer."""
from collections import namedtuple

import numpy as np

PRECEDING, FOLLOWING = 0, 1
FLOAT32, FLOAT64 = 9, 10

Scalar = namedtuple("Scalar", "value valid type")


def _valid(col):
    vals, valid, _ = col
    return np.ones(len(vals), bool) if valid is None else valid


def _has_nulls(col):
    return col[1] is not None and not col[1].all()


def copy(col):
    """A copy of the column; an empty column has no mask."""
    return col[0].copy(), None if col[1] is None or len(col[0]) == 0 else col[1].copy()


def replace_nulls_column(col, repl):
    """valid(in) ? in : repl; a mask only when repl has nulls; an input without nulls is a copy."""
    if col[2] != repl[2]:
        raise TypeError("Data type mismatch")
    if len(col[0]) != len(repl[0]):
        raise RuntimeError("Column size mismatch")
    vals, valid, _ = col
    if len(vals) == 0 or not _has_nulls(col):
        return copy(col)
    out = np.where(valid, vals, repl[0])
    return out, (valid | _valid(repl)) if _has_nulls(repl) else None


def replace_nulls_scalar(col, s):
    """Null rows take the scalar; no mask. An input without nulls or a null scalar is a copy, with no type check."""
    vals, valid, t = col
    if len(vals) == 0 or not _has_nulls(col) or not s.valid:
        return copy(col)
    if s.type != t:
        raise TypeError("Data type mismatch")
    return np.where(valid, vals, np.array(s.value, vals.dtype)), None


def replace_nulls_policy(col, policy):
    """The nearest valid row at or before (PRECEDING) / at or after (FOLLOWING) each row; a leading / trailing run stays null."""
    vals, valid, _ = col
    if len(vals) == 0 or not _has_nulls(col):
        return copy(col)
    n = len(vals)
    idx = np.arange(n)
    if policy == PRECEDING:
        src = np.maximum.accumulate(np.where(valid, idx, -1))
        ok = src >= 0
    else:
        src = np.minimum.accumulate(np.where(valid, idx, n)[::-1])[::-1]
        ok = src < n
    out = np.where(ok, vals[np.where(ok, src, 0)], 0).astype(vals.dtype)
    return out, ok


def replace_nans(col, repl):
    """A valid NaN row takes the replacement's value and validity (repl: a column or a Scalar). A mask when the input has
    nulls or the replacement a mask; the scalar form always has one."""
    vals, valid, t = col
    scalar = isinstance(repl, Scalar)
    if not scalar and len(repl[0]) != len(vals):
        raise RuntimeError("Input and replacement must be of the same size")
    if t not in (FLOAT32, FLOAT64):
        raise RuntimeError("NAN is not supported in a Non-floating point type column")
    if (repl.type if scalar else repl[2]) != t:
        raise RuntimeError("Input and replacement must be of the same type")
    if len(vals) == 0:
        return copy(col)
    v = _valid(col)
    nan = v & np.isnan(vals)
    rv = np.array(repl.value, vals.dtype) if scalar else repl[0]
    rok = np.full(len(vals), bool(repl.valid)) if scalar else _valid(repl)
    out = np.where(nan, rv, vals).astype(vals.dtype)
    ov = np.where(nan, rok, v)
    has_mask = _has_nulls(col) or scalar or repl[1] is not None
    return out, ov if has_mask else None


def find_and_replace_all(col, old, new):
    """C++ == (-0.0 == +0.0, NaN equals nothing); the first duplicate wins; a null new value nulls the row."""
    if len(old[0]) != len(new[0]):
        raise RuntimeError("values_to_replace and replacement_values size mismatch.")
    if not (col[2] == old[2] == new[2]):
        raise TypeError("Columns type mismatch")
    if _has_nulls(old):
        raise RuntimeError("values_to_replace must not have nulls")
    vals, valid, _ = col
    if len(vals) == 0 or len(old[0]) == 0:
        return copy(col)
    v = _valid(col)
    nv = _valid(new)
    o = old[0]
    keep = ~np.isnan(o) if o.dtype.kind == "f" else np.ones(len(o), bool)
    keys, first = np.unique(o[keep], return_index=True)  # the first occurrence of each value (-0.0 and +0.0 are one)
    pos = np.nonzero(keep)[0][first]
    out, ov = vals.copy(), v.copy()
    if len(keys):
        at = np.minimum(np.searchsorted(keys, vals), len(keys) - 1)
        hit = v & (keys[at] == vals)
        out[hit] = new[0][pos[at[hit]]]
        ov[hit] = nv[pos[at[hit]]]
    has_mask = _has_nulls(col) or _has_nulls(new)
    return out, ov if has_mask else None


def clamp(col, lo, lo_replace, hi, hi_replace):
    """lo / hi / replacements: Scalar; x < lo -> lo_replace, x > hi -> hi_replace; a null bound is not applied; the input's
    mask."""
    if lo.type != hi.type:
        raise TypeError("mismatching types of limit scalars")
    if lo_replace.type != hi_replace.type:
        raise TypeError("mismatching types of replace scalars")
    if lo.type != lo_replace.type:
        raise TypeError("mismatching types of limit and replace scalars")
    vals, valid, t = col
    if len(vals) == 0 or (not lo.valid and not hi.valid):
        return copy(col)
    if lo.valid and not lo_replace.valid:
        raise RuntimeError("lo_replace can't be null if lo is not null")
    if hi.valid and not hi_replace.valid:
        raise RuntimeError("hi_replace can't be null if hi is not null")
    if t != lo.type:
        raise TypeError("mismatching types of scalar and input")
    out = vals.copy()
    if lo.valid:
        out = np.where(vals < np.array(lo.value, vals.dtype), np.array(lo_replace.value, vals.dtype), out)
    if hi.valid:
        out = np.where(vals > np.array(hi.value, vals.dtype), np.array(hi_replace.value, vals.dtype), out)
    return out.astype(vals.dtype), None if valid is None else valid.copy()


def normalize_nans_and_zeros(col):
    """Every NaN as the canonical quiet NaN, -0.0 as +0.0 (bit for bit); the input's mask."""
    vals, valid, t = col
    if len(vals) == 0:
        return copy(col)
    if t not in (FLOAT32, FLOAT64):
        raise RuntimeError("Expects float or double input")
    out = vals.copy()
    out[np.isnan(out)] = np.array(np.nan, vals.dtype)  # numpy's nan is C's quiet_NaN() pattern
    out[out == 0] = 0
    return out, None if valid is None else valid.copy()

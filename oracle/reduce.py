"""reduce / scan / segmented_reduce semantics:
  cpp/src/reductions/reductions.cpp:474-536, simple.cuh:47-85,373-447 (accumulator rule), compound.cuh (mean)
  cpp/src/reductions/scan/{scan.cpp,scan_inclusive.cu:36-145,198-240,scan_exclusive.cu:32-104}
  cpp/src/reductions/segmented/{reductions.cpp:112-168,simple.cuh:57-104}; validity rule
  cpp/include/cudf/detail/null_mask.cuh:785-843."""
from __future__ import annotations

import numpy as np

SUM, PRODUCT, MIN, MAX, COUNT_VALID, COUNT_ALL, MEAN = 0, 2, 3, 4, 5, 6, 10
EXCLUDE, INCLUDE = 0, 1


def _identity(kind, dtype):
    dtype = np.dtype(dtype)
    if kind == SUM:
        return dtype.type(0)
    if kind == PRODUCT:
        return dtype.type(1)
    if dtype.kind == "f":
        return dtype.type(np.inf if kind == MIN else -np.inf)
    if dtype == np.bool_:
        return np.bool_(kind == MIN)
    info = np.iinfo(dtype)
    return dtype.type(info.max if kind == MIN else info.min)


def _acc_dtype(in_dtype, out_dtype):
    """simple.cuh:407-412: same type -> accumulate in it; else int64 for integral inputs, double otherwise."""
    in_dtype, out_dtype = np.dtype(in_dtype), np.dtype(out_dtype)
    if in_dtype == out_dtype:
        return in_dtype
    return np.dtype(np.int64) if in_dtype.kind in "iub" else np.dtype(np.float64)


def _fold(kind, x, acc_dtype):
    with np.errstate(over="ignore", invalid="ignore"):
        if kind == SUM:
            if acc_dtype == np.bool_:
                return np.bool_(x.any())
            return x.sum(dtype=acc_dtype) if len(x) else acc_dtype.type(0)
        if kind == PRODUCT:
            if acc_dtype == np.bool_:
                return np.bool_(x.all())
            return x.prod(dtype=acc_dtype) if len(x) else acc_dtype.type(1)
        if kind == MIN:
            # NaN ranks above +inf: fmin is NaN only when every value is NaN (maximum propagates NaN already)
            return np.fmin.reduce(x) if len(x) else _identity(MIN, acc_dtype)
        if kind == MAX:
            return x.max() if len(x) else _identity(MAX, acc_dtype)
    raise ValueError(kind)


def reduce(values, valid, kind, out_dtype, init=None):
    """-> (value | None, is_valid). init = (value, is_valid) or None."""
    values = np.asarray(values)
    out_dtype = np.dtype(out_dtype)
    n = len(values)
    nvalid = n if valid is None else int(np.asarray(valid).sum())
    if kind in (MIN, MAX) and values.dtype != out_dtype:
        raise RuntimeError("min/max operation requires matching output type")
    if nvalid == 0:
        return None, False  # reduce_no_data: invalid default scalar
    x = values if valid is None else values[np.asarray(valid)]
    if kind == MEAN:
        if out_dtype.kind != "f":
            raise TypeError("Unsupported output data type")
        s = x.astype(out_dtype).sum(dtype=out_dtype)
        return out_dtype.type(s / out_dtype.type(nvalid)), True
    acc = _acc_dtype(values.dtype, out_dtype)
    r = _fold(kind, x.astype(acc) if acc != np.bool_ else x.astype(bool), acc)
    ok = True
    if init is not None:
        iv, ivalid = init
        if ivalid:
            r = _fold(kind, np.array([r, acc.type(iv)], dtype=acc), acc)
        ok = bool(ivalid)
    with np.errstate(over="ignore", invalid="ignore"):
        return (np.array([r]).astype(out_dtype)[0] if out_dtype != np.bool_ else np.bool_(r != 0)), ok


def scan(values, valid, kind, inclusive=True, null_handling=EXCLUDE):
    """-> (values, valid | None); output type == input type (INT32 for counts)."""
    values = np.asarray(values)
    n = len(values)
    nullable = valid is not None
    v = np.ones(n, bool) if valid is None else np.asarray(valid, dtype=bool)
    # output mask
    if null_handling == EXCLUDE:
        out_valid = v.copy() if nullable else None
    elif nullable:
        nulls = np.nonzero(~v)[0]
        first = int(nulls[0]) if len(nulls) else n
        pos = min(n, first + (0 if inclusive else 1))
        out_valid = np.arange(n) < pos
    else:
        out_valid = None
    if kind in (COUNT_VALID, COUNT_ALL):
        ones = np.ones(n, dtype=np.int32)
        if kind == COUNT_VALID and out_valid is not None:
            ones = out_valid.astype(np.int32)
        c = np.cumsum(ones, dtype=np.int32)
        if not inclusive:
            c = np.concatenate([[0], c[:-1]]).astype(np.int32)
        return c, out_valid
    dt = values.dtype
    ident = _identity(kind, dt)
    x = np.where(v, values, ident).astype(dt)
    with np.errstate(over="ignore", invalid="ignore"):
        if kind == SUM:
            r = np.cumsum(x, dtype=dt) if dt != np.bool_ else np.logical_or.accumulate(x)
        elif kind == PRODUCT:
            r = np.cumprod(x, dtype=dt) if dt != np.bool_ else np.logical_and.accumulate(x)
        elif kind == MIN:
            # NaN ranks above +inf, so a prefix is NaN only while all its valid values are; nulls take NaN, the top
            r = np.fmin.accumulate(np.where(v, values, np.nan).astype(dt) if dt.kind == "f" else x)
        elif kind == MAX:
            r = np.maximum.accumulate(x)
        else:
            raise RuntimeError("Unsupported aggregation operator for scan")
    if not inclusive:
        r = np.concatenate([np.array([ident], dtype=dt), r[:-1]]).astype(dt) if n else r
        if kind == MIN and dt.kind == "f":
            r[: (int(np.argmax(v)) if v.any() else n) + 1] = ident  # an empty prefix: +inf, as in the reference
    return r, out_valid


def segmented_reduce(values, valid, offsets, kind, out_dtype, null_handling=EXCLUDE, init=None):
    """-> (values, valid). valid rule: null_mask.cuh:833-840 (a mask is always produced)."""
    values = np.asarray(values)
    out_dtype = np.dtype(out_dtype)
    offsets = np.asarray(offsets, dtype=np.int64)
    if len(values) == 0 and len(offsets) == 0:
        return np.empty(0, dtype=out_dtype), None
    if len(offsets) == 0:
        raise RuntimeError("`offsets` should have at least 1 element.")
    nseg = len(offsets) - 1
    mean = kind == MEAN
    acc = np.dtype(out_dtype) if mean else _acc_dtype(values.dtype, out_dtype)
    has_init = init is not None
    init_valid = bool(init[1]) if has_init else False
    out = np.empty(nseg, dtype=out_dtype)
    ov = np.empty(nseg, dtype=bool)
    for s in range(nseg):
        b, e = offsets[s], offsets[s + 1]
        seg = values[b:e]
        m = np.ones(e - b, bool) if valid is None else np.asarray(valid[b:e], dtype=bool)
        x = seg[m]
        r = _fold(SUM if mean else kind, x.astype(acc) if acc != np.bool_ else x.astype(bool), acc)
        if has_init and init_valid:
            r = _fold(kind, np.array([acc.type(init[0]), r], dtype=acc), acc)
        if mean and len(x):
            r = acc.type(r / acc.type(len(x)))
        with np.errstate(over="ignore", invalid="ignore"):
            out[s] = np.array([r]).astype(out_dtype)[0] if out_dtype != np.bool_ else (r != 0)
        length, vc = e - b, int(m.sum())
        if valid is None:
            ov[s] = init_valid if has_init else length > 0
        elif null_handling == EXCLUDE:
            ov[s] = init_valid or vc > 0
        else:
            ov[s] = (init_valid if has_init else length > 0) and vc == length
    return out, ov

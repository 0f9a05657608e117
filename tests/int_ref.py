"""Exact references for integer reductions, scans, segmented reductions and groupby aggregations, in Python ints.

The reference's rules, applied explicitly:
- Accumulator: the input type when the output type is the input type; otherwise int64 for integral inputs (BOOL8 included)
  (cpp/src/reductions/simple.cuh:407-419, segmented/simple.cuh reduce_numeric). Sums and products wrap modulo 2^64 into the
  accumulator's range; a narrower accumulator wraps modulo its own width.
- Conversion of an integer to FLOAT64 / FLOAT32: one correctly rounded step (round half to even) from the exact integer, as
  C++ `(double)int64_t` / `(float)int64_t` do. int -> double -> float32 would round twice.
- reduce / segmented_reduce MEAN: each value converted to the output float type, then summed in that type (compound.cuh); the
  result depends on the summation order, so `mean_terms` returns the converted values for a bound check (tests/exact_ref.py).
- groupby MEAN (hash and sort paths): double(wrapped INT64 SUM) / double(valid count), exactly rounded: compared bit for bit.
- groupby SUM / PRODUCT / SUM_OF_SQUARES of integers: INT64, wrapping; MIN / MAX in the value type.
Values are numpy arrays; results are Python ints, floats or bools (None for a null result).
"""
from __future__ import annotations

import math

import numpy as np

SUM, PRODUCT, MIN, MAX, MEAN = "sum", "product", "min", "max", "mean"


def bounds(dt):
    """(min, max) of an integral dtype (BOOL8: 0, 1)."""
    dt = np.dtype(dt)
    if dt == np.bool_:
        return 0, 1
    if dt.kind == "m":
        dt = np.dtype(np.int64)
    i = np.iinfo(dt)
    return int(i.min), int(i.max)


def wrap(i: int, dt) -> int:
    """i modulo 2^bits into the range of the integral dtype (two's complement), as a C++ integer conversion does."""
    dt = np.dtype(dt)
    if dt == np.bool_:
        return int(i != 0)
    bits = dt.itemsize * 8
    i &= (1 << bits) - 1
    if dt.kind in "im" and i >= 1 << (bits - 1):
        i -= 1 << bits
    return i


def round_int(i: int, mant_bits: int) -> float:
    """The integer i rounded to mant_bits significant bits, half to even (exact in a Python float for 24 and 53 bits)."""
    a = abs(i)
    n = a.bit_length()
    if n > mant_bits:
        shift = n - mant_bits
        q, r = divmod(a, 1 << shift)
        half = 1 << (shift - 1)
        if r > half or (r == half and q & 1):
            q += 1
        a = q << shift
    return math.copysign(float(a), -1.0 if i < 0 else 1.0) if a else 0.0


def to_float(i: int, dt) -> float:
    """C++ conversion of an integer to float / double: correctly rounded from the exact value."""
    return round_int(i, 24 if np.dtype(dt) == np.float32 else 53)


def convert(i: int, out_dt):
    """An accumulator value (integer) as the output type."""
    out_dt = np.dtype(out_dt)
    if out_dt.kind == "f":
        return to_float(i, out_dt)
    if out_dt == np.bool_:
        return i != 0
    return wrap(i, out_dt)


def ints(vals, valid=None):
    """The valid values as Python ints."""
    v = np.asarray(vals)
    if v.dtype.kind == "m":
        v = v.view(np.int64)
    x = [int(a) for a in v.tolist()]
    return x if valid is None else [a for a, ok in zip(x, np.asarray(valid, bool).tolist()) if ok]


def fold(kind, xs, acc_dt, start=None):
    """SUM / PRODUCT / MIN / MAX of ints xs in the accumulator type acc_dt (wrapping); start: a first operand (an initial value).
    Wrapping commutes with + and *, so a sum or product is wrapped once at the end; MIN / MAX compare the values themselves
    (their accumulator is always the value type)."""
    acc_dt = np.dtype(acc_dt)
    if start is not None:
        xs = [start] + list(xs)
    if kind == SUM:
        return wrap(sum(xs), acc_dt)
    if kind == PRODUCT:
        r = 1
        for a in xs:
            r = (r * a) & 0xFFFFFFFFFFFFFFFF  # the low 64 bits are all that any accumulator keeps
            if r == 0:
                break
        return wrap(r, acc_dt)
    if not xs:
        return None
    return min(xs) if kind == MIN else max(xs)


def acc_dtype(in_dt, out_dt):
    in_dt, out_dt = np.dtype(in_dt), np.dtype(out_dt)
    return in_dt if in_dt == out_dt else np.dtype(np.int64)


def reduce(vals, valid, kind, out_dt, init=None):
    """cudf::reduce of an integral column -> (value | None, valid). init = (value, valid) or None. Not MEAN (see mean_terms)."""
    return reduce_ints(ints(vals, valid), np.asarray(vals).dtype, kind, out_dt, init)


def reduce_ints(xs, in_dt, kind, out_dt, init=None):
    """reduce() over the valid values already as Python ints (lets a caller convert a long column once)."""
    in_dt, out_dt = np.dtype(in_dt), np.dtype(out_dt)
    if not xs:
        return None, False  # no valid value: an invalid scalar, whatever the initial value
    acc = acc_dtype(in_dt, out_dt)
    ok = True
    start = None
    if init is not None:
        ok = bool(init[1])
        if ok:
            start = int(init[0])
    r = fold(kind, xs, acc, start)
    return convert(r, out_dt), ok


def mean_terms(vals, valid, out_dt):
    """The valid values converted one by one to the output float type: MEAN sums these in that type and divides by their count."""
    return [to_float(a, out_dt) for a in ints(vals, valid)]


def segmented_reduce(vals, valid, offsets, kind, out_dt, include_nulls=False, init=None):
    """-> [(value | None, valid)] per segment; validity rule of cpp/include/cudf/detail/null_mask.cuh:833-840. Not MEAN."""
    in_dt = np.asarray(vals).dtype
    acc = acc_dtype(in_dt, out_dt)
    out = []
    has_init = init is not None
    init_valid = has_init and bool(init[1])
    for b, e in zip(offsets[:-1], offsets[1:]):
        seg_valid = None if valid is None else np.asarray(valid[b:e], bool)
        xs = ints(vals[b:e], seg_valid)
        length, vc = e - b, len(xs)
        if valid is None:
            ok = init_valid if has_init else length > 0
        elif not include_nulls:
            ok = init_valid or vc > 0
        else:
            ok = (init_valid if has_init else length > 0) and vc == length
        r = fold(kind, xs, acc, int(init[0]) if init_valid else None)
        out.append((convert(r, out_dt) if ok and r is not None else None, ok))
    return out


def scan(vals, valid, kind, inclusive=True, include_nulls=False):
    """cudf::scan (output type == input type) -> (values with None where null, valid mask | None)."""
    dt = np.asarray(vals).dtype
    x = ints(vals)
    n = len(x)
    v = [True] * n if valid is None else np.asarray(valid, bool).tolist()
    if not include_nulls:
        out_valid = None if valid is None else list(v)
    elif valid is not None:
        first = v.index(False) if False in v else n
        pos = min(n, first + (0 if inclusive else 1))
        out_valid = [i < pos for i in range(n)]
    else:
        out_valid = None
    lo, hi = bounds(dt)
    ident = {SUM: 0, PRODUCT: 1, MIN: hi, MAX: lo}[kind]
    run = ident
    res = []
    for i in range(n):
        before = run
        if v[i]:
            a = x[i] if dt != np.bool_ else int(x[i] != 0)
            if kind == SUM:
                run = wrap(run + a, dt)
            elif kind == PRODUCT:
                run = wrap(run * a, dt)
            elif kind == MIN:
                run = min(run, a)
            else:
                run = max(run, a)
        r = run if inclusive else before
        res.append(r if out_valid is None or out_valid[i] else None)
    if dt == np.bool_:
        res = [None if r is None else bool(r) for r in res]
    return res, out_valid


# ---- groupby ----------------------------------------------------------------------------------------------------------
def group_rows(keys, kmask=None, include_nulls=False):
    """{key (None for the null key): row indices in row order}."""
    k = np.asarray(keys)
    if k.dtype.kind == "m":
        k = k.view(np.int64)
    out = {}
    km = None if kmask is None else np.asarray(kmask, bool).tolist()
    for r, key in enumerate(k.tolist()):
        if km is not None and not km[r]:
            if not include_nulls:
                continue
            key = None
        out.setdefault(key, []).append(r)
    return out


def prepare(vals, valid):
    """(dtype, values as Python ints, validity as a list): a column converted once for many group_agg / group_scan calls."""
    x = ints(vals)
    return np.asarray(vals).dtype, x, [True] * len(x) if valid is None else np.asarray(valid, bool).tolist()


def group_agg(vals, valid, rows, kind, prepared=None):
    """One group's aggregation over rows (hash and sort paths alike) -> (value | None, valid), or ([rows holding it], valid)
    for ARG*. kinds: sum, product, min, max, mean, sum_of_squares, count, count_all, argmin, argmax."""
    dt, x, ok = prepared or prepare(vals, valid)
    vr = [r for r in rows if ok[r]]
    xs = [x[r] for r in vr]
    if kind == "count":
        return len(xs), True
    if kind == "count_all":
        return len(rows), True
    if not xs:
        return None, False
    i64 = np.dtype(np.int64)
    if kind == "sum":
        return fold(SUM, xs, i64), True
    if kind == "product":
        return fold(PRODUCT, xs, i64), True
    if kind == "sum_of_squares":
        return wrap(sum(wrap(wrap(a, i64) * wrap(a, i64), i64) for a in xs), i64), True
    if kind == "mean":
        return to_float(fold(SUM, xs, i64), np.float64) / float(len(xs)), True
    if kind in ("min", "max", "argmin", "argmax"):
        ext = min(xs) if kind in ("min", "argmin") else max(xs)
        if kind in ("min", "max"):
            return (ext if dt != np.bool_ else bool(ext)), True
        return [r for r, a in zip(vr, xs) if a == ext], True
    raise ValueError(kind)


def group_scan(vals, valid, rows, kind, prepared=None):
    """Grouped inclusive scan over one group's rows (in order) -> [value | None] per row. SUM in INT64 (wrapping), MIN / MAX in
    the value type, COUNT (valid rows so far); a null row gives a null result (SUM / MIN / MAX) and is skipped by the scan."""
    _, x, ok = prepared or prepare(vals, valid)
    out, run, cnt = [], None, 0
    i64 = np.dtype(np.int64)
    for r in rows:
        if kind == "count":
            cnt += ok[r]
            out.append(cnt)
            continue
        if ok[r]:
            a = x[r]
            if kind == "sum":
                run = wrap((run or 0) + a, i64)
            elif run is None:
                run = a
            else:
                run = min(run, a) if kind == "min" else max(run, a)
            out.append(run)
        else:
            out.append(None)
    return out

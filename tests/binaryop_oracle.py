"""cudf::binary_operation semantics restated in numpy (cpp/src/binaryop/binaryop.cpp and cpp/src/binaryop/compiled/ of the
reference, as include/cudf_b200.h states them).

An operand is (values, valid, type_id): values a numpy array of the storage type (chrono operands as their integers), valid a
bool array or None; a scalar operand has 0-d values and a bool validity. `binop` returns the output values, validity and a
`defined` mask: the rows whose value C++ defines (division by zero, INT_MIN / -1, out-of-range shifts and float-to-integer
conversions, integer-only operators with a float compute type are not). Tests compare values at rows both valid and defined."""
from __future__ import annotations

import numpy as np

INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8 = range(1, 12)
NUMERIC = list(range(1, 12))
NP = {INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, UINT8: np.uint8, UINT16: np.uint16, UINT32: np.uint32,
      UINT64: np.uint64, FLOAT32: np.float32, FLOAT64: np.float64, BOOL8: np.bool_}
TIMESTAMP_DAYS, DURATION_NANOSECONDS = 12, 21
NUM_TYPE_IDS = 29

(ADD, SUB, MUL, DIV, TRUE_DIV, FLOOR_DIV, MOD, PMOD, PYMOD, POW, INT_POW, LOG_BASE, ATAN2, SHIFT_LEFT, SHIFT_RIGHT,
 SHIFT_RIGHT_UNSIGNED, BITWISE_AND, BITWISE_OR, BITWISE_XOR, LOGICAL_AND, LOGICAL_OR, EQUAL, NOT_EQUAL, LESS, GREATER, LESS_EQUAL,
 GREATER_EQUAL, NULL_EQUALS, NULL_NOT_EQUALS, NULL_MAX, NULL_MIN, GENERIC_BINARY, NULL_LOGICAL_AND, NULL_LOGICAL_OR,
 INVALID_BINARY) = range(35)
ALL_OPS = [op for op in range(34) if op != GENERIC_BINARY]
NULL_AWARE = {NULL_EQUALS, NULL_NOT_EQUALS, NULL_MAX, NULL_MIN, NULL_LOGICAL_AND, NULL_LOGICAL_OR}
BOOL_OPS = {LOGICAL_AND, LOGICAL_OR, EQUAL, NOT_EQUAL, LESS, GREATER, LESS_EQUAL, GREATER_EQUAL, NULL_EQUALS, NULL_NOT_EQUALS,
            NULL_LOGICAL_AND, NULL_LOGICAL_OR}
INTEGER_OPS = {INT_POW, SHIFT_LEFT, SHIFT_RIGHT, SHIFT_RIGHT_UNSIGNED, BITWISE_AND, BITWISE_OR, BITWISE_XOR}
COMPARISONS = {EQUAL, NOT_EQUAL, LESS, GREATER, LESS_EQUAL, GREATER_EQUAL}
DOUBLE_OPS = {TRUE_DIV, POW, LOG_BASE, ATAN2}  # computed in double whatever C is
INEXACT_OPS = {POW, LOG_BASE, ATAN2}          # libm results: compared within a few ulp


def is_chrono(t: int) -> bool:
    return TIMESTAMP_DAYS <= t <= DURATION_NANOSECONDS


def storage(t: int) -> int:
    if is_chrono(t):
        return INT32 if t in (12, 17) else INT64
    return t


def _width(t: int) -> int:
    return np.dtype(NP[t]).itemsize


def _signed(t: int) -> bool:
    return t in (INT8, INT16, INT32, INT64)


def _integral(t: int) -> bool:
    return t not in (FLOAT32, FLOAT64)


def common_type(a: int, b: int) -> int:
    """std::common_type of two numeric types: a type with itself is itself; otherwise the usual arithmetic conversions."""
    if a == b:
        return a
    if FLOAT64 in (a, b):
        return FLOAT64
    if FLOAT32 in (a, b):
        return FLOAT32
    a, b = (INT32 if _width(a) < 4 else a), (INT32 if _width(b) < 4 else b)
    if a == b:
        return a
    if _signed(a) == _signed(b):
        return a if _width(a) >= _width(b) else b
    s, u = (a, b) if _signed(a) else (b, a)
    return u if _width(u) >= _width(s) else s


def is_supported(out: int, lhs: int, rhs: int, op: int) -> bool:
    """cpp/src/binaryop/compiled/util.cpp over the numeric types; chrono only against the same type (comparisons -> BOOL8,
    NULL_MAX / NULL_MIN -> the same type)."""
    for t in (out, lhs, rhs):
        if not 0 <= t < NUM_TYPE_IDS:
            raise RuntimeError("Invalid type_id")
    if is_chrono(lhs) or is_chrono(rhs):
        if lhs != rhs:
            return False
        if op in COMPARISONS or op in (NULL_EQUALS, NULL_NOT_EQUALS):
            return out == BOOL8
        if op in (NULL_MAX, NULL_MIN):
            return out == lhs
        return False
    if not all(t in NUMERIC for t in (out, lhs, rhs)):
        return False
    if op in BOOL_OPS:
        return out == BOOL8
    c = common_type(lhs, rhs)
    if op == SHIFT_RIGHT_UNSIGNED:
        return _integral(c) and c != BOOL8
    if op in INTEGER_OPS:
        return _integral(c)
    return ADD <= op <= ATAN2 or op in (NULL_MAX, NULL_MIN)


def compute_type(out: int, lhs: int, rhs: int) -> int:
    """C = std::common_type<out, lhs, rhs> (a chrono pair: its storage type)."""
    if is_chrono(lhs):
        return storage(lhs)
    return common_type(common_type(out, lhs), rhs)


def _unsigned_of(t):
    return {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[np.dtype(t).itemsize]


def _int_pow(x, y):
    """Exponentiation by squaring with wrap-around, x and y of one integer dtype; 0 for a negative exponent."""
    ut = _unsigned_of(x.dtype)
    b, e = x.astype(ut), y.astype(ut)
    r = np.ones_like(b)
    for _ in range(8 * np.dtype(ut).itemsize):
        r = np.where(e & ut(1), r * b, r)
        b = b * b
        e = e >> ut(1)
    r = r.astype(x.dtype)
    r = np.where(y == 0, x.dtype.type(1), np.where(x == 0, x.dtype.type(0), r))
    if np.dtype(x.dtype).kind == "i":
        r = np.where(y < 0, x.dtype.type(0), r)
    return r


def _c_div(x, y):
    """C++ integer division (truncation), y != 0."""
    if x.dtype.kind == "u":
        return x // y
    q = np.floor_divide(x, y)
    fix = (x - q * y != 0) & ((x < 0) != (y < 0))
    return q + fix.astype(x.dtype)


def _values(op, x, y, c):
    """op in compute type c: x, y already converted to c. Returns (result, defined)."""
    p = INT32 if (_integral(c) and _width(c) < 4) else c  # integral promotion
    pt = NP[p]
    n = len(x)
    defined = np.ones(n, bool)
    if op in INTEGER_OPS and not _integral(c):
        return np.zeros(n, pt), np.zeros(n, bool)
    if op == SHIFT_RIGHT_UNSIGNED:
        u = x.astype(_unsigned_of(NP[c]))
        u = u.astype(np.int32) if _width(c) < 4 else u
        w = 8 * u.dtype.itemsize
        yy = y.astype(np.int64)
        defined = (yy >= 0) & (yy < w)
        return u >> np.where(defined, yy, 0).astype(u.dtype), defined
    x, y = x.astype(pt), y.astype(pt)
    integral = _integral(p)
    if integral and op in (DIV, FLOOR_DIV, MOD, PMOD, PYMOD):
        defined = y != 0
        if _signed(p):
            defined &= ~((x == np.iinfo(pt).min) & (y == -1))
        y = np.where(defined, y, pt(1))
        x = np.where(defined, x, pt(0))
    if op == ADD:
        return x + y, defined
    if op == SUB:
        return x - y, defined
    if op == MUL:
        return x * y, defined
    if op == DIV:
        return (_c_div(x, y) if integral else x / y), defined
    if op == TRUE_DIV:
        return x.astype(np.float64) / y.astype(np.float64), defined
    if op == FLOOR_DIV:
        return (x // y if integral else np.floor(x / y)), defined  # numpy's integer // rounds toward -inf
    if op == MOD:
        return np.fmod(x, y), defined
    if op == PMOD:
        r = np.fmod(x, y)
        if integral and not _signed(p):
            return r, defined
        return np.where(r < 0, np.fmod(r + y, y), r), defined
    if op == PYMOD:
        if integral:
            return np.fmod(np.fmod(x, y) + y, y), defined
        a, b = x.astype(np.float64), y.astype(np.float64)
        return np.fmod(np.fmod(a, b) + b, b), defined
    if op == POW:
        return np.power(x.astype(np.float64), y.astype(np.float64)), defined
    if op == INT_POW:
        return _int_pow(x, y), defined
    if op == LOG_BASE:
        return np.log(x.astype(np.float64)) / np.log(y.astype(np.float64)), defined
    if op == ATAN2:
        return np.arctan2(x.astype(np.float64), y.astype(np.float64)), defined
    if op in (SHIFT_LEFT, SHIFT_RIGHT):
        w = 8 * np.dtype(pt).itemsize
        yy = y.astype(np.int64)
        defined = (yy >= 0) & (yy < w)
        s = np.where(defined, yy, 0)
        if op == SHIFT_LEFT:
            ut = _unsigned_of(pt)
            return (x.astype(ut) << s.astype(ut)).astype(pt), defined
        return x >> s.astype(pt), defined
    if op == BITWISE_AND:
        return x & y, defined
    if op == BITWISE_OR:
        return x | y, defined
    if op == BITWISE_XOR:
        return x ^ y, defined
    if op == LOGICAL_AND:
        return (x != 0) & (y != 0), defined
    if op == LOGICAL_OR:
        return (x != 0) | (y != 0), defined
    cmp = {EQUAL: np.equal, NOT_EQUAL: np.not_equal, LESS: np.less, GREATER: np.greater, LESS_EQUAL: np.less_equal,
           GREATER_EQUAL: np.greater_equal}
    return cmp[op](x, y), defined


def _cast(r, out):
    """static_cast<Out>(r); also returns where the conversion is defined."""
    ot = NP[storage(out)]
    if out == BOOL8:
        return r != 0, np.ones(len(r), bool)
    defined = np.ones(len(r), bool)
    if r.dtype.kind == "f" and np.dtype(ot).kind in "iu":
        info = np.iinfo(ot)
        t = np.trunc(r.astype(np.float64))
        # the bounds as doubles: 2^63 and 2^64 are exact, so `t < max + 1` is the exact test
        defined = ~np.isnan(t) & (t >= float(info.min)) & (t < float(info.max) + 1.0)
        r = np.where(defined, r, 0)
    return r.astype(ot), defined


def _broadcast(operand, n):
    vals, valid, t = operand
    vals = np.asarray(vals)
    if vals.ndim == 0:
        return np.full(n, vals, dtype=vals.dtype), np.full(n, bool(valid)), t
    return vals, (np.ones(n, bool) if valid is None else np.asarray(valid, bool)), t


def binop(op: int, lhs, rhs, out: int):
    """(values, valid, defined, nullable) of binary_operation(lhs, rhs, op, out); nullable = the output carries a mask.
    Raises as the library does: ValueError (size mismatch), RuntimeError (type id), TypeError (unsupported)."""
    lcol, rcol = np.asarray(lhs[0]).ndim == 1, np.asarray(rhs[0]).ndim == 1
    if lcol and rcol and len(lhs[0]) != len(rhs[0]):
        raise ValueError("Column sizes don't match")
    if not is_supported(out, lhs[2], rhs[2], op):
        raise TypeError("Unsupported operator for these types")
    n = len(lhs[0]) if lcol else len(rhs[0])
    (lv, lm, lt), (rv, rm, rt) = _broadcast(lhs, n), _broadcast(rhs, n)
    c = compute_type(out, lt, rt)
    with np.errstate(all="ignore"):
        x = lv.astype(NP[storage(lt)]).astype(NP[c])
        y = rv.astype(NP[storage(rt)]).astype(NP[c])
        if op in NULL_AWARE:
            both = lm & rm
            if op in (NULL_EQUALS, NULL_NOT_EQUALS):
                eq = np.where(both, x == y, ~lm & ~rm)
                r, valid = (eq if op == NULL_EQUALS else ~eq), np.ones(n, bool)
            elif op in (NULL_MAX, NULL_MIN):
                pick = (x > y) if op == NULL_MAX else (x < y)
                r = np.where(both, np.where(pick, x, y), np.where(lm, x, y))
                valid = lm | rm
            else:
                xt, yt = x != 0, y != 0
                if op == NULL_LOGICAL_AND:
                    lf, rf = lm & ~xt, rm & ~yt
                    r, valid = both & ~lf & ~rf, lf | rf | both
                else:
                    lt_, rt_ = lm & xt, rm & yt
                    r, valid = lt_ | rt_, lt_ | rt_ | both
            defined = np.ones(n, bool)
        else:
            r, defined = _values(op, x, y, c)
            valid = lm & rm
        vals, cast_ok = _cast(np.asarray(r), out)
    has_nulls = [(v is not None and not np.all(v)) if col else not bool(v) for (_, v, _), col in ((lhs, lcol), (rhs, rcol))]
    nullable = n > 0 and (op in NULL_AWARE or any(has_nulls))  # an empty output has no mask
    return vals, valid, defined & cast_ok, nullable

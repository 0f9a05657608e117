"""cudf::unary_operation, cast, is_null / is_valid and is_nan / is_not_nan restated in numpy (cpp/src/unary/ of the reference, as
include/cudf_b200.h states it). Chrono arithmetic uses Python ints.

A column is (values, valid, type_id): values a numpy array of the storage type (chrono columns as their integers), valid a bool
array or None. `unary` and `cast` return (values, valid, defined): `valid` is the input's (None when it has no mask) and
`defined` marks the rows whose value C++ defines (float -> integer conversions out of range or of NaN, ABS / NEGATE of the
32- and 64-bit minima, chrono results out of the target's range are not). Unsupported pairs raise the classes the library maps
its errors to: RuntimeError (cudf::logic_error) and TypeError (cudf::data_type_error)."""
from __future__ import annotations

import numpy as np

INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8 = range(1, 12)
NUMERIC = list(range(1, 12))
TIMESTAMP_D, TIMESTAMP_S, TIMESTAMP_MS, TIMESTAMP_US, TIMESTAMP_NS = range(12, 17)
TIMESTAMPS = list(range(12, 17))
DURATIONS = list(range(17, 22))
FIXED_WIDTH = list(range(1, 22))
DECIMALS = [25, 26, 27]
NUM_TYPE_IDS = 29
NP = {INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, UINT8: np.uint8, UINT16: np.uint16, UINT32: np.uint32,
      UINT64: np.uint64, FLOAT32: np.float32, FLOAT64: np.float64, BOOL8: np.bool_}
for _t in TIMESTAMPS + DURATIONS:
    NP[_t] = np.int32 if _t in (12, 17) else np.int64

(SIN, COS, TAN, ARCSIN, ARCCOS, ARCTAN, SINH, COSH, TANH, ARCSINH, ARCCOSH, ARCTANH, EXP, LOG, SQRT, CBRT, CEIL, FLOOR, ABS, RINT,
 BIT_COUNT, BIT_INVERT, NOT, NEGATE) = range(24)
ALL_OPS = list(range(24))
# libm results on float inputs: compared within 4 ulp of the float64 oracle (rounded to float32 for FLOAT32)
INEXACT_OPS = {SIN, COS, TAN, ARCSIN, ARCCOS, ARCTAN, SINH, COSH, TANH, ARCSINH, ARCCOSH, ARCTANH, EXP, LOG, CBRT}
_NUMPY_FN = {SIN: np.sin, COS: np.cos, TAN: np.tan, ARCSIN: np.arcsin, ARCCOS: np.arccos, ARCTAN: np.arctan, SINH: np.sinh,
             COSH: np.cosh, TANH: np.tanh, ARCSINH: np.arcsinh, ARCCOSH: np.arccosh, ARCTANH: np.arctanh, EXP: np.exp, LOG: np.log,
             SQRT: np.sqrt, CBRT: np.cbrt, CEIL: np.ceil, FLOOR: np.floor, RINT: np.rint}
TICKS_PER_DAY = [1, 86400, 86400 * 10**3, 86400 * 10**6, 86400 * 10**9]  # DAYS, SECONDS, MILLI-, MICRO-, NANOSECONDS


def is_timestamp(t: int) -> bool:
    return 12 <= t <= 16


def is_duration(t: int) -> bool:
    return 17 <= t <= 21


def is_chrono(t: int) -> bool:
    return 12 <= t <= 21


def is_float(t: int) -> bool:
    return t in (FLOAT32, FLOAT64)


def is_integral(t: int) -> bool:  # std::is_integral: the integer types and bool
    return t in NUMERIC and not is_float(t)


def is_signed(t: int) -> bool:
    return t in (INT8, INT16, INT32, INT64)


def _check_id(t: int):
    if not 0 <= t < NUM_TYPE_IDS:
        raise RuntimeError("Invalid type_id")


def output_type(op: int, t: int) -> int | None:
    """The output type of op on t (math_ops.cu's dispatchers), None when the pair is unsupported."""
    arith = t in NUMERIC
    if SIN <= op <= ABS:
        return t if arith else None
    if op == RINT:
        return t if is_float(t) else None
    if op == BIT_COUNT:
        return INT32 if is_integral(t) else None
    if op == BIT_INVERT:
        return t if is_integral(t) else None
    if op == NOT:
        return BOOL8 if arith else None
    if op == NEGATE:
        return t if (is_signed(t) or is_float(t) or is_duration(t)) else None
    return None


def empty_output_type(op: int, t: int) -> int:
    return BOOL8 if op == NOT else INT32 if op == BIT_COUNT else t


def _to_type(d: np.ndarray, t: int) -> tuple[np.ndarray, np.ndarray]:
    """static_cast<T> of float64 values: (values, defined). Integers truncate; NaN or a truncation out of range is undefined."""
    if t == BOOL8:
        return d != 0, np.ones(len(d), bool)
    if is_float(t):
        with np.errstate(over="ignore", invalid="ignore"):
            return d.astype(NP[t]), np.ones(len(d), bool)
    info = np.iinfo(NP[t])
    with np.errstate(invalid="ignore"):
        tr = np.trunc(d)
        ok = np.isfinite(tr) & (tr >= float(info.min)) & (tr <= float(info.max))
        # float(info.max) rounds up for 64-bit types: 2^63 (2^64) itself does not fit
        if info.bits == 64:
            ok &= tr < float(2**63 if info.min < 0 else 2**64)
    out = np.zeros(len(d), NP[t])
    out[ok] = tr[ok].astype(NP[t])
    return out, ok


def _int_values(v: np.ndarray, t: int) -> np.ndarray:
    """The values as Python ints (object array): integers as they are, bool as 0 / 1."""
    return np.array([int(x) for x in v.astype(np.int64 if t == BOOL8 else v.dtype)], dtype=object)


def _wrap(ints, t: int) -> np.ndarray:
    """Python ints converted to integer type t modulo 2^bits (the two's-complement narrowing of C++)."""
    info = np.iinfo(NP[t])
    m = 1 << info.bits
    out = [(int(x) % m) for x in ints]
    if info.min < 0:
        out = [x - m if x > info.max else x for x in out]
    return np.array(out, dtype=NP[t]) if len(out) else np.zeros(0, NP[t])


def math_double(op: int, v: np.ndarray, t: int) -> np.ndarray:
    """The float64 value op computes before the conversion back to t (the oracle of the integer types and BOOL8)."""
    with np.errstate(all="ignore"):
        return _NUMPY_FN[op](v.astype(np.float64))


def unary(op: int, col) -> tuple[np.ndarray, np.ndarray | None, np.ndarray]:
    vals, valid, t = col
    _check_id(t)
    if not (SIN <= op <= NEGATE):
        raise RuntimeError("Undefined unary operation")
    if not 1 <= t <= 21:
        raise TypeError("only fixed-width column types are supported")
    n = len(vals)
    if n == 0:
        return np.zeros(0, NP[empty_output_type(op, t)]), valid, np.zeros(0, bool)
    out_t = output_type(op, t)
    if out_t is None:
        raise RuntimeError("Unsupported data type for this unary operation")
    ones = np.ones(n, bool)
    if op in _NUMPY_FN and is_float(t):
        if op in INEXACT_OPS:  # the float64 value rounded to t: the kernel is held to 4 ulp of it
            with np.errstate(all="ignore"):
                return _NUMPY_FN[op](vals.astype(np.float64)).astype(NP[t]), valid, ones
        with np.errstate(all="ignore"):
            return _NUMPY_FN[op](vals), valid, ones
    if op in _NUMPY_FN:  # integers and BOOL8 compute in double
        out, ok = _to_type(math_double(op, vals, t), t)
        return out, valid, ok
    if op == ABS:
        if is_float(t):
            return np.abs(vals), valid, ones
        if not is_signed(t):
            return vals.copy(), valid, ones
        ints = _int_values(vals, t)
        ok = ones if np.iinfo(NP[t]).bits < 32 else vals != np.iinfo(NP[t]).min
        return _wrap([abs(x) for x in ints], t), valid, ok
    if op == BIT_COUNT:
        if t == BOOL8:
            return vals.astype(np.int32), valid, ones
        u = vals.view(np.dtype(NP[t]).str.replace("i", "u"))
        return np.bitwise_count(u).astype(np.int32), valid, ones
    if op == BIT_INVERT:
        if t == BOOL8:
            return np.ones(n, bool), valid, ones
        return ~vals, valid, ones
    if op == NOT:
        return vals == 0, valid, ones
    # NEGATE
    if is_float(t):
        return -vals, valid, ones
    st = NP[t]
    ints = _int_values(vals, t)
    ok = ones if np.iinfo(st).bits < 32 else vals != np.iinfo(st).min
    storage = {np.int32: INT32, np.int64: INT64}.get(st, t)
    return _wrap([-x for x in ints], storage), valid, ok


def is_supported_cast(f: int, to: int) -> bool:
    """cast_ops.cu's rule over the ids held here; decimal pairs are not supported (the one deviation from the reference)."""
    _check_id(f)
    _check_id(to)
    if not (1 <= f <= 21 and 1 <= to <= 21):
        return False
    return not (is_timestamp(f) and to in NUMERIC) and not (f in NUMERIC and is_timestamp(to))


def chrono_ticks(x: int, f: int, to: int) -> int:
    """cuda::std::chrono::floor of x ticks of unit f in unit to, as a Python int (before the narrowing to the target's rep)."""
    pf, pt = TICKS_PER_DAY[(f - 12) % 5], TICKS_PER_DAY[(to - 12) % 5]
    return x * (pt // pf) if pt >= pf else x // (pf // pt)  # Python's // floors


def _storage(t: int) -> int:
    return {np.int32: INT32, np.int64: INT64}[NP[t]] if is_chrono(t) else t


def cast(col, to: int) -> tuple[np.ndarray, np.ndarray | None, np.ndarray]:
    vals, valid, f = col
    _check_id(to)
    if to in DECIMALS:
        raise TypeError("cast: decimal types are not supported")
    if not 1 <= to <= 21:
        raise RuntimeError("Unary cast type must be fixed-width.")
    if not 1 <= f <= 21:
        raise TypeError("only fixed-width column types are supported")
    if not is_supported_cast(f, to):
        raise RuntimeError("Unsupported cast between a timestamp and a numeric type")
    n = len(vals)
    ones = np.ones(n, bool)
    if is_chrono(f) and is_chrono(to):
        st = NP[to]
        info = np.iinfo(st)
        ticks = [chrono_ticks(int(x), f, to) for x in vals]
        ok = np.array([info.min <= x <= info.max for x in ticks], bool) if n else np.zeros(0, bool)
        # an up-cast that overflows int64 is undefined too
        ok &= np.array([-2**63 <= x < 2**63 for x in ticks], bool) if n else np.zeros(0, bool)
        return _wrap(ticks, _storage(to)), valid, ok
    fs, ts = _storage(f), _storage(to)  # numeric <-> duration: the tick count as a number
    v = vals
    if is_float(fs):
        out, ok = _to_type(v.astype(np.float64), ts)
        if ts == FLOAT32 and fs == FLOAT32:
            out = v.copy()
        return out, valid, ok
    if ts == BOOL8:
        return v != 0, valid, ones
    if is_float(ts):
        with np.errstate(over="ignore"):
            return v.astype(NP[ts]), valid, ones
    return _wrap(_int_values(v, fs), ts), valid, ones


def is_null(col) -> np.ndarray:
    vals, valid, _ = col
    return np.zeros(len(vals), bool) if valid is None else ~valid


def is_valid(col) -> np.ndarray:
    return ~is_null(col)


def is_nan(col, want_nan: bool = True) -> np.ndarray:
    vals, valid, t = col
    if not is_float(t):
        raise RuntimeError("NAN is not supported in a Non-floating point type column")
    v = np.ones(len(vals), bool) if valid is None else valid
    nan = np.isnan(vals) & v
    return nan if want_nan else ~nan

"""CPU: the unary oracle (tests/unary_oracle.py) against C++ and against the reference's known answers.

tests/cpp/unary_types.cpp, compiled here with g++, reports the type traits behind the support rules (which numeric types each
operator's dispatcher accepts, which chrono / numeric pairs cast), std::chrono::floor between every pair of chrono units, and the
promotion-sensitive values of the integral overloads (BOOL8 BIT_INVERT / NOT / BIT_COUNT, ABS / NEGATE of narrow minima, NOT of
NaN and -0.0, BIT_COUNT of negative narrow integers, bool of NaN)."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import unary_oracle as ou
from tests.golden.unary_cases import CASES

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def cxx(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = tmp_path_factory.mktemp("unary") / "unary_types"
    r = subprocess.run(["g++", "-std=c++17", "-O0", str(ROOT / "tests" / "cpp" / "unary_types.cpp"), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = [line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n") if line]
    return {k: [row[1:] for row in out if row[0] == k] for k in "scfv"}


def _col(vals, t, valid=None):
    dt = ou.NP[t]
    return np.array(vals, dtype=np.float64 if np.dtype(dt).kind == "f" else object).astype(dt), valid, t


def test_support_matches_cxx(cxx):
    assert len(cxx["s"]) == 24 * 11
    for op, t, v in ((int(a), int(b), int(c)) for a, b, c in cxx["s"]):
        assert (ou.output_type(op, t) is not None) == bool(v), (op, t)


def test_cast_rule_matches_cxx(cxx):
    assert len(cxx["c"]) == 21 * 21
    for f, t, v in ((int(a), int(b), int(c)) for a, b, c in cxx["c"]):
        assert ou.is_supported_cast(f, t) == bool(v), (f, t)
    for f in ou.FIXED_WIDTH:
        for d in ou.DECIMALS + [0, 22, 23, 24, 28]:
            assert not ou.is_supported_cast(f, d) and not ou.is_supported_cast(d, f)


def test_chrono_floor_matches_cxx(cxx):
    assert len(cxx["f"]) == 10 * 10 * 16
    for f, t, x, want in ((int(a), int(b), int(c), int(d)) for a, b, c, d in cxx["f"]):
        exact = ou.chrono_ticks(x, f, t)
        if not -2**63 <= exact < 2**63:  # an up-cast that overflows int64: undefined
            continue
        assert exact == want, (f, t, x)
        st = ou.NP[t]
        if np.iinfo(st).min <= want <= np.iinfo(st).max:
            src = np.array([x], dtype=ou.NP[f]) if np.iinfo(ou.NP[f]).min <= x <= np.iinfo(ou.NP[f]).max else None
            if src is not None:
                vals, _, ok = ou.cast((src, None, f), t)
                assert ok[0] and int(vals[0]) == want, (f, t, x)


def test_promotion_values_match_cxx(cxx):
    v = {name: int(val) for name, val in cxx["v"]}
    U = lambda op, vals, t: ou.unary(op, _col(vals, t))[0]  # noqa: E731
    assert bool(U(ou.BIT_INVERT, [True], ou.BOOL8)[0]) == bool(v["bit_invert_true"])
    assert bool(U(ou.BIT_INVERT, [False], ou.BOOL8)[0]) == bool(v["bit_invert_false"])
    assert bool(U(ou.NOT, [True], ou.BOOL8)[0]) == bool(v["not_true"])
    assert bool(U(ou.NOT, [False], ou.BOOL8)[0]) == bool(v["not_false"])
    assert int(U(ou.BIT_COUNT, [True], ou.BOOL8)[0]) == v["bit_count_true"]
    assert int(U(ou.ABS, [-128], ou.INT8)[0]) == v["abs_int8_min"]
    assert int(U(ou.ABS, [-32768], ou.INT16)[0]) == v["abs_int16_min"]
    assert int(U(ou.NEGATE, [-128], ou.INT8)[0]) == v["negate_int8_min"]
    assert int(U(ou.NEGATE, [-32768], ou.INT16)[0]) == v["negate_int16_min"]
    assert bool(U(ou.NOT, [np.nan], ou.FLOAT64)[0]) == bool(v["not_nan"])
    assert bool(U(ou.NOT, [-0.0], ou.FLOAT64)[0]) == bool(v["not_neg_zero"])
    assert int(U(ou.BIT_COUNT, [-1], ou.INT8)[0]) == v["bit_count_int8_m1"]
    assert int(U(ou.BIT_COUNT, [-128], ou.INT8)[0]) == v["bit_count_int8_min"]
    assert int(U(ou.BIT_COUNT, [-2], ou.INT16)[0]) == v["bit_count_int16_m2"]
    assert bool(ou.cast(_col([np.nan], ou.FLOAT64), ou.BOOL8)[0][0]) == bool(v["bool_of_nan"])
    assert int(U(ou.BIT_INVERT, [5], ou.UINT8)[0]) == v["bit_invert_uint8_5"]


def _ulps(a, b):
    it = np.int32 if a.dtype == np.float32 else np.int64
    ia, ib = a.view(it).astype(np.int64), b.view(it).astype(np.int64)
    ia = np.where(ia < 0, np.iinfo(it).min - ia, ia)
    ib = np.where(ib < 0, np.iinfo(it).min - ib, ib)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    return np.where(same, 0, np.abs(ia - ib))


def golden_input(c):
    return _col(c["values"], c["type"], None if c["valid"] is None else np.array(c["valid"], bool))


def oracle_of(c):
    """The oracle's answer for a golden case: (values, valid, defined)."""
    col = golden_input(c)
    if c["fn"] == "unary":
        return ou.unary(c["op"], col)
    if c["fn"] == "cast":
        for to in (c["to"] if isinstance(c["to"], list) else [c["to"]]):
            vals, valid, ok = ou.cast(col, to)
            col = (vals, valid, to)
        return vals, valid, ok
    fn = {"is_null": ou.is_null, "is_valid": ou.is_valid, "is_nan": ou.is_nan,
          "is_not_nan": lambda x: ou.is_nan(x, want_nan=False)}[c["fn"]]
    out = fn(col)
    return out, None, np.ones(len(out), bool)


@pytest.mark.parametrize("i", range(len(CASES)))
def test_oracle_matches_golden(i):
    c = CASES[i]
    if "raises" in c:
        with pytest.raises({"RuntimeError": RuntimeError, "TypeError": TypeError}[c["raises"]]):
            oracle_of(c)
        return
    vals, valid, ok = oracle_of(c)
    assert ok.all(), c["src"]
    exp = c["expect"]
    got_valid = np.ones(len(vals), bool) if valid is None else valid
    assert [e is not None for e in exp] == list(got_valid), c["src"]
    e = np.array([0 if x is None else x for x in exp], dtype=np.float64 if vals.dtype.kind == "f" else object).astype(vals.dtype)
    keep = got_valid
    if c.get("approx"):
        assert (_ulps(vals[keep], e[keep]) <= 4).all(), c["src"]
    elif vals.dtype.kind == "f":
        assert ((vals[keep] == e[keep]) | (np.isnan(vals[keep]) & np.isnan(e[keep]))).all(), c["src"]
    else:
        assert np.array_equal(vals[keep], e[keep]), (c["src"], vals, e)


def test_undefined_rows_are_marked():
    _, _, ok = ou.cast(_col([np.nan, 1e20, -0.5, 3.9, -1.0], ou.FLOAT64), ou.UINT8)
    assert list(ok) == [False, False, True, True, False]
    _, _, ok = ou.unary(ou.ABS, _col([-2**31, 5], ou.INT32))
    assert list(ok) == [False, True]
    _, _, ok = ou.unary(ou.EXP, _col([10, 1], ou.INT8))
    assert list(ok) == [False, True]
    _, _, ok = ou.cast(_col([2**40 * 86400, 86400], 18), 17)  # seconds -> DURATION_DAYS: 2^40 days do not fit int32
    assert list(ok) == [False, True]
    assert ou.unary(ou.RINT, _col([], ou.INT32))[0].dtype == np.int32  # empty: no type check

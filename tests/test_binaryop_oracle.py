"""CPU: the binary-operation oracle (tests/binaryop_oracle.py) against C++ and against the reference's known answers.

The common-type table and the supported-operation rule are checked against a program compiled here with g++
(tests/cpp/binaryop_types.cpp), which asks the compiler: std::common_type of every pair and triple of the 11 numeric types, and
whether each operator's expression is well-formed on std::common_type<lhs, rhs> with a result constructible as the output."""
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import binaryop_oracle as ob
from tests.golden.binaryop_cases import CASES, SUPPORTED_SPOTS
from tests.helpers import make_col

ROOT = Path(__file__).resolve().parent.parent
TYPE_ID = {"int8": 1, "int16": 2, "int32": 3, "int64": 4, "uint8": 5, "uint16": 6, "uint32": 7, "uint64": 8, "float32": 9,
           "float64": 10, "bool": 11}
EXC = {"ValueError": ValueError, "RuntimeError": RuntimeError, "TypeError": TypeError}


@pytest.fixture(scope="module")
def cxx(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = tmp_path_factory.mktemp("binop") / "binaryop_types"
    r = subprocess.run(["g++", "-std=c++17", "-O0", str(ROOT / "tests" / "cpp" / "binaryop_types.cpp"), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    rows = [tuple(int(v) for v in line.split()[1:]) for line in out if line]
    kinds = [line[0] for line in out if line]
    return {k: [r for r, kk in zip(rows, kinds) if kk == k] for k in "cts"}


def test_common_type_pairs(cxx):
    assert len(cxx["c"]) == 121
    for a, b, t in cxx["c"]:
        assert ob.common_type(a, b) == t, (a, b)


def test_common_type_triples(cxx):
    assert len(cxx["t"]) == 11 ** 3
    for o, a, b, t in cxx["t"]:
        assert ob.compute_type(o, a, b) == t, (o, a, b)


def test_is_supported_matches_cxx(cxx):
    assert len(cxx["s"]) == 34 * 11 ** 3
    for op, o, a, b, v in cxx["s"]:
        assert ob.is_supported(o, a, b, op) == bool(v), (op, o, a, b)


@pytest.mark.parametrize("spot", SUPPORTED_SPOTS)
def test_is_supported_spots(spot):
    op, o, a, b, want = spot
    assert ob.is_supported(o, a, b, op) == want


def operand(spec):
    if isinstance(spec, dict):
        v = spec["scalar"]
        return np.array(0 if v is None else v, dtype=np.dtype(spec["dtype"])), v is not None, TYPE_ID[spec["dtype"]]
    vals, valid = make_col(*spec)
    return vals, valid, TYPE_ID[spec[1]]


def out_type(case):
    return case["out"] if isinstance(case["out"], int) else TYPE_ID[case["out"]]


@pytest.mark.parametrize("case", CASES, ids=[c["src"] for c in CASES])
def test_oracle_golden(case):
    lhs, rhs = operand(case["lhs"]), operand(case["rhs"])
    if "raises" in case:
        with pytest.raises(EXC[case["raises"]]):
            ob.binop(case["op"], lhs, rhs, out_type(case))
        return
    vals, valid, defined, _ = ob.binop(case["op"], lhs, rhs, out_type(case))
    got = [v.item() if ok else None for v, ok in zip(vals, valid)]
    assert got == case["expect"]
    assert defined[valid].all()


def test_oracle_semantics():
    """The rules the golden cases do not reach: narrow integers compute in int and wrap on the cast; comparisons use C; INT_POW
    wraps and is 0 for a negative exponent; PYMOD and PMOD signs; undefined rows."""
    i8 = (np.array([100, -128, 7, -7], np.int8), None, ob.INT8)
    v, _, d, _ = ob.binop(ob.ADD, i8, i8, ob.INT8)
    assert v.tolist() == [-56, 0, 14, -14] and d.all()
    v, _, _, _ = ob.binop(ob.ADD, i8, i8, ob.INT16)
    assert v.tolist() == [200, -256, 14, -14]
    v, _, _, _ = ob.binop(ob.SHIFT_RIGHT_UNSIGNED, (np.array([-1], np.int8), None, ob.INT8), (np.array([1], np.int8), None, ob.INT8),
                          ob.INT8)
    assert v.tolist() == [127]
    big = (np.array([2**24 + 1], np.int64), None, ob.INT64)
    f32 = (np.array([2**24], np.float32), None, ob.FLOAT32)
    assert ob.binop(ob.GREATER, big, f32, ob.BOOL8)[0].tolist() == [False]  # compared in float32
    x = (np.array([-7, 7, -7, 3], np.int32), None, ob.INT32)
    y = (np.array([2, -2, -2, -1], np.int32), None, ob.INT32)
    assert ob.binop(ob.FLOOR_DIV, x, y, ob.INT32)[0].tolist() == [-4, -4, 3, -3]
    assert ob.binop(ob.MOD, x, y, ob.INT32)[0].tolist() == [-1, 1, -1, 0]
    assert ob.binop(ob.PMOD, x, y, ob.INT32)[0].tolist() == [1, 1, -1, 0]
    assert ob.binop(ob.PYMOD, x, y, ob.INT32)[0].tolist() == [1, -1, -1, 0]
    assert ob.binop(ob.INT_POW, (np.array([2, 3, 2], np.int32), None, ob.INT32), (np.array([31, 21, -1], np.int32), None, ob.INT32),
                    ob.INT32)[0].tolist() == [-2**31, 3**21 % 2**32, 0]
    _, _, d, _ = ob.binop(ob.DIV, (np.array([1, -2**31], np.int32), None, ob.INT32), (np.array([0, -1], np.int32), None, ob.INT32),
                          ob.INT32)
    assert not d.any()
    _, _, d, _ = ob.binop(ob.SHIFT_LEFT, x, (np.array([0, 31, 32, -1], np.int32), None, ob.INT32), ob.INT32)
    assert d.tolist() == [True, True, False, False]
    _, _, d, _ = ob.binop(ob.TRUE_DIV, x, (np.array([0, 1, 2, 4], np.int32), None, ob.INT32), ob.INT8)
    assert d.tolist() == [False, True, True, True]  # -7 / 0 = -inf does not convert
    _, _, d, _ = ob.binop(ob.BITWISE_AND, x, y, ob.FLOAT64)  # C is double: no value
    assert not d.any()

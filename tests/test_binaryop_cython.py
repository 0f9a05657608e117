"""The compiled binding's binary operations (cudf_b200.pylibcudf_cy.binaryop) against the oracle: linked against the kernel
emulator's library on the CPU, and against the product library on the GPU."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

BODY = r"""
import numpy as np
from tests import binaryop_oracle as ob
B = cy.binaryop
rng = np.random.default_rng(3)
n = 3 * 1024 + 7
a, av = rng.integers(-1000, 1000, n).astype(np.int64), rng.random(n) < 0.8
b = rng.normal(size=n) * 100
ca, cb = cy.Column.from_numpy(a, av), cy.Column.from_numpy(b)
def same(got, op, lhs, rhs, out):
    vals, valid, defined, _ = ob.binop(op, lhs, rhs, out)
    gv, gm = got.to_numpy()
    gm = np.ones(n, bool) if gm is None else gm
    assert np.array_equal(gm, valid) and got.null_count() == int((~valid).sum()), op
    keep = valid & defined
    assert np.array_equal(gv[keep], vals[keep]), op
f64, i64, b8 = cy.DataType(cy.TypeId.FLOAT64), cy.DataType(cy.TypeId.INT64), cy.DataType(cy.TypeId.BOOL8)
same(B.binary_operation(ca, cb, B.BinaryOperator.ADD, f64), ob.ADD, (a, av, ob.INT64), (b, None, ob.FLOAT64), ob.FLOAT64)
same(B.binary_operation(ca, cy.Scalar.from_py(7, i64), B.BinaryOperator.FLOOR_DIV, i64), ob.FLOOR_DIV, (a, av, ob.INT64),
     (np.asarray(np.int64(7)), True, ob.INT64), ob.INT64)
same(B.binary_operation(cy.Scalar.from_py(0.5, f64), cb, B.BinaryOperator.GREATER, b8), ob.GREATER,
     (np.asarray(0.5), True, ob.FLOAT64), (b, None, ob.FLOAT64), ob.BOOL8)
same(B.binary_operation(ca, cy.Scalar.from_py(None, i64), B.BinaryOperator.NULL_MAX, i64), ob.NULL_MAX, (a, av, ob.INT64),
     (np.asarray(np.int64(0)), False, ob.INT64), ob.INT64)
assert B.is_supported_operation(f64, i64, f64, B.BinaryOperator.ADD)
assert not B.is_supported_operation(f64, f64, f64, B.BinaryOperator.BITWISE_AND)
for fn, exc in ((lambda: B.binary_operation(ca, cb, B.BinaryOperator.BITWISE_AND, f64), TypeError),
                (lambda: B.binary_operation(ca, cy.Column.from_numpy(b[:5]), B.BinaryOperator.ADD, f64), ValueError)):
    try:
        fn()
        raise SystemExit("no error")
    except exc:
        pass
print('CY_BINOP_OK')
"""


def test_cython_binaryop_on_the_emulator():
    code = "import sys\nsys.path.insert(0, '.')\nfrom tests.emu import harness\ncy = harness.install_cy()\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_BINOP_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_cython_binaryop_gpu():
    code = "import sys\nsys.path.insert(0, '.')\nimport __graft_entry__ as g\ng.build()\nimport cudf_b200.pylibcudf_cy as cy\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_BINOP_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

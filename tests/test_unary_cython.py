"""The compiled binding's unary operations and casts (cudf_b200.pylibcudf_cy.unary) against the oracle: linked against the kernel
emulator's library on the CPU, and against the product library on the GPU."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

BODY = r"""
import numpy as np
from tests import unary_oracle as ou
U = cy.unary
rng = np.random.default_rng(3)
n = 3 * 1024 + 7
x, xv = rng.normal(size=n) * 100, rng.random(n) < 0.8
x[::17] = np.nan
k = rng.integers(-1000, 1000, n).astype(np.int32)
cx, ck = cy.Column.from_numpy(x, xv), cy.Column.from_numpy(k)
def same(got, vals, valid, defined=None):
    gv, gm = got.to_numpy()
    assert (gm is None) == (valid is None)
    m = np.ones(n, bool) if valid is None else valid
    assert gm is None or np.array_equal(gm, m)
    keep = m if defined is None else m & defined
    assert np.array_equal(gv[keep], vals[keep], equal_nan=gv.dtype.kind == "f")
same(U.unary_operation(cx, U.UnaryOperator.SQRT), *ou.unary(ou.SQRT, (x, xv, ou.FLOAT64)))
same(U.unary_operation(ck, U.UnaryOperator.NEGATE), *ou.unary(ou.NEGATE, (k, None, ou.INT32)))
same(U.cast(ck, cy.DataType(cy.TypeId.FLOAT64)), *ou.cast((k, None, ou.INT32), ou.FLOAT64))
same(U.cast(cx, cy.DataType(cy.TypeId.INT16)), *ou.cast((x, xv, ou.FLOAT64), ou.INT16))
same(U.is_null(cx), ~xv, None)
same(U.is_valid(cx), xv, None)
same(U.is_nan(cx), ou.is_nan((x, xv, ou.FLOAT64)), None)
same(U.is_not_nan(cx), ou.is_nan((x, xv, ou.FLOAT64), want_nan=False), None)
b = U.bit_cast(cx, cy.DataType(cy.TypeId.INT64))
bv, bm = b.to_numpy()
assert np.array_equal(bv, x.view(np.int64)) and np.array_equal(bm, xv)
assert U.is_supported_cast(cy.DataType(cy.TypeId.INT32), cy.DataType(cy.TypeId.DURATION_SECONDS))
assert not U.is_supported_cast(cy.DataType(cy.TypeId.INT32), cy.DataType(cy.TypeId.TIMESTAMP_SECONDS))
for fn, exc in ((lambda: U.unary_operation(ck, U.UnaryOperator.RINT), RuntimeError),
                (lambda: U.is_nan(ck), RuntimeError),
                (lambda: U.cast(ck, cy.DataType(cy.TypeId.TIMESTAMP_DAYS)), RuntimeError),
                (lambda: U.cast(ck, cy.DataType(cy.TypeId.DECIMAL32)), TypeError),
                (lambda: U.bit_cast(ck, cy.DataType(cy.TypeId.INT64)), RuntimeError)):
    try:
        fn()
        raise SystemExit("no error")
    except exc:
        pass
print('CY_UNARY_OK')
"""


def test_cython_unary_on_the_emulator():
    code = "import sys\nsys.path.insert(0, '.')\nfrom tests.emu import harness\ncy = harness.install_cy()\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_UNARY_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_cython_unary_gpu():
    code = "import sys\nsys.path.insert(0, '.')\nimport __graft_entry__ as g\ng.build()\nimport cudf_b200.pylibcudf_cy as cy\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_UNARY_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

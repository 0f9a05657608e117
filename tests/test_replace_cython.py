"""The compiled binding's replacement (cudf_b200.pylibcudf_cy.replace) against the oracle: linked against the kernel emulator's
library on the CPU, and against the product library on the GPU."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

BODY = r"""
import numpy as np
from tests import replace_oracle as orp
R = cy.replace
rng = np.random.default_rng(3)
n = 3 * 1024 + 7
x, xv = rng.normal(size=n), rng.random(n) < 0.6
x[::17] = np.nan
x[::19] = -0.0
k = rng.integers(-20, 20, n).astype(np.int32)
kv = rng.random(n) < 0.5
cx, ck = cy.Column.from_numpy(x, xv), cy.Column.from_numpy(k, kv)
f64, i32 = cy.DataType(cy.TypeId.FLOAT64), cy.DataType(cy.TypeId.INT32)
def same(got, vals, valid, bitwise=False):
    gv, gm = got.to_numpy()
    assert (gm is None) == (valid is None)
    m = np.ones(n, bool) if valid is None else valid
    assert gm is None or np.array_equal(gm, m)
    if bitwise:
        assert np.array_equal(gv[m].view(np.uint64), vals[m].view(np.uint64))
    else:
        assert np.array_equal(gv[m], vals[m], equal_nan=gv.dtype.kind == "f")
same(R.replace_nulls(ck, cy.Scalar.from_py(7, i32)), *orp.replace_nulls_scalar((k, kv, 3), orp.Scalar(7, True, 3)))
same(R.replace_nulls(ck, cy.Column.from_numpy(-k)), *orp.replace_nulls_column((k, kv, 3), (-k, None, 3)))
same(R.replace_nulls(ck, R.ReplacePolicy.PRECEDING), *orp.replace_nulls_policy((k, kv, 3), orp.PRECEDING))
same(R.replace_nulls(ck, R.ReplacePolicy.FOLLOWING), *orp.replace_nulls_policy((k, kv, 3), orp.FOLLOWING))
old, new = np.array([1, 2, 2, 99], np.int32), np.array([10, 20, 30, 40], np.int32)
same(R.find_and_replace_all(ck, cy.Column.from_numpy(old), cy.Column.from_numpy(new)),
     *orp.find_and_replace_all((k, kv, 3), (old, None, 3), (new, None, 3)))
same(R.clamp(cx, cy.Scalar.from_py(-0.5, f64), cy.Scalar.from_py(0.5, f64)),
     *orp.clamp((x, xv, 10), *[orp.Scalar(v, True, 10) for v in (-0.5, -0.5, 0.5, 0.5)]))
same(R.clamp(cx, cy.Scalar.from_py(-0.5, f64), cy.Scalar.from_py(0.5, f64), cy.Scalar.from_py(-9.0, f64), cy.Scalar.from_py(9.0, f64)),
     *orp.clamp((x, xv, 10), *[orp.Scalar(v, True, 10) for v in (-0.5, -9.0, 0.5, 9.0)]))
same(R.normalize_nans_and_zeros(cx), *orp.normalize_nans_and_zeros((x, xv, 10)), bitwise=True)
c2 = cy.Column.from_numpy(x, xv)
assert R.normalize_nans_and_zeros(c2, inplace=True) is None
same(c2, *orp.normalize_nans_and_zeros((x, xv, 10)), bitwise=True)
for fn, exc in ((lambda: R.replace_nulls(ck, 3), TypeError),
                (lambda: R.replace_nulls(ck, cx), TypeError),
                (lambda: R.clamp(cx, cy.Scalar.from_py(0.0, f64), cy.Scalar.from_py(1.0, f64), cy.Scalar.from_py(0.0, f64)), ValueError),
                (lambda: R.normalize_nans_and_zeros(ck), RuntimeError)):
    try:
        fn()
        raise SystemExit("no error")
    except exc:
        pass
print('CY_REPLACE_OK')
"""


def test_cython_replace_on_the_emulator():
    code = "import sys\nsys.path.insert(0, '.')\nfrom tests.emu import harness\ncy = harness.install_cy()\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_REPLACE_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_cython_replace_gpu():
    code = "import sys\nsys.path.insert(0, '.')\nimport __graft_entry__ as g\ng.build()\nimport cudf_b200.pylibcudf_cy as cy\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_REPLACE_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

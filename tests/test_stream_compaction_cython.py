"""The compiled binding's stream_compaction (cudf_b200.pylibcudf_cy, _core.pyx) against the oracle: linked against the kernel
emulator's library on the CPU, and against the product library on the GPU."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

BODY = r"""
import numpy as np
from oracle import stream_compaction as osc
from tests.helpers import assert_columns_equal
sc = cy.stream_compaction
rng = np.random.default_rng(41)
def tab(cols):
    return cy.Table([cy.Column.from_numpy(v, m) for v, m in cols])
def check(t, exp, what):
    got = [c.to_numpy() for c in t.columns()]
    assert len(got) == len(exp), what
    for j, (g, e) in enumerate(zip(got, exp)):
        assert_columns_equal(g, e, what=f"{what} {j}")
n = 3 * 8192 + 11
k = np.sort(rng.integers(0, 40, n)).astype(np.int64)
f = rng.integers(0, 4, n) * 0.5; f[rng.random(n) < 0.1] = np.nan
cols = [(k, rng.random(n) < 0.9), (f, rng.random(n) < 0.8), (np.arange(n, dtype=np.int32), None)]
t = tab(cols)
mv, mm = rng.random(n) < 0.5, rng.random(n) < 0.9
mask = cy.Column.from_numpy(mv, mm)
check(sc.apply_boolean_mask(t, mask), osc.apply_boolean_mask(cols, (mv, mm)), "mask")
check(sc.apply_deletion_mask(t, mask), osc.apply_boolean_mask(cols, (mv, mm), True), "deletion")
check(sc.drop_nulls(t, [0, 1]), osc.drop_nulls(cols, [0, 1]), "nulls")
check(sc.drop_nulls(t, [0, 1], 1), osc.drop_nulls(cols, [0, 1], 1), "nulls 1")
check(sc.drop_nans(t, [1]), osc.drop_nans(cols, [1]), "nans")
for keep in (1, 2, 3):
    for ne in (0, 1):
        check(sc.unique(t, [0], keep, ne), osc.unique(cols, [0], keep, ne), ("unique", keep, ne))
        for nan in (0, 1):
            check(sc.stable_distinct(t, [0, 1], keep, ne, nan), osc.stable_distinct(cols, [0, 1], keep, ne, nan), ("sd", keep, ne, nan))
            check(sc.distinct(t, [0, 1], keep, ne, nan), osc.stable_distinct(cols, [0, 1], keep, ne, nan), ("d", keep, ne, nan))
            idx = sc.distinct_indices(tab(cols[:2]), keep, ne, nan).to_numpy()[0]
            assert np.array_equal(idx, osc.distinct_indices(cols[:2], keep, ne, nan)), (keep, ne, nan)
for fn, exc in ((lambda: sc.drop_nulls(t, [3]), IndexError), (lambda: sc.drop_nans(t, [0]), RuntimeError),
                (lambda: sc.apply_boolean_mask(t, cy.Column.from_numpy(k)), RuntimeError)):
    try:
        fn()
        raise SystemExit("no error")
    except exc:
        pass
print('CY_SC_OK')
"""


def test_cython_stream_compaction_on_the_emulator():
    code = "import sys\nsys.path.insert(0, '.')\nfrom tests.emu import harness\ncy = harness.install_cy()\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_SC_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_cython_stream_compaction_gpu():
    code = "import sys\nsys.path.insert(0, '.')\nimport __graft_entry__ as g\ng.build()\nimport cudf_b200.pylibcudf_cy as cy\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_SC_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

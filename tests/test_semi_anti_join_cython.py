"""The compiled binding's semi / anti join (cudf_b200.pylibcudf_cy: FilteredJoin, left_semi_join, left_anti_join) against the
oracle: linked against the kernel emulator's library on the CPU, and against the product library on the GPU."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

BODY = r"""
import numpy as np
from tests import semi_anti_oracle as osa
J = cy.join
rng = np.random.default_rng(42)
def tab(cols):
    return cy.Table([cy.Column.from_numpy(v, m) for v, m in cols])
def ids(c):
    return c.to_numpy()[0]
n = 3 * 8192 + 11
packed = ([(rng.integers(0, 300, n).astype(np.int64), rng.random(n) < 0.9)], [(rng.integers(0, 300, 120).astype(np.int64), rng.random(120) < 0.9)])
wide = ([(rng.integers(0, 20, n).astype(np.int64), None), (rng.integers(0, 4, n) * 0.5, rng.random(n) < 0.9)],
        [(rng.integers(0, 20, 50).astype(np.int64), None), (rng.integers(0, 4, 50) * 0.5, rng.random(50) < 0.9)])
for left, right in (packed, wide):
    for ne in (0, 1):
        fj = J.FilteredJoin(tab(right), ne)
        lt = tab(left)
        es, ea = osa.left_semi_join(left, right, ne), osa.left_anti_join(left, right, ne)
        assert np.array_equal(ids(fj.semi_join(lt)), es), (len(left), ne)
        assert np.array_equal(ids(fj.anti_join(lt)), ea), (len(left), ne)
        assert np.array_equal(ids(J.left_semi_join(lt, tab(right), ne)), es)
        assert np.array_equal(ids(J.left_anti_join(lt, tab(right), ne)), ea)
assert ids(J.FilteredJoin(cy.Table([]), 0).anti_join(tab(packed[0]))).tolist() == list(range(n))
for fn, exc in ((lambda: J.FilteredJoin(tab(packed[1]), 0, 0.0), ValueError),
                (lambda: J.FilteredJoin(tab(packed[1]), 0).semi_join(tab(wide[0])), ValueError)):
    try:
        fn()
        raise SystemExit("no error")
    except exc:
        pass
print('CY_SEMI_ANTI_OK')
"""


def test_cython_semi_anti_join_on_the_emulator():
    code = "import sys\nsys.path.insert(0, '.')\nfrom tests.emu import harness\ncy = harness.install_cy()\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_SEMI_ANTI_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_cython_semi_anti_join_gpu():
    code = "import sys\nsys.path.insert(0, '.')\nimport __graft_entry__ as g\ng.build()\nimport cudf_b200.pylibcudf_cy as cy\n" + BODY
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert "CY_SEMI_ANTI_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

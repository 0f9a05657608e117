"""The range tier with estimated bases (radix_sort.cu::run_est_range) on the GPU: the shared checks forced on at small sizes with
B2_SORT_EST=1, windows forced too small with B2_SORT_EST_CAP (every call reruns on the exact plan), and one input at the default
settings large enough to take it: no digit histogram, one key sample per call."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

PRELUDE = r"""
import sys
sys.path.insert(0, '.')
import numpy as np
import cudf_b200.pylibcudf as plc
from cudf_b200 import _lib as L
from oracle import sort as osort
"""


def _run(code, marker, **env):
    e = dict(os.environ, **env)
    r = subprocess.run([sys.executable, "-c", PRELUDE + code], capture_output=True, text=True, env=e, cwd=ROOT, timeout=900)
    assert marker in r.stdout and r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]


@pytest.mark.parametrize("carry", ["1", "0"])
def test_est_small_inputs(carry):
    from tests.snippets.sort_est import CODE

    _run("SIZES = (3, 2049, 20011, 300_007)\nEXPECT_RERUN = False\n" + CODE, "EST_OK", B2_SORT_EST="1", B2_SORT_CARRY=carry)


def test_est_forced_overflow():
    from tests.snippets.sort_est import CODE

    _run("SIZES = (2049, 300_007)\nEXPECT_RERUN = True\n" + CODE, "EST_OK", B2_SORT_EST="1", B2_SORT_EST_CAP="16")


def test_est_default_settings(plc):
    """2^27 + 5 uniform keys take the estimated-base range tier by default: bit-exact against a stable argsort, with one sample
    launch and no histogram per call."""
    from cudf_b200 import _lib as L

    rng = np.random.default_rng(23)
    n = (1 << 27) + 5
    keys = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    vals = rng.integers(0, 1 << 50, n).astype(np.int64)
    kc = plc.Column.from_numpy(keys)
    order = np.argsort(keys, kind="stable")

    def profiled(fn):
        L.lib.b2_profile_reset()
        L.lib.b2_profile_enable(1)
        r = fn()
        L.lib.b2_profile_enable(0)
        assert L.profile_get("histogram")[1] == 0
        assert L.profile_get("est_sample")[1] == 1
        assert L.profile_get("range_bounds")[1] == 1
        return r

    got = profiled(lambda: plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([kc]), [0], []).columns()[0].to_numpy()[0])
    assert np.array_equal(got, vals[order])
    got = profiled(lambda: plc.sorting.sorted_order(plc.Table([kc]), [], []).to_numpy()[0])
    assert np.array_equal(got, order)
    got = profiled(lambda: plc.sorting.sort(plc.Table([kc]), [1], []).columns()[0].to_numpy()[0])
    assert np.array_equal(got, keys[order][::-1])

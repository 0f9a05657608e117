"""The range tier of the hybrid sort (radix_sort.cu::range_sort_kernel) on the GPU, forced on at small sizes with
B2_SORT_RANGE=1, plus one input at the default settings large enough to take it."""
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
L.lib.b2_profile_enable(1)
"""
RAN = "\nassert L.profile_get('range_bounds')[1] > 0\n"


def _run(code, marker, **env):
    e = dict(os.environ, B2_SORT_RANGE="1", B2_SORT_HYBRID_MIN="0", **env)
    r = subprocess.run([sys.executable, "-c", PRELUDE + code + RAN], capture_output=True, text=True, env=e, cwd=ROOT, timeout=900)
    assert marker in r.stdout and r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]


@pytest.mark.parametrize("carry", ["1", "0"])
def test_range_tier_small_inputs(carry):
    from tests.snippets.range_sort import CODE

    # FILL = 200: the float keys' top byte takes few values, so their range id has two digits (65 536 ranges)
    _run("FILL = 200\n" + CODE, "RANGE_OK", B2_SORT_CARRY=carry)


@pytest.mark.parametrize("carry", ["1", "0"])
def test_range_tier_hybrid_inputs(carry):
    from tests.snippets.hybrid_sort import CODE

    _run("SIZES = (3, 100, 2047, 2049, 6145, 20011, 300_007)\n" + CODE, "HYBRID_OK", B2_SORT_CARRY=carry)


def test_range_tier_default_settings(plc):
    """2^27 + 5 uniform keys take the range tier by default (16-bit range id, ~2 K rows per range)."""
    from cudf_b200 import _lib as L

    rng = np.random.default_rng(22)
    n = (1 << 27) + 5
    keys = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    vals = rng.integers(0, 1 << 50, n).astype(np.int64)
    kc = plc.Column.from_numpy(keys)
    L.lib.b2_profile_reset()
    L.lib.b2_profile_enable(1)
    got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([kc]), [0], []).columns()[0].to_numpy()[0]
    L.lib.b2_profile_enable(0)
    assert L.profile_get("range_bounds")[1] == 1
    order = np.argsort(keys, kind="stable")
    assert np.array_equal(got, vals[order])
    assert np.array_equal(plc.sorting.sorted_order(plc.Table([kc]), [], []).to_numpy()[0], order)
    assert np.array_equal(plc.sorting.sort(plc.Table([kc]), [1], []).columns()[0].to_numpy()[0], keys[order][::-1])

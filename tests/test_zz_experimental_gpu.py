"""The aliased sort_by_key(T, T) shortcut (B2_SORT_ALIAS=1): the keys are sorted by the keys-only radix sort and the sorted
keys are the payload. It is opt-in and has not yet been run on hardware, so this check runs it in a subprocess with its switch,
is skipped unless B2_RUN_EXPERIMENTAL=1, and is marked xfail(strict=False) so that a hardware run reports its state
(XPASS / XFAIL) without gating the suite."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Never-run code can hang a kernel; the default GPU suite must not depend on it. Set B2_RUN_EXPERIMENTAL=1 to run it.
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("B2_RUN_EXPERIMENTAL", "0") != "1",
                                 reason="opt-in path not yet validated on hardware: set B2_RUN_EXPERIMENTAL=1")]


@pytest.mark.xfail(strict=False, reason="aliased sort_by_key(T, T) -> keys-only radix (B2_SORT_ALIAS=1) not yet run on hardware")
def test_sort_by_key_alias_shortcut():
    code = r"""
import numpy as np, sys
sys.path.insert(0, '.')
import cudf_b200.pylibcudf as plc
rng = np.random.default_rng(11)
for n in (1, 33, 6145, 200_003, 3_000_001):
    for dt in (np.int64, np.int32, np.uint16, np.int8, np.uint64):
        keys = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
        for order in (0, 1):
            c = plc.Column.from_numpy(keys)
            got = plc.sorting.sort_by_key(plc.Table([c]), plc.Table([c]), [order], []).columns()[0].to_numpy()[0]
            exp = np.sort(keys, kind='stable')
            if order == 1:
                exp = exp[::-1]
            assert np.array_equal(got, exp), (n, dt, order)
print('ALIAS_OK')
"""
    env = dict(os.environ, B2_SORT_ALIAS="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=300)
    assert "ALIAS_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-2500:]

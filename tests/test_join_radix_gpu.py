"""The partitioned join (radix_join.cu) on the GPU.

test_radix_join_cases runs tests/snippets/radix_join.py with B2_JOIN_RADIX_ROWS=1: keys built from their mixed hash so that
they land on the chunk, slot, piece and partition boundaries of the join kernel, key types through the pack kernel, sliced
views, the output-size rerun, and the conditions that send a join to the hash table. test_radix_join_switch_point checks, with no switches set, that 2^24 rows on both sides take the
path and 2^24 - 1 rows on one side do not."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

PRELUDE = r"""
import sys
sys.path.insert(0, '.')
import numpy as np
import cudf_b200.pylibcudf as plc
from cudf_b200 import _lib as L
from oracle import join as ojoin
"""

SWITCHES = ("B2_JOIN_RADIX_ROWS", "B2_JOIN_RADIX_CAPACITY", "B2_SORT_PORTION")


def _run(code, marker, **env):
    e = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    e.update(env)
    r = subprocess.run([sys.executable, "-c", PRELUDE + code], capture_output=True, text=True, env=e, cwd=ROOT, timeout=900)
    assert marker in r.stdout and r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]


def test_radix_join_cases():
    from tests.snippets.radix_join import CODE

    _run("FULL = True\n" + CODE, "RADIX_JOIN_CASES_OK", B2_JOIN_RADIX_ROWS="1")


def test_radix_join_portions():
    from tests.snippets.radix_join import PORTION_CODE

    _run("FULL = True\n" + PORTION_CODE, "RADIX_JOIN_PORTIONS_OK", B2_JOIN_RADIX_ROWS="1", B2_SORT_PORTION=str(3 * 6144))


SWITCH_POINT = r"""
rng = np.random.default_rng(24)
N = 1 << 24

def join_walks(kind, l, r):
    L.lib.b2_profile_reset()
    L.lib.b2_profile_enable(1)
    res = getattr(plc.join, kind)(plc.Table([plc.Column.from_numpy(l)]), plc.Table([plc.Column.from_numpy(r)]), 0)
    L.lib.b2_profile_enable(0)
    got = ojoin.canonical(res[0].to_numpy()[0], res[1].to_numpy()[0])
    del res
    exp = getattr(ojoin, kind)([(l, None)], [(r, None)])
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (kind, len(l), len(r), len(got[0]), len(exp[0]))
    return L.profile_get('rjoin_join')[1]

for nl, nr, walks in ((N, N, 1), (N, N - 1, 0)):
    r = rng.integers(-2**62, 2**62, nr)
    l = rng.integers(-2**62, 2**62, nl)
    planted = rng.random(nl) < 0.1                    # 10 % of the probe rows match a build row
    l[planted] = r[rng.integers(0, nr, int(planted.sum()))]
    l[rng.integers(0, nl, 50_000)] = 42               # a hot key: 3 build rows, ~50 000 probe rows
    r[rng.integers(0, nr, 3)] = 42
    for kind in ('left_join', 'full_join'):
        got = join_walks(kind, l, r)
        assert got == walks, (kind, nl, nr, 'rjoin_join scopes', got, 'expected', walks)
print('SWITCH_POINT_OK')
"""


def test_radix_join_switch_point():
    _run(SWITCH_POINT, "SWITCH_POINT_OK")

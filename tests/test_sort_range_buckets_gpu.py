"""The range tier's bucket sort (radix_sort.cu::range_sort_kernel) on the GPU, forced on at small sizes with B2_SORT_RANGE=1:
runs of equal keys with distinct payloads, buckets taken below constant bytes, and a bucket of exactly the bucket cap next to
one of cap + 1 (overflow and rerun)."""
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
from oracle import sort as osort
"""


@pytest.mark.parametrize("carry", ["1", "0"])
def test_range_tier_buckets(carry):
    from tests.snippets.range_sort_buckets import CODE

    e = dict(os.environ, B2_SORT_RANGE="1", B2_SORT_HYBRID_MIN="0", B2_SORT_CARRY=carry)
    r = subprocess.run([sys.executable, "-c", PRELUDE + "FILL = 200\n" + CODE], capture_output=True, text=True, env=e, cwd=ROOT,
                       timeout=900)
    assert "BUCKETS_OK" in r.stdout and r.returncode == 0, r.stdout[-1500:] + r.stderr[-2500:]

"""The range sort's digest walk on the estimated-window tier (tests/snippets/sort_est_digest.py) on the GPU, forced on with
B2_SORT_EST=1."""
import pytest

from tests.test_sort_est_gpu import _run

pytestmark = pytest.mark.gpu


def test_est_digest_walk():
    from tests.snippets.sort_est_digest import CODE

    _run("SIZES = (2049, 20011, 300_007)\n" + CODE, "DIGEST_OK", B2_SORT_EST="1")

"""The range sort's boundaries on the estimated-window tier (tests/snippets/sort_est_walk.py) on the GPU, forced on with
B2_SORT_EST=1."""
import pytest

from tests.test_sort_est_gpu import _run

pytestmark = pytest.mark.gpu


def test_est_walk_boundaries():
    from tests.snippets.sort_est_walk import CODE

    _run(CODE, "WALK_OK", B2_SORT_EST="1")

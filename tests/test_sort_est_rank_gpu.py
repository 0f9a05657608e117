"""The range sort's bounded walk on the estimated-window tier (tests/snippets/sort_est_rank.py) on the GPU,
forced on with B2_SORT_EST=1."""
import pytest

from tests.test_sort_est_gpu import _run

pytestmark = pytest.mark.gpu


def test_est_rank_and_walk_tail():
    from tests.snippets.sort_est_rank import CODE

    _run(CODE, "RANK_OK", B2_SORT_EST="1")

"""The range sort's bounded walk on the estimated-window tier (tests/snippets/sort_est_rank.py) on the CPU
emulator, forced on with B2_SORT_EST=1: buckets of K and K + 1 rows and at the bucket cap, warps whose rows all finish in the walk's
tail, long buckets at the end of a range, digest ties and equal keys in long buckets, every buckets-per-thread count of the scan,
range lengths around the thread count, and the bucket overflow that reruns on the exact plan."""
from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)


def test_emu_sort_est_rank(emu_lib):
    from tests.snippets.sort_est_rank import CODE

    run(CODE, "RANK_OK", env={"B2_SORT_EST": "1"})

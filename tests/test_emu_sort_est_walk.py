"""The range sort's boundaries on the estimated-window tier (tests/snippets/sort_est_walk.py) on the CPU emulator, forced on with
B2_SORT_EST=1: range lengths around the thread count and RANGE_CAP, every buckets-per-thread count of the scan, full buckets, digest
ties across warp boundaries, and the range and bucket overflows that rerun on the exact plan."""
from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)


def test_emu_sort_est_walk(emu_lib):
    from tests.snippets.sort_est_walk import CODE

    run(CODE, "WALK_OK", env={"B2_SORT_EST": "1"})

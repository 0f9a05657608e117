"""The range tier's bucket sort (radix_sort.cu::range_sort_kernel) on the CPU emulator, forced on at small sizes with
B2_SORT_RANGE=1: runs of equal keys with distinct payloads, buckets taken below constant bytes, and a bucket of exactly the
bucket cap next to one of cap + 1 (overflow and rerun)."""
import pytest

from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)

ENV = {"B2_SORT_RANGE": "1", "B2_SORT_HYBRID_MIN": "0"}


@pytest.mark.parametrize("carry", ["1", "0"])
def test_emu_sort_range_buckets(emu_lib, carry):
    from tests.snippets.range_sort_buckets import CODE

    run("FILL = 40\n" + CODE, "BUCKETS_OK", env=dict(ENV, B2_SORT_CARRY=carry))

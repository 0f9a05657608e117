"""The range tier of the hybrid sort (radix_sort.cu::range_sort_kernel) on the CPU emulator, forced on at small sizes with
B2_SORT_RANGE=1: range sizes 0, 1, RANGE_CAP and RANGE_CAP + 1 (overflow and rerun), a one-key range longer than the walk
window, float keys, both payload widths, sliced views, and the hybrid plan's skewed and correlated inputs."""
import pytest

from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)

ENV = {"B2_SORT_RANGE": "1", "B2_SORT_HYBRID_MIN": "0"}


@pytest.mark.parametrize("carry", ["1", "0"])
def test_emu_sort_range(emu_lib, carry):
    from tests.snippets.range_sort import CODE

    run("FILL = 40\n" + CODE, "RANGE_OK", env=dict(ENV, B2_SORT_CARRY=carry))


def test_emu_sort_range_hybrid_inputs(emu_lib):
    """The hybrid plan's checks with the range tier on: hot key, equal top bytes (overflow, reruns), duplicate runs, NaN / -0.0."""
    from tests.snippets.hybrid_sort import CODE

    run("SIZES = (3, 2049, 20011)\n" + CODE, "HYBRID_OK", env=ENV)

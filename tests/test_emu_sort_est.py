"""The range tier with estimated bases (radix_sort.cu::run_est_range) on the CPU emulator, forced on at small sizes with
B2_SORT_EST=1: uniform signed and unsigned keys (partial tiles at window ends, empty windows, n not a multiple of the tile), both
payload widths, sorted_order and keys-only sort in both orders, sliced and misaligned views, float keys, a range-sort bucket over
64 equal keys and a constant top digit (both run the exact plan), and windows forced too small by B2_SORT_EST_CAP (every call
overflows and reruns on the exact plan)."""
import pytest

from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)


@pytest.mark.parametrize("carry", ["1", "0"])
def test_emu_sort_est(emu_lib, carry):
    from tests.snippets.sort_est import CODE

    run("SIZES = (3, 2049, 20011)\nEXPECT_RERUN = False\n" + CODE, "EST_OK", env={"B2_SORT_EST": "1", "B2_SORT_CARRY": carry})


def test_emu_sort_est_overflow(emu_lib):
    from tests.snippets.sort_est import CODE

    run("SIZES = (2049, 20011)\nEXPECT_RERUN = True\n" + CODE, "EST_OK", env={"B2_SORT_EST": "1", "B2_SORT_EST_CAP": "16"})

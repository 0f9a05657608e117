"""The partitioned join (radix_join.cu) on the CPU emulator, forced on at small sizes with B2_JOIN_RADIX_ROWS=1: build
chunks of exactly the chunk capacity and one more, the wrap of the slot table, matches in the second half of a probe piece,
the first and last partition, key types and sliced views through the pack kernel, the output-size guess and its rerun, and
the conditions that send a join to the hash table. Each call is also checked for the number of walks it made
(tests/snippets/radix_join.py)."""
from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)


def test_emu_join_radix(emu_lib):
    from tests.snippets.radix_join import CODE

    run("FULL = False\n" + CODE, "RADIX_JOIN_CASES_OK", env={"B2_JOIN_RADIX_ROWS": "1"}, timeout=1800)


def test_emu_join_radix_portions(emu_lib):
    """Several portions per partition pass (B2_SORT_PORTION = three 6144-row tiles)."""
    from tests.snippets.radix_join import PORTION_CODE

    run("FULL = False\n" + PORTION_CODE, "RADIX_JOIN_PORTIONS_OK", env={"B2_JOIN_RADIX_ROWS": "1", "B2_SORT_PORTION": str(3 * 6144)})

"""The range sort's digest walk on the estimated-window tier (tests/snippets/sort_est_digest.py) on the CPU emulator, forced on at
small sizes with B2_SORT_EST=1: keys that agree on their digest and differ below it, equal keys with distinct payloads, and keys
whose varying bits all lie in the digest."""
from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)


def test_emu_sort_est_digest(emu_lib):
    from tests.snippets.sort_est_digest import CODE

    run("SIZES = (2049, 20011)\n" + CODE, "DIGEST_OK", env={"B2_SORT_EST": "1"})

"""The payload-carrying 64-bit sort_by_key pass on the CPU emulator: 8-byte payloads take 512 x 20 tiles, one CTA per SM, key
tiles by one bulk async copy (which the emulator replays with ordinary loads); 4-byte payloads keep the 384 x 16 tile with two
CTAs per SM (the SLICED cases include one)."""
from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (emu_lib is a fixture)

TILE = 512 * 20

# views at row offsets: 8-byte keys at +16 bytes keep every full tile 16-byte aligned (bulk copy); odd offsets do not
# (per-thread loads); the values column is offset independently of the keys
SLICED = r"""
rng = np.random.default_rng(11)
n = 2 * TILE + 5
for koff, voff, vdt in ((0, 0, np.int64), (1, 0, np.int64), (2, 1, np.int64), (3, 2, np.float64), (2, 4, np.int32)):
    for order in (0, 1):
        keys = rng.integers(-2**63, 2**63 - 1, n + 7, dtype=np.int64)
        vals = rng.integers(0, 1 << 30, n + 7).astype(vdt)
        kc = plc.Column.from_numpy(keys).slice(koff, koff + n)
        vc = plc.Column.from_numpy(vals).slice(voff, voff + n)
        got = plc.sorting.sort_by_key(plc.Table([vc]), plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
        exp = osort.sort_by_key([(vals[voff:voff + n], None)], [(keys[koff:koff + n], None)], [order])[0][0]
        assert np.array_equal(got, exp), (koff, voff, vdt, order)
print('SLICED_OK')
"""

# several portions per pass (B2_SORT_PORTION = 2 tiles): per-portion tile counters, look-back rows and digit bases
PORTIONS = r"""
rng = np.random.default_rng(12)
for n in (2 * TILE, 5 * TILE + 77):
    for order in (0, 1):
        keys = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
        keys[::5] = keys[0]
        vals = rng.integers(0, 1 << 62, n).astype(np.int64)
        got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([plc.Column.from_numpy(keys)]), [order], [])
        exp = osort.sort_by_key([(vals, None)], [(keys, None)], [order])[0][0]
        assert np.array_equal(got.columns()[0].to_numpy()[0], exp), (n, order)
print('PORTIONS_OK')
"""


def test_emu_sort_carry_sliced(emu_lib):
    run(f"TILE = {TILE}\n" + SLICED, "SLICED_OK")


def test_emu_sort_carry_portions(emu_lib):
    run(f"TILE = {TILE}\n" + PORTIONS, "PORTIONS_OK", env={"B2_SORT_PORTION": str(2 * TILE), "B2_SORT_HYBRID": "0"})


def test_emu_sort_carry_hybrid_multi_tile(emu_lib):
    """The hybrid plan and its full-LSD rerun over inputs of several 10 240-row tiles."""
    from tests.snippets.hybrid_sort import CODE

    run("SIZES = (10241, 30011)\n" + CODE, "HYBRID_OK", env={"B2_SORT_HYBRID_MIN": "0", "B2_SORT_FIX_FAST": "0"})

"""Shared body of the checks of the range tier with estimated bases (radix_sort.cu::run_est_range: a key sample instead of the
digit histogram, both one-sweep passes into digit windows of `cap` rows, the second one over the first one's gapped windows, the
range sort from the windows into the dense output). Run by tests/test_emu_sort_est.py on the CPU emulator and by
tests/test_sort_est_gpu.py on the GPU with B2_SORT_EST=1 (and B2_SORT_EST_CAP for the forced overflow). `plc`, `np`, `osort`, `L`
are provided by the caller; SIZES scales the cases, EXPECT_RERUN says whether every est attempt must fall back to the exact plan."""
CODE = r"""
rng = np.random.default_rng(11)
L.lib.b2_profile_enable(1)
def prof(name):
    return L.profile_get(name)[1]
def calls(fn):
    # (sample launches, histogram launches) of one call
    s0, h0 = prof('est_sample'), prof('histogram')
    r = fn()
    return r, prof('est_sample') - s0, prof('histogram') - h0
def check(keys, vals=None, order=0, koff=0, voff=0, est=True):
    n = len(keys) - koff
    kc = plc.Column.from_numpy(keys).slice(koff, koff + n)
    keys = keys[koff:]
    outcomes = []
    so, s, h = calls(lambda: plc.sorting.sorted_order(plc.Table([kc]), [order], []).to_numpy()[0])
    outcomes.append(h)
    assert np.array_equal(so, osort.sorted_order([(keys, None)], [order])), ("sorted_order", keys.dtype, n, order)
    if keys.dtype.kind in "iu":
        got, s, h = calls(lambda: plc.sorting.sort(plc.Table([kc]), [order], []).columns()[0].to_numpy()[0])
        outcomes.append(h)
        e = np.sort(keys, kind="stable"); e = e[::-1] if order else e
        assert np.array_equal(got, e), ("sort", keys.dtype, n, order)
    if vals is not None:
        vc = plc.Column.from_numpy(vals).slice(voff, voff + n)
        got, s, h = calls(lambda: plc.sorting.sort_by_key(plc.Table([vc]), plc.Table([kc]), [order], []).columns()[0].to_numpy()[0])
        outcomes.append(h)
        ex = osort.sort_by_key([(vals[voff:voff + n], None)], [(keys, None)], [order])[0][0]
        assert np.array_equal(got, ex), ("sort_by_key", keys.dtype, vals.dtype, n, order, koff, voff)
    if est is None:
        return
    if est and not EXPECT_RERUN:
        assert all(h == 0 for h in outcomes), ("est mode fell back", keys.dtype, n, order, outcomes)
    else:
        assert all(h > 0 for h in outcomes), ("exact plan expected", keys.dtype, n, order, outcomes)
for n in SIZES:
    for order in (0, 1):
        # uniform signed / unsigned keys, 8- and 4-byte payloads: partial tiles at every window end, n not a multiple of the tile
        k = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
        check(k, rng.integers(0, 1 << 62, n).astype(np.int64), order)
        check(k.view(np.uint64), rng.integers(0, 1 << 30, n).astype(np.int32), order)
        # top bytes in a few values only: most windows empty
        k = (rng.integers(0, 3, n).astype(np.int64) << 56) | (rng.integers(0, 5, n).astype(np.int64) << 48) | rng.integers(0, 1 << 48, n)
        check(k, rng.standard_normal(n), order, est=None)  # skewed top byte: the sample may decline
# sliced and misaligned views of keys and payload
n = SIZES[-1]
k = rng.integers(-2**63, 2**63 - 1, n + 3, dtype=np.int64)
for koff, voff, vdt in ((1, 0, np.int64), (2, 1, np.int64), (3, 2, np.int32)):
    check(k, rng.integers(0, 1 << 30, n + 3).astype(vdt), koff % 2, koff, voff)
# float keys, ascending (descending float row ids need the NaN count: exact plan); results only
f = rng.standard_normal(n) * 1e10
f[rng.integers(0, n, 20)] = np.nan   # a few: more than 64 equal keys in one range-sort bucket would overflow it
f[rng.integers(0, n, 20)] = -0.0
check(f, rng.integers(0, 1 << 40, n).astype(np.int64), 0, est=None)  # few exponents: at larger n the sample declines
if not EXPECT_RERUN:
    # a bucket of the range sort over 64 rows of one key: the range sort overflows and the exact plan reruns
    k = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    k[rng.integers(0, n, 200)] = 123456789
    check(k, rng.integers(0, 1 << 40, n).astype(np.int64), 0, est=False)
    # a constant top digit: est mode is not taken
    k = rng.integers(0, 1 << 56, n, dtype=np.int64) | (np.int64(7) << 56)
    check(k, rng.integers(0, 1 << 40, n).astype(np.int64), 1, est=False)
print('EST_OK')
"""

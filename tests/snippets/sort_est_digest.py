"""Shared body of the checks of the range sort's digest walk on the estimated-window tier (radix_sort.cu::range_sort_kernel<VT,
true>: the bucket order holds a 16-bit key digest beside each local row, and only rows whose digests are equal are compared by
whole keys). Run by tests/test_emu_sort_est_digest.py on the CPU emulator and tests/test_sort_est_digest_gpu.py on the GPU, with
B2_SORT_EST=1. `plc`, `np`, `osort`, `L` are provided by the caller; SIZES scales the cases. Every call must take the tier (no
digit histogram)."""
CODE = r"""
rng = np.random.default_rng(23)
L.lib.b2_profile_enable(1)
def check(keys, vals, what):
    kc, vc = plc.Column.from_numpy(keys), plc.Column.from_numpy(vals)
    for order in (0, 1):
        h0 = L.profile_get('histogram')[1]
        got = plc.sorting.sort_by_key(plc.Table([vc]), plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
        ex = osort.sort_by_key([(vals, None)], [(keys, None)], [order])[0][0]
        assert np.array_equal(got, ex), ("sort_by_key", what, len(keys), order)
        so = plc.sorting.sorted_order(plc.Table([kc]), [order], []).to_numpy()[0]
        assert np.array_equal(so, osort.sorted_order([(keys, None)], [order])), ("sorted_order", what, len(keys), order)
        s = plc.sorting.sort(plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
        e = np.sort(keys, kind="stable")
        assert np.array_equal(s, e[::-1] if order else e), ("sort", what, len(keys), order)
        assert L.profile_get('histogram')[1] == h0, ("the estimated-window tier was not taken", what, len(keys), order)
for n in SIZES:
    vals = rng.integers(0, 1 << 62, n).astype(np.int64)
    # groups of up to 6 keys that agree on bits 24..63 (range id, bucket and the 16 digest bits below it while ranges hold at
    # most 256 rows) and differ only below: every comparison inside a group goes past the digest to the whole keys
    base = rng.integers(-2**63, 2**63 - 1, (n + 5) // 6, dtype=np.int64) & ~np.int64((1 << 24) - 1)
    k = np.repeat(base, 6)[:n] | rng.integers(0, 1 << 24, n)
    check(k[rng.permutation(n)], vals, "equal digests")
    # the same groups with equal keys: ties keep the input order (distinct payloads)
    k = np.repeat(base, 6)[:n] | rng.integers(0, 4, n)
    check(k[rng.permutation(n)], vals, "ties")
    # only bits 48..63 and 0..9 vary: the bucket bits lie below bit 16, so the digest holds every varying bit
    k = (rng.integers(-2**15, 2**15 - 1, n, dtype=np.int64) << 48) | rng.integers(0, 1 << 10, n)
    check(k, vals, "low bits only")
print('DIGEST_OK')
"""

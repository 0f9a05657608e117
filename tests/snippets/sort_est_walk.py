"""Shared body of the boundary checks of the range sort on the estimated-window tier (radix_sort.cu::range_sort_kernel<VT, true>,
1024 threads: per = 2^max(nb - 10, 0) buckets per thread in the scan, 16 rows per thread in the walk, which walks the buckets of
RANGE_WALK_ROWS rows side by side). Run by tests/test_sort_est_walk_gpu.py on the GPU and tests/test_emu_sort_est_walk.py on the
CPU emulator, where the kernel keeps 512 threads (per up to 16, 32 rows per thread), with B2_SORT_EST=1; B2_SORT_EST_CAP is set per input to its widest digit window, so no key sample decides. `plc`,
`np`, `osort`, `L` are provided by the caller.

Every range is built bucket by bucket: the range sort buckets a range of m rows by the nb = min(ceil(log2 m), 13) key bits below
bit 48 (bit 47 varies over each input), and orders a bucket by the 16 bits below those (the digest), then by whole keys."""
CODE = r"""
import os
rng = np.random.default_rng(29)
L.lib.b2_profile_enable(1)
SIGN = np.uint64(1 << 63)

def range_keys(rid, counts, tie=()):
    # counts[b] rows in bucket b of range rid; the rows of a bucket in `tie` share their digest and differ only below it, often not
    # at all (equal keys keep their input order)
    m = int(sum(counts))
    nb = min((m - 1).bit_length(), 13)
    bshift = 48 - nb
    dshift = bshift - 16
    out = []
    for b, c in enumerate(counts):
        if c == 0:
            continue
        hi = (rid << 48) | (b << bshift)
        if b in tie:
            low = (int(rng.integers(0, 1 << 16)) << dshift) + rng.integers(0, 3, c)
        else:
            low = rng.integers(0, 1 << bshift, c)
        out.append(np.uint64(hi) + low.astype(np.uint64))
    return np.concatenate(out)

def spread(m):
    # m rows evenly over the range's buckets
    nb = min((m - 1).bit_length(), 13)
    return [int(c) for c in np.bincount(np.arange(m) * (1 << nb) // m, minlength=1 << nb)]

def with_bucket(m, big):
    # buckets 5, 6, ... hold big[0], big[1], ... rows; one row in each of the next buckets up to m rows
    c = [1] * 5 + list(big)
    c += [1] * (m - sum(c))
    return c

def straddle(m, size):
    # single-row buckets except two tie buckets of `size` rows, at positions 28 .. 27 + size from either end: both orders put one
    # across the first warp's 32 positions
    n1 = m - 2 * size
    c = [1] * 28 + [size] + [1] * (n1 - 56) + [size] + [1] * 28
    return c, (28, 28 + 1 + n1 - 56)

def check(parts, what, tier=True):
    u = np.concatenate([range_keys((i + 1) << 8 | (37 * i + 11) & 255, c, t) for i, (c, t) in enumerate(parts)])
    u = u[rng.permutation(len(u))]
    os.environ['B2_SORT_EST_CAP'] = str(max(sum(c) for c, _ in parts) + 15 & ~15)
    keys = (u ^ SIGN).view(np.int64)
    n = len(keys)
    kc = plc.Column.from_numpy(keys)
    for order in (0, 1):
        for vdt in (np.int64, np.int32):
            vals = rng.integers(0, 1 << 30, n).astype(vdt)
            h0 = L.profile_get('histogram')[1]
            got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
            ex = osort.sort_by_key([(vals, None)], [(keys, None)], [order])[0][0]
            assert np.array_equal(got, ex), ("sort_by_key", what, vdt, order)
            assert (L.profile_get('histogram')[1] == h0) == tier, ("tier taken" if not tier else "tier not taken", what, vdt, order)
        h0 = L.profile_get('histogram')[1]
        so = plc.sorting.sorted_order(plc.Table([kc]), [order], []).to_numpy()[0]
        assert np.array_equal(so, osort.sorted_order([(keys, None)], [order])), ("sorted_order", what, order)
        s = plc.sorting.sort(plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
        e = np.sort(keys, kind="stable")
        assert np.array_equal(s, e[::-1] if order else e), ("sort", what, order)
        assert (L.profile_get('histogram')[1] == h0) == tier, ("tier taken" if not tier else "tier not taken", what, order)

# range lengths around the thread count and RANGE_CAP; nb = 0, 5, 10 (per 1), 11 (per 2), 12 (per 4), 13 (per 8)
check([(spread(m), ()) for m in (1, 31, 32, 1023, 1024, 1025, 2048, 4000, 16384)], "range lengths")
# crowded buckets: all rows of a range in one to three buckets
check([([m], ()) for m in (2, 31, 64)] + [([40, 0, 3, 0, 21], ())], "crowded buckets")
# a bucket of exactly RANGE_BUCKET_CAP rows beside one of 63; three such buckets in a row, all digest ties; tie buckets across the
# first warp's 32 positions at per = 1, 4 and 8
check([(with_bucket(2048, (64, 63)), ()), (with_bucket(1500, (64, 64, 64)), (5, 6, 7)), straddle(1024, 8), straddle(3000, 40),
       straddle(8000, 64)], "bucket sizes and ties")
# overflows: a range over RANGE_CAP rows, a bucket of 65 rows; the exact plan reruns
check([(spread(16385), ())], "range over RANGE_CAP", tier=False)
check([(with_bucket(2048, (64, 65)), ())], "bucket over RANGE_BUCKET_CAP", tier=False)
print('WALK_OK')
"""

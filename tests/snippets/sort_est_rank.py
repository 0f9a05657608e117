"""Shared body of the checks of the range sort's bounded walk on the estimated-window tier (radix_sort.cu::range_sort_kernel<VT,
true>): the walk takes RANGE_WALK_STEPS = 4 unrolled steps over each row's bucket and finishes longer buckets in a tail loop. Run by
tests/test_sort_est_rank_gpu.py on the GPU (1024 threads) and tests/test_emu_sort_est_rank.py on the CPU emulator (512 threads),
with B2_SORT_EST=1 and B2_SORT_EST_CAP set to the widest range. `plc`, `np`, `L` are provided by the caller.

Every range is built bucket by bucket, as in tests/snippets/sort_est_walk.py: the range sort buckets a range of m rows by the
nb = min(ceil(log2 m), 13) key bits below bit 48, and orders a bucket by the 16 bits below those (the digest), then by whole keys.
Payloads are distinct, so a result is bit-exact against a stable numpy argsort of the keys only if every row lands in place."""
CODE = r"""
import os
rng = np.random.default_rng(31)
L.lib.b2_profile_enable(1)
SIGN = np.uint64(1 << 63)
K = 4  # RANGE_WALK_STEPS

def range_keys(rid, counts, tie={}):
    # counts[b] rows in bucket b of range rid; the rows of a bucket b in `tie` share one digest and take tie[b] distinct values
    # below it (1: all keys of the bucket are equal)
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
            low = (int(rng.integers(0, 1 << 16)) << dshift) + rng.integers(0, tie[b], c)
        else:
            low = rng.integers(0, 1 << bshift, c)
        out.append(np.uint64(hi) + low.astype(np.uint64))
    return np.concatenate(out)

def pad(m, c):
    # the buckets c, then single-row buckets up to m rows
    return list(c) + [1] * (m - sum(c))

def clustered(m, spread):
    # m rows over the first 1 / spread of the range's buckets: ~spread times the usual rows per bucket, so many buckets run past
    # the K unrolled steps; no bucket over RANGE_BUCKET_CAP
    nb = min((m - 1).bit_length(), 13)
    while True:
        c = np.bincount(rng.integers(0, max((1 << nb) // spread, 1), m), minlength=1 << nb)
        if c.max() <= 64:
            return [int(x) for x in c]

def check(parts, what, tier=True):
    u = np.concatenate([range_keys((i + 1) << 8 | (37 * i + 11) & 255, c, t) for i, (c, t) in enumerate(parts)])
    u = u[rng.permutation(len(u))]
    os.environ['B2_SORT_EST_CAP'] = str(max(sum(c) for c, _ in parts) + 15 & ~15)
    keys = (u ^ SIGN).view(np.int64)
    n = len(keys)
    kc = plc.Column.from_numpy(keys)
    order = np.argsort(keys, kind="stable")
    h0 = L.profile_get('histogram')[1]
    for vdt in (np.int64, np.int32):
        vals = rng.permutation(n).astype(vdt)
        got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([kc]), [0], []).columns()[0].to_numpy()[0]
        assert np.array_equal(got, vals[order]), ("sort_by_key", what, vdt)
    so = plc.sorting.sorted_order(plc.Table([kc]), [0], []).to_numpy()[0]
    assert np.array_equal(so, order), ("sorted_order", what)
    assert (L.profile_get('histogram')[1] == h0) == tier, ("tier taken" if not tier else "tier not taken", what)

parts = [
    # buckets of exactly K and K + 1 rows and of RANGE_BUCKET_CAP rows, side by side and apart (per = 2)
    (pad(2048, [1, K, K + 1, 1, 64, K, 2, K + 1, 64, K + 1, K]), {}),
    # every bucket longer than K: every row of every warp finishes in the tail (per = 4)
    ([6, 7, 9, 12, 33, 64, 8, 6] * 20 + [15], {}),
    # long buckets at the last positions before m, at m = 1025 and at a thread-count multiple
    (pad(1025 - 20 - 64, []) + [20, 64], {}),
    (pad(2048 - 7 - K - 1, []) + [7, K + 1], {}),
    # digest ties inside long buckets: tied rows in the unrolled steps and in the tail, a tie bucket of exactly K + 1 rows, and
    # buckets of equal keys (payloads keep their input order)
    (pad(3000, [1, 40, 3, K + 1, 64, 12, 2, 9]), {1: 3, 3: 1, 4: 2, 5: 1, 7: 2}),
    # long and short buckets at every buckets-per-thread count of the scan: per = 1, 2, 4, 8 at 1024 threads
    (clustered(1000, 3), {}), (clustered(2000, 3), {}), (clustered(4000, 4), {}), (clustered(16000, 3), {}),
    # range lengths around the thread count (512 on the emulator, 1024 on the GPU), twice it, and RANGE_CAP
] + [(clustered(m, 3), {}) for m in (511, 513, 1023, 1024, 2047, 2048, 16384)]
check(parts, "walk steps and tail")
# a bucket of 65 rows overflows, and the exact plan reruns
check([(pad(2048, [1, K + 1, 65]), {})], "bucket over RANGE_BUCKET_CAP", tier=False)
print('RANK_OK')
"""

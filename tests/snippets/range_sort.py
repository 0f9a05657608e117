"""Shared body of the checks of the hybrid sort's range tier (radix_sort.cu::range_sort_kernel: LSD passes over the top
digit(s) only, then each range of rows sharing them is sorted in shared memory). Run by tests/test_emu_sort_range.py on the CPU
emulator and by tests/test_sort_range_gpu.py on the GPU, both with B2_SORT_RANGE=1 and B2_SORT_HYBRID_MIN=0 so that small
inputs take the tier. `plc`, `np`, `osort`, `L` are provided by the caller; FILL is the number of rows of every other top byte."""
CODE = r"""
rng = np.random.default_rng(9)
CAP = 16384
def check(keys, vals=None, order=0, koff=0, voff=0):
    n = len(keys) - koff
    kc = plc.Column.from_numpy(keys).slice(koff, koff + n)
    keys = keys[koff:]
    so = plc.sorting.sorted_order(plc.Table([kc]), [order], []).to_numpy()[0]
    assert np.array_equal(so, osort.sorted_order([(keys, None)], [order])), ("sorted_order", keys.dtype, n, order)
    if keys.dtype.kind in "iu":
        s = plc.sorting.sort(plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
        e = np.sort(keys, kind="stable"); e = e[::-1] if order else e
        assert np.array_equal(s, e), ("sort", keys.dtype, n, order)
    if vals is not None:
        vc = plc.Column.from_numpy(vals).slice(voff, voff + n)
        got = plc.sorting.sort_by_key(plc.Table([vc]), plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
        ex = osort.sort_by_key([(vals[voff:voff + n], None)], [(keys, None)], [order])[0][0]
        assert np.array_equal(got, ex), ("sort_by_key", keys.dtype, vals.dtype, n, order, koff, voff)
def by_top_byte(sizes):
    # keys whose top byte b occurs sizes[b] times (the ranges of the one-digit range id), random low 56 bits, shuffled
    top = np.repeat(np.arange(256, dtype=np.uint64), sizes)
    k = (top << np.uint64(56)) | rng.integers(0, 1 << 56, len(top), dtype=np.uint64)
    return rng.permutation(k).view(np.int64) ^ np.int64(-2**63)   # signed: the twiddle maps the top byte back to b
for big in (CAP, CAP + 1):   # a range of RANGE_CAP rows fits; one more row overflows and reruns on the hybrid plan
    sizes = np.full(256, FILL); sizes[0] = 0; sizes[1] = 1; sizes[2] = big
    k = by_top_byte(sizes)
    for order in (0, 1):
        check(k, rng.integers(0, 1 << 62, len(k)).astype(np.int64), order)
        check(k, rng.standard_normal(len(k)).astype(np.float32), order)
# one range that is all one key, much longer than the walk window
sizes = np.full(256, FILL); sizes[5] = 3000
k = by_top_byte(sizes)
k[(k >> 56) == (5 - 128)] = (5 - 128) << 56 | 1234567
for order in (0, 1):
    check(k, rng.integers(0, 1 << 62, len(k)).astype(np.int64), order)
# key and value views at row offsets (the first pass takes per-thread loads for unaligned tiles)
k = by_top_byte(np.full(256, FILL))
k = np.concatenate([k, k[:3]])
for koff, voff, vdt in ((1, 0, np.int64), (2, 1, np.int64), (3, 2, np.int32)):
    check(k, rng.integers(0, 1 << 30, len(k)).astype(vdt), 1, koff, voff)
# float keys: NaN, -0.0 and +0.0, both orders
f = rng.standard_normal(256 * FILL) * 1e10
f[rng.integers(0, len(f), len(f) // 10)] = np.nan
f[rng.integers(0, len(f), len(f) // 10)] = -0.0
f[rng.integers(0, len(f), len(f) // 10)] = 0.0
for order in (0, 1):
    check(f, rng.integers(0, 1 << 62, len(f)).astype(np.int64) if order == 0 else None, order)
print('RANGE_OK')
"""

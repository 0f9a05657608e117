"""Shared body of the checks of the range tier's bucket sort (radix_sort.cu::range_sort_kernel: each range is grouped by the
bits below its range id that vary over the input, then every bucket is ordered by (key, input row)). Run by
tests/test_emu_sort_range_buckets.py on the CPU emulator and by tests/test_sort_range_buckets_gpu.py on the GPU, both with
B2_SORT_RANGE=1 and B2_SORT_HYBRID_MIN=0 so that small inputs take the tier. `plc`, `np`, `osort`, `L` are provided by the
caller; FILL is the number of rows of every range (top byte) but one, which holds BIG rows.

Whether a sort reran without the tier is read from the profiling scopes: the range sort runs under `segment_fix`, and a rerun
on the hybrid plan adds a second `segment_fix` scope."""
CODE = r"""
rng = np.random.default_rng(31)
BIG = 200          # rows of range 3: 8 bucket bits, i.e. the byte just below the range id when that byte varies
BUCKET_CAP = 64    # rows of one bucket; one more raises the overflow flag

def build(sizes, low_of):
    # range b holds sizes[b] keys (b << 56) | low_of(b, sizes[b]), shuffled; signed keys whose twiddled top byte is b
    parts = [(np.uint64(b) << np.uint64(56)) | low_of(b, int(c)) for b, c in enumerate(sizes)]
    return rng.permutation(np.concatenate(parts)).view(np.int64) ^ np.int64(-2**63)

def rand56(b, c):
    return rng.integers(0, 1 << 56, c, dtype=np.uint64)

def runs(b, c):
    # half the rows of every range take one of six values: many short runs of equal keys next to distinct ones
    x = rand56(b, c)
    pool = rng.integers(0, 1 << 56, 6, dtype=np.uint64)
    pick = rng.random(c) < 0.5
    x[pick] = pool[rng.integers(0, 6, int(pick.sum()))]
    return x

def const_below(b, c):
    # bytes 6 and 5 are the same in every key: the buckets must come from the bits below them
    return rng.integers(0, 1 << 40, c, dtype=np.uint64) | np.uint64(0x5A5A << 40)

def crafted(hot):
    # range 3: exactly `hot` rows whose byte 6 (their bucket) is 0x5A, no other row of the range has it
    def low(b, c):
        x = rand56(b, c)
        if b == 3:
            d6 = rng.integers(0, 255, c, dtype=np.uint64)
            d6[d6 >= 0x5A] += np.uint64(1)
            d6[:hot] = 0x5A
            x = (x & np.uint64((1 << 48) - 1)) | (d6 << np.uint64(48))
        return x
    return low

def check(keys, order, rerun, vdt):
    n = len(keys)
    vals = rng.permutation(n).astype(vdt)   # distinct payloads: equal keys must keep their input order
    kc = plc.Column.from_numpy(keys)
    L.lib.b2_profile_reset()
    L.lib.b2_profile_enable(1)
    got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
    L.lib.b2_profile_enable(0)
    assert L.profile_get('range_bounds')[1] == 1, 'the range tier was not taken'
    assert L.profile_get('segment_fix')[1] == (2 if rerun else 1), ('rerun expected' if rerun else 'unexpected rerun', order)
    ex = osort.sort_by_key([(vals, None)], [(keys, None)], [order])[0][0]
    assert np.array_equal(got, ex), ('sort_by_key', order, vdt)
    so = plc.sorting.sorted_order(plc.Table([kc]), [order], []).to_numpy()[0]
    assert np.array_equal(so, osort.sorted_order([(keys, None)], [order])), ('sorted_order', order)
    s = plc.sorting.sort(plc.Table([kc]), [order], []).columns()[0].to_numpy()[0]
    e = np.sort(keys, kind='stable')
    assert np.array_equal(s, e[::-1] if order else e), ('sort', order)

sizes = np.full(256, FILL)
sizes[3] = BIG
for order, vdt in ((0, np.int64), (1, np.int32)):
    check(build(sizes, runs), order, False, vdt)
    check(build(sizes, const_below), order, False, vdt)
for hot, rerun in ((BUCKET_CAP, False), (BUCKET_CAP + 1, True)):
    check(build(sizes, crafted(hot)), 0, rerun, np.int64)
print('BUCKETS_OK')
"""

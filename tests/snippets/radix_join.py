"""Shared body of the checks of the partitioned join (radix_join.cu: rj_join_kernel) at the constants where its index
arithmetic can go wrong. Run by tests/test_emu_join_radix.py on the CPU
emulator and by tests/test_join_radix_gpu.py on the GPU, both with B2_JOIN_RADIX_ROWS=1 so that small inputs take the
path. `plc`, `np`, `ojoin`, `L` are provided by the caller; FULL = False drops the slowest sizes of a case (the emulator).

The keys are built from the value the kernels work on: h = mix64(packed key) is a bijection, so a case picks h and uses
unmix64(h) as its key. The partition of a row is h >> 48 and its slot is bits 33..47 of h. Within a partition both sides
keep their input order (the partition passes are stable), so a case also decides which build chunk and which probe piece a
row lands in.

Which path ran is read from the profiling scopes: radix_join opens one `rjoin_join` scope per walk, so a call that took the
hash table shows 0, a normal call 1 and a call whose output outgrew the size guess (and walked again) 2."""
HELPERS = r"""
import os
rng = np.random.default_rng(2024)
CAP = 16384      # build rows per shared-memory chunk (RJ_CAP)
PIECE = 65536    # probe rows per work item (RJ_PIECE): 64 rows per thread
U = np.uint64

def mix64(k):
    k = np.array(k, dtype=U)
    k ^= k >> U(33); k *= U(0xff51afd7ed558ccd)
    k ^= k >> U(33); k *= U(0xc4ceb9fe1a85ec53)
    k ^= k >> U(33)
    return k

def unmix64(k):
    k = np.array(k, dtype=U)
    k ^= k >> U(33); k *= U(0x9cb4b2f8129337db)
    k ^= k >> U(33); k *= U(0x4f74430c22a54005)
    k ^= k >> U(33)
    return k

_t = rng.integers(0, 2**64, 100_000, dtype=U, endpoint=False)
assert np.array_equal(mix64(unmix64(_t)), _t) and np.array_equal(unmix64(mix64(_t)), _t)

def k1_slot(h):
    return (h >> U(33)) & U(32767)

def f64_ok(h):
    # the key bits must survive the float64 normalisation unchanged: no NaN, no -0.0
    k = unmix64(h)
    return ~np.isnan(k.view(np.float64)) & (k != U(1 << 63))

def draw(n, part, low_bits=48, fixed=0):
    # n distinct h in partition `part`: bits below low_bits random, `fixed` or-ed in
    out = np.empty(0, U)
    while len(out) < n:
        c = (U(part) << U(48)) | U(fixed) | rng.integers(0, 1 << low_bits, 2 * n + 16, dtype=U)
        out = np.unique(np.concatenate([out, c[f64_ok(c)]]))
    return rng.permutation(out)[:n]

def draw_outside(n, avoid):
    # n distinct h in random partitions other than those in `avoid`
    out = np.empty(0, U)
    while len(out) < n:
        c = rng.integers(0, 2**64, 2 * n + 16, dtype=U, endpoint=False)
        c = c[f64_ok(c) & ~np.isin(c >> U(48), np.array(list(avoid), U))]
        out = np.unique(np.concatenate([out, c]))
    return rng.permutation(out)[:n]

def cols(h, form):
    # the key column(s) whose packed form is unmix64(h)
    k = unmix64(h)
    if form == 'i64':   # one 8-byte integer column: partitioned in place
        return [(k.view(np.int64), None)]
    if form == 'i32x2':  # low and high halves: packed by rj_pack_kernel
        return [((k & U(0xFFFFFFFF)).astype(np.uint32).view(np.int32), None), ((k >> U(32)).astype(np.uint32).view(np.int32), None)]
    if form == 'f64':   # a float key is always packed (normalised)
        return [(k.view(np.float64), None)]
    raise ValueError(form)

CASE = ''

def table(cs, off):
    out = []
    for v, m in cs:
        if off:
            # the view starts `off` rows into its buffer; the rows in front are other keys of the same column, so a kernel that
            # ignores the offset pairs the wrong rows
            pad = rng.permutation(np.resize(v, off))
            c = plc.Column.from_numpy(np.concatenate([pad, v]), None if m is None else np.concatenate([np.ones(off, bool), m]))
            c = c.slice(off, off + len(v))
        else:
            c = plc.Column.from_numpy(v, m)
        out.append(c)
    return plc.Table(out)

def check(l, r, kinds, expect_rjoin_calls, off=(0, 0)):
    # the join of the left table `l` with the right table `r` as canonical pairs against the oracle, and the number of
    # rjoin_join scopes it opened
    for kind in kinds:
        exp = getattr(ojoin, kind)(l, r)
        tl, tr = table(l, off[0]), table(r, off[1])
        L.lib.b2_profile_reset()
        L.lib.b2_profile_enable(1)
        res = getattr(plc.join, kind)(tl, tr, 0)
        L.lib.b2_profile_enable(0)
        calls = L.profile_get('rjoin_join')[1]
        got = ojoin.canonical(res[0].to_numpy()[0], res[1].to_numpy()[0])
        same = len(got[0]) == len(exp[0]) and np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
        assert same, (CASE, kind, 'pairs', len(got[0]), 'expected', len(exp[0]))
        assert calls == expect_rjoin_calls, (CASE, kind, 'rjoin_join scopes', calls, 'expected', expect_rjoin_calls)
"""

CASES = r"""
FORMS = ('i64', 'i32x2', 'f64')
# a full join is the left join's walk plus the unmatched build rows appended by hash_join_finalize_full
ALL = ('inner_join', 'left_join', 'full_join') if FULL else ('inner_join', 'left_join')

# ---- build chunks: one partition with CAP, CAP + 1, 2 CAP and 2 CAP + 1 distinct build keys (chunk loop c0 += CAP) ----
P = 0x1234
for i, nb in enumerate((CAP, CAP + 1, 2 * CAP, 2 * CAP + 1) if FULL else (CAP + 1, 2 * CAP + 1)):
    CASE = f'chunks nb={nb}'
    h = draw(nb + 1500, P)
    bh, absent = h[:nb], h[nb:]
    others = draw_outside(1500, {P})
    b = np.concatenate([bh, others[:500]])           # build rows of other partitions that no probe row has
    p = rng.permutation(np.concatenate([bh, absent, others[500:]]))
    form = FORMS[i % 3]
    check(cols(p, form), cols(b, form), ALL, 1)

# ---- the 32768-slot table wraps: ~3000 build keys of one partition all in slot 32767 ----
CASE = 'slot wrap'
P = 0x4321
W = 3000 if FULL else 400
h = draw(W + W // 3, P, low_bits=33, fixed=32767 << 33)
assert (k1_slot(h) == 32767).all() and (h >> U(48) == P).all()
bh, absent = h[:W], h[W:]
p = rng.permutation(np.concatenate([bh, absent, bh[:W // 2]]))
check(cols(p, 'i64'), cols(bh, 'i64'), ('inner_join', 'left_join'), 1)

# ---- probe pieces: matches only in the second half of a piece (k >= 32: the `32 + __ffs` branch) and only in build chunk 2 ----
P = 0xBEEF
for i, n_probe in enumerate((PIECE - 1, PIECE, PIECE + 1, 2 * PIECE + 1) if FULL else (PIECE + 1,)):
    CASE = f'pieces n_probe={n_probe}'
    nb = CAP + 600
    h = draw(nb + 3000, P)
    bh, absent = h[:nb], h[nb:]
    second = bh[CAP:]                                 # the build rows of chunk 2 (partition order is input order)
    j = np.arange(n_probe) % PIECE
    late = j >= PIECE // 2                           # row k * threads + tid of its piece with k >= 32
    p = absent[rng.integers(0, len(absent), n_probe)]
    p[late] = second[rng.integers(0, len(second), int(late.sum()))]
    form = FORMS[i % 3]
    check(cols(p, form), cols(bh, form), ('inner_join', 'left_join'), 1)

# ---- partitions 0 and 65535 only (rj_bounds_kernel at both ends); left joins whose probe partition has no build rows ----
CASE = 'edge partitions'
h0, h1 = draw(700, 0), draw(700, 0xFFFF)
b = np.concatenate([h0[:400], h1[:400]])
p = rng.permutation(np.concatenate([h0[200:], h1[200:], h1[:50]]))
check(cols(p, 'i64'), cols(b, 'i64'), ALL, 1)
CASE = 'probe partition without build rows'
check(cols(h1, 'i64'), cols(h0[:300], 'i64'), ALL, 1)
check(cols(h0, 'f64'), cols(h1[:300], 'f64'), ALL, 1)

# ---- key types through rj_pack_kernel: pack_row's normalisation against the oracle's row equality ----
# The right (build) side holds each key at most once, so no call outgrows the one-pair-per-probe-row guess.
def pool_keys(pool, n):
    return pool[rng.integers(0, len(pool), n)]
def some_of(pool):
    u = rng.permutation(np.unique(pool))
    return u[:max(1, len(u) * 3 // 4)]
ii = lambda t: np.iinfo(t)
for dt, pool in ((np.int8, np.arange(-128, 128, dtype=np.int8)),
                 (np.int16, np.array([ii(np.int16).min, -1, 0, 1, 255, 256, ii(np.int16).max] + list(range(-300, 300, 7)), np.int16)),
                 (np.int32, np.array([ii(np.int32).min, -1, 0, 1, ii(np.int32).max] + list(range(-5000, 5000, 37)), np.int32)),
                 (np.uint32, np.array([0, 1, 2**31, 2**32 - 1] + list(range(0, 2**32 - 1, 2**32 // 257)), np.uint32)),
                 (np.uint64, np.array([0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 1] + [2**63 + 3 * i for i in range(200)], np.uint64)),
                 (np.int64, np.array([ii(np.int64).min, ii(np.int64).min + 1, -1, 0, 1, ii(np.int64).max - 1, ii(np.int64).max], np.int64))):
    CASE = f'keys {np.dtype(dt).name}'
    check([(pool_keys(pool, 3000), None)], [(some_of(pool), None)], ('inner_join', 'full_join') if FULL else ('inner_join',), 1)
CASE = 'keys bool'   # inner: exactly one pair per probe row, the size of the guess (the m == capacity hand-back)
check([(rng.random(300) < 0.3, None)], [(np.array([True, False]), None)], ('inner_join', 'left_join'), 1)
nan64 = np.array([0x7ff8000000000000, 0x7ff0000000000001, 0xfff8000000000000, 0x7fffffffffffffff, 0xfff0000000000abc], U).view(np.float64)
nan32 = np.array([0x7fc00000, 0x7f800001, 0xffc00000, 0x7fffffff, 0xff800abc], np.uint32).view(np.float32)
for dt, nans in ((np.float64, nan64), (np.float32, nan32)):
    CASE = f'keys {np.dtype(dt).name} specials'
    tiny = 2.0 ** -1074 if dt == np.float64 else 1e-45
    normal = rng.standard_normal(200).astype(dt)
    pool = np.concatenate([nans, np.array([0.0, -0.0, np.inf, -np.inf, tiny, -tiny], dt), normal])
    # one NaN (payload 4, not the canonical one) and -0.0 on the build side; every payload and both zeros on the probe side
    build = rng.permutation(np.concatenate([nans[3:4], np.array([-0.0, np.inf, -np.inf, tiny], dt), normal[:150]]))
    check([(pool_keys(pool, 3000), None)], [(build, None)], ALL, 1)
CASE = 'packed int32 + int16 + int8 + bool (8 bytes)'
grid = np.stack(np.meshgrid(np.arange(-3, 3), np.arange(-2, 2), np.arange(-2, 2), np.arange(2), indexing='ij'), -1).reshape(-1, 4)
def four(rows):
    return [((rows[:, 0] * 1_000_003).astype(np.int32), None), ((rows[:, 1] * 4099).astype(np.int16), None),
            ((rows[:, 2] * 63).astype(np.int8), None), (rows[:, 3].astype(bool), None)]
check(four(grid[rng.integers(0, len(grid), 4000)]), four(grid[rng.permutation(len(grid))[:150]]), ALL, 1)

# ---- sliced views: src = data + offset (in-place int64 path) and kc.offset (packed path) ----
for form in ('i64', 'i32x2'):
    CASE = f'sliced {form}'
    h = draw_outside(6000, set())
    bh = h[:3000]
    p = rng.permutation(np.concatenate([bh[:2000], h[3000:]]))
    check(cols(p, form), cols(bh, form), ALL, 1, off=(37, 1000))

# ---- inner joins build on the smaller side and swap the outputs back ----
for nl, nr in ((5000, 3000), (3000, 5000), (4000, 4000)):
    CASE = f'build side nl={nl} nr={nr}'
    check([(rng.integers(0, 20_000, nl), None)], [(rng.integers(0, 20_000, nr), None)], ('inner_join',), 1)

# ---- the output-size guess: one pair per probe row (left joins 1.25) and the exact-size rerun ----
CASE = 'rerun: 4 build copies of every key'
keys = draw_outside(2000, set())
b = rng.permutation(np.repeat(keys, 4))
p = keys[rng.integers(0, len(keys), 10_000)]
check(cols(p, 'i64'), cols(b, 'i64'), ALL, 2)
CASE = 'left join between 1 and 1.25 pairs per probe row'
b = rng.permutation(np.concatenate([keys, keys[:200]]))      # 10 % of the keys twice
p = keys[rng.integers(0, len(keys), 10_000)]
m = len(ojoin.left_join(cols(p, 'i64'), cols(b, 'i64'))[0])
assert 10_000 < m < 12_500, m
check(cols(p, 'i64'), cols(b, 'i64'), ('left_join', 'full_join'), 1)
CASE = 'output size hook'
p = rng.permutation(np.concatenate([keys[:1500], keys[:300], draw_outside(500, set())]))
b = rng.permutation(np.concatenate([keys, keys[:700]]))
m = len(ojoin.inner_join(cols(p, 'i64'), cols(b, 'i64'))[0])
for cap, walks in ((m, 1), (m - 1, 2), (m + 1, 1)):
    os.environ['B2_JOIN_RADIX_CAPACITY'] = str(cap)
    CASE = f'output size hook capacity={cap} pairs={m}'
    check(cols(p, 'i64'), cols(b, 'i64'), ('inner_join',), walks)
del os.environ['B2_JOIN_RADIX_CAPACITY']

# ---- tile edges of the partition passes (384 x 16 = 6144-row tiles) ----
parts = rng.integers(0, 1 << 16, 40)
def spread(n):
    return (U(parts[rng.integers(0, len(parts), n)]) << U(48)) | rng.integers(0, 1 << 12, n, dtype=U)
for nl, nr in ((6143, 6145), (6144, 6144), (6145, 6143)):
    CASE = f'tile edges nl={nl} nr={nr}'
    check(cols(spread(nl), 'i64'), cols(spread(nr), 'i64'), ('inner_join', 'left_join'), 1)

# ---- radix_join_applicable: nulls and wide keys take the hash table, a mask without nulls and 1-row sides do not ----
CASE = 'nulls'
a, c = rng.integers(0, 20_000, 3000), rng.integers(0, 20_000, 2000)
check([(a, rng.random(3000) < 0.8)], [(c, rng.random(2000) < 0.9)], ALL, 0)
CASE = 'mask without nulls'
check([(a, np.ones(3000, bool))], [(c, np.ones(2000, bool))], ALL, 1)
CASE = '16-byte keys'
check([(a, None), (a * 7, None)], [(c, None), (c * 7, None)], ALL, 0)
CASE = 'one row each'
check([(np.array([5]), None)], [(np.array([5]), None)], ALL, 1)
check([(np.array([5]), None)], [(np.array([6]), None)], ALL, 1)
CASE = 'one row against many'
v, cnt = np.unique(a, return_counts=True)
once = np.array([v[cnt == 1][0]])   # a left join of one probe row guesses one pair
check([(once, None)], [(a, None)], ALL, 1)
check([(a, None)], [(once, None)], ALL, 1)
print('RADIX_JOIN_CASES_OK')
"""

# several portions per partition pass: per-portion tile counters and digit bases of radix_partition_top16_mix. Run with
# B2_SORT_PORTION set to a few 6144-row tiles (read once per process).
PORTIONS = r"""
parts = rng.integers(0, 1 << 16, 40)
def spread(n):
    return (U(parts[rng.integers(0, len(parts), n)]) << U(48)) | rng.integers(0, 1 << 14, n, dtype=U)
for nl, nr in ((50_000, 43_007), (18_432, 18_433)):
    CASE = f'portions nl={nl} nr={nr}'
    for form in ('i64', 'i32x2'):
        check(cols(spread(nl), form), cols(spread(nr), form), ('inner_join', 'left_join'), 1)
print('RADIX_JOIN_PORTIONS_OK')
"""

CODE = HELPERS + CASES
PORTION_CODE = HELPERS + PORTIONS

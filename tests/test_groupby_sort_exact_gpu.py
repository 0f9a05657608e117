"""The sort-based groupby (groupby_aggregate_sorted, cudf_b200/csrc/groupby.cu) against exact references written here.

MEDIAN is the reference's group_quantiles(..., {0.5}, LINEAR) (cpp/src/groupby/sort/aggregate.cpp:376-394): the group's valid
values ranked ascending (stable, -0 == +0, NaN last), a and b the values at floor and ceil of (m - 1) / 2, f the fraction
between them, and the result (1 - f) * double(a) + f * double(b) (cpp/src/quantiles/quantiles_util.hpp:23-36,73-89). f is 0
or 0.5, so both products are exact unless they halve a subnormal, and the kernel rounds each product on its own: the expected
value is that expression in float64, compared bit for bit (NaN equals NaN). The formula has consequences that are part of the
result: an odd count whose middle value is +-inf gives NaN (1 * inf + 0 * inf), {-inf, 5} gives -inf, {-1.5e308, 1.5e308} gives 0.

M2 / VARIANCE / STD take two passes on the sort path, as in the reference (group_m2.cu:34-58, group_std.cu:19-52): the group
MEAN, then (x - mean)^2 per valid row (divided by n - ddof for VARIANCE), summed per group; STD is the square root of VARIANCE.
They are held to that algorithm's bound (exact_ref.two_pass_bounds) on every way into the sort path, and those ways agree bit for
bit. The hash path keeps the one-pass formula sumsq - sum^2 / n (cpp/src/groupby/common/m2_var_std.cu), as the reference's does.
"""
import math
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from tests import exact_ref as X
from tests.impls import PlcImpl

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
FLOATS = [np.float32, np.float64]
SIZES = [1, 2, 3, 4, 31, 32, 33, 3000]
DMAX = float(np.finfo(np.float64).max)
SUB = 5e-324  # the smallest float64 subnormal
MOMENTS = ["m2", "var0", "var", "var2", "std0", "std", "std2"]
DDOF = {"var0": 0, "var": 1, "var2": 2, "std0": 0, "std": 1, "std2": 2}


# ---- calls ----------------------------------------------------------------------------------------------------------
def column(plc, v, m=None, off=0):
    """The values as a view starting at row `off` of a longer column (unaligned data, mask read at a bit offset)."""
    if not off:
        return plc.Column.from_numpy(v, m)
    pv = np.concatenate([np.zeros(off, v.dtype), v])
    pm = None if m is None else np.concatenate([np.ones(off, bool), m])
    return plc.Column.from_numpy(pv, pm).slice(off, off + len(v))


def run(plc, keys, kmask, vals, vmask, kinds, off=0, include_nulls=False, keys_sorted=False):
    """One groupby aggregate -> {key (None for the null key): {kind: (value, valid)}}."""
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_numpy(keys, kmask)]), plc.NullPolicy.INCLUDE if include_nulls else plc.NullPolicy.EXCLUDE,
                             plc.Sorted.YES if keys_sorted else plc.Sorted.NO)
    impl = PlcImpl(plc)
    k, res = gb.aggregate([plc.groupby.GroupByRequest(column(plc, vals, vmask, off), [impl._agg(x) for x in kinds])])
    kv, km = k.columns()[0].to_numpy()
    cols = [c.to_numpy() for c in res[0].columns()]
    out = {}
    for g in range(len(kv)):
        key = None if (km is not None and not km[g]) else int(kv[g])
        assert key not in out, f"group {key} returned twice"
        out[key] = {kind: (float(v[g]), True if m is None else bool(m[g])) for kind, (v, m) in zip(kinds, cols)}
    return out


_WORKER = r"""
import os, pickle, sys
sys.path.insert(0, '.')
import torch
if os.environ.get('B2_EMU_RUN') == '1' and not torch.cuda.is_available():
    from tests.emu.harness import install
    install()
import cudf_b200.pylibcudf as plc
from tests.test_groupby_sort_exact_gpu import run
with open(sys.argv[1], 'rb') as f:
    jobs = pickle.load(f)
with open(sys.argv[2], 'wb') as f:
    pickle.dump([run(plc, *job) for job in jobs], f)
print('WORKER_OK')
"""


def run_forced_sort(jobs):
    """`run` over jobs in a fresh process with B2_GROUPBY_SORT=1, which sends every groupby down the sort path (read per call,
    but kept out of this process so that no other test sees it)."""
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.pkl"), os.path.join(d, "out.pkl")
        with open(src, "wb") as f:
            pickle.dump(jobs, f)
        r = subprocess.run([sys.executable, "-c", _WORKER, src, dst], capture_output=True, text=True,
                           env=dict(os.environ, B2_GROUPBY_SORT="1"), cwd=ROOT, timeout=1800)
        assert "WORKER_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
        with open(dst, "rb") as f:
            return pickle.load(f)


# ---- inputs ---------------------------------------------------------------------------------------------------------
def assemble(rng, groups, dt, shuffle=True):
    """groups: [(values, valid | None)] -> (int64 keys, values, valid | None, key of each group); rows shuffled so that the sort
    has to bring each group together (a group's rows keep their relative order, which the ranking's ties depend on)."""
    keys = np.concatenate([np.full(len(v), g * 7919 - 1_000_000, np.int64) for g, (v, _) in enumerate(groups)])
    vals = np.concatenate([np.asarray(v, dt) for v, _ in groups])
    valid = np.concatenate([np.ones(len(v), bool) if m is None else np.asarray(m, bool) for v, m in groups])
    if shuffle:
        p = rng.permutation(len(keys))
        keys, vals, valid = keys[p], vals[p], valid[p]
    return keys, vals, (None if valid.all() else valid), [g * 7919 - 1_000_000 for g in range(len(groups))]


def group_rows(keys, kmask, key):
    """Rows of one group in row order; key None is the null-key group."""
    if key is None:
        return np.nonzero(~kmask)[0]
    sel = keys == key
    if kmask is not None:
        sel &= kmask
    return np.nonzero(sel)[0]


# ---- MEDIAN ---------------------------------------------------------------------------------------------------------
def ref_median(vals):
    """The reference's MEDIAN of one group's valid values (numpy array of the value type); None for no values."""
    if len(vals) == 0:
        return None
    r = sorted(vals.tolist(), key=lambda a: (a != a, 0 if a != a else a))  # stable; -0 == +0; NaN last
    m = len(r)
    lo, hi = (m - 1) // 2, m // 2
    f = 0.0 if lo == hi else 0.5
    a, b = float(r[lo]), float(r[hi])  # integers round to nearest even, as the device's conversion to double does
    return (1.0 - f) * a + f * b


def same_bits(got, exp):
    g, e = np.float64(got), np.float64(exp)
    return bool(np.isnan(g) and np.isnan(e)) or g.view(np.uint64) == e.view(np.uint64)


def special_groups(dt):
    """Groups whose MEDIAN a formula other than the reference's gets wrong, or where the conversion to double rounds."""
    dt = np.dtype(dt)
    if dt == np.int64:
        t62, t63 = 2 ** 62, 2 ** 63
        return [[t62 + 1, t62 + 513], [t62 - 1, t62 + 1025], [-t62 - 1, -t62 + 511], [t63 - 1, t63 - 1], [t63 - 1], [-t63, -t63 + 1],
                [-t63, t63 - 1], [t63 - 1, t63 - 512, t63 - 1025], [-t63, -t63, 5], [t63 - 1, t63 - 2, 0, -t63]]
    if dt == np.uint64:
        t63 = 2 ** 63
        return [[t63 + 2048], [t63 + 2048, t63 + 2048], [t63 + 2048, 2 ** 64 - 1], [0, 2 ** 64 - 1], [t63, t63 + 1], [1, t63 + 4096, 2 ** 64 - 1],
                [t63 - 1, t63, t63 + 1, 2 ** 64 - 2049]]
    if dt.kind in "iu":
        lo, hi = int(np.iinfo(dt).min), int(np.iinfo(dt).max)
        return [[lo, hi], [hi, hi], [lo, lo], [lo, lo + 1, hi], [hi - 1, hi]]
    inf, nan = math.inf, math.nan
    big = DMAX if dt == np.float64 else float(np.finfo(np.float32).max)
    one_up = float(np.nextafter(np.float32(1), np.float32(2))) if dt == np.float32 else float(np.nextafter(1.0, 2.0))
    g = [[inf], [-inf], [inf, inf], [-inf, -inf], [-inf, inf], [-inf, 5.0], [5.0, inf], [1.0, inf, inf], [-inf, 0.0, inf], [-inf, -inf, 2.0],
         [nan], [nan, nan], [1.0, nan], [1.0, 2.0, nan], [1.0, nan, nan], [1.0, 2.0, nan, nan], [1.0, 2.0, 3.0, nan], [-inf, nan], [inf, nan],
         [-0.0], [-0.0, -0.0], [0.0, -0.0], [-0.0, 0.0], [0.0, -0.0, 0.0], [-0.0, 0.0, -0.0], [-0.0, 0.0, 0.0, -0.0],
         [-big * 0.8, big * 0.8], [big, big], [-big, big], [-big, -big], [big, -big, 1.0], [big * 0.8, big * 0.9], [-big, -big * 0.9],
         [1.0, one_up], [one_up, 1.0, 1.0, one_up], [-one_up, -1.0]]
    if dt == np.float64:
        g += [[-1.5e308, 1.5e308], [1.049001171530397, 6.40422650443282],
              [SUB], [SUB, SUB], [SUB, 3 * SUB], [-SUB, SUB], [3 * SUB, 5 * SUB], [-3 * SUB, SUB], [-SUB, -SUB], [7 * SUB, 9 * SUB, 0.0, 1 * SUB]]
    else:
        s32 = float(np.finfo(np.float32).smallest_subnormal)
        g += [[s32], [s32, 3 * s32], [-s32, s32], [1.0000001, 1.0000002]]
    return g


def random_values(rng, dt, n, ties=False):
    dt = np.dtype(dt)
    if ties:
        return rng.integers(-3, 4, n).astype(dt) if dt.kind != "u" else rng.integers(0, 4, n).astype(dt)
    if dt.kind in "iu":
        return rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
    return (rng.standard_normal(n) * 10).astype(dt)


def median_groups(rng, dt):
    groups = []
    for s in SIZES:
        groups.append((random_values(rng, dt, s), None))
        if s <= 33:
            groups.append((random_values(rng, dt, s, ties=True), None))
        if s >= 3:  # nulls inside the group; the median is over the valid values only
            groups.append((random_values(rng, dt, s), rng.random(s) >= 0.2))
    groups.append((random_values(rng, dt, 5), np.zeros(5, bool)))        # all null: a null result, valid results around it
    groups.append((random_values(rng, dt, 4), [False, True, False, True]))
    groups += [(np.array(v, dtype=object).astype(dt) if np.dtype(dt).kind in "iu" else np.array(v, dt), None) for v in special_groups(dt)]
    # enough groups for gb_median_kernel to run on more than one 256-thread CTA
    groups += [(random_values(rng, dt, int(s)), None) for s in rng.integers(1, 12, 300)]
    return groups


def check_median(res, keys, kmask, vals, vmask, what):
    for key, r in res.items():
        rows = group_rows(keys, kmask, key)
        v = vals[rows] if vmask is None else vals[rows][vmask[rows]]
        got, ok = r["median"]
        exp = ref_median(v)
        w = f"{what} key={key} values={v[:8].tolist()}{'...' if len(v) > 8 else ''}"
        assert ok == (exp is not None), f"{w}: valid {ok}"
        if exp is not None:
            assert same_bits(got, exp), f"{w}: got {got!r}, expected {exp!r}"


@pytest.mark.parametrize("dt", INTS + FLOATS, ids=lambda d: np.dtype(d).name)
def test_median_bit_exact(plc, dt):
    rng = np.random.default_rng(200 + np.dtype(dt).num)
    keys, vals, vmask, gkeys = assemble(rng, median_groups(rng, dt), dt)
    for off in (0, 45):  # 45: a view whose data is unaligned and whose mask starts at a bit offset that is not a multiple of 32
        res = run(plc, keys, None, vals, vmask, ["median", "count"], off)
        assert sorted(res) == sorted(gkeys)
        check_median(res, keys, None, vals, vmask, f"{np.dtype(dt)} off={off}")


@pytest.mark.parametrize("dt", [np.int32, np.uint64, np.float64])
def test_median_nullable_keys(plc, dt):
    """Null keys form one group under INCLUDE and are dropped under EXCLUDE; values may be null too."""
    rng = np.random.default_rng(230)
    n = 2000
    keys = rng.integers(0, 40, n).astype(np.int64)
    kmask = rng.random(n) >= 0.1
    vals = random_values(rng, dt, n)
    if np.dtype(dt).kind == "f":
        vals[rng.random(n) < 0.05] = np.nan
        vals[rng.random(n) < 0.02] = np.inf
    vmask = rng.random(n) >= 0.15
    vmask[keys == 7] = False  # a group with no valid value
    for inc in (False, True):
        for off in (0, 3):
            res = run(plc, keys, kmask, vals, vmask, ["median"], off, include_nulls=inc)
            assert (None in res) == inc
            assert len(res) == len(np.unique(keys[kmask])) + inc
            check_median(res, keys, kmask, vals, vmask, f"{np.dtype(dt)} include_nulls={inc} off={off}")


# ---- M2 / VARIANCE / STD ----------------------------------------------------------------------------------------------
def moment_cases():
    """(name, keys, values, valid | None, expect every group finite). Integer values stay where the reference's INT64 SUM
    (its sort path's MEAN) cannot wrap: 2000 values near 2^40 sum below 2^51."""
    rng = np.random.default_rng(240)
    cases = []

    def add(name, groups, dt):
        keys, vals, valid, _ = assemble(rng, groups, dt)
        cases.append((name, keys, vals, valid))

    small = [(1, None), (2, None), (3, None), (33, None)]
    add("f64-1e8-normal", [(1e8 + rng.standard_normal(s), m) for s, m in [(3000, None), (500, None)] + small], np.float64)
    add("f64-1e15-ints", [(1e15 + rng.integers(-5, 6, s), m) for s, m in [(700, None), (40, None)] + small], np.float64)
    add("f32-1e4", [((1e4 + rng.standard_normal(s)).astype(np.float32), None) for s in (2500, 64, 1, 2, 3)], np.float32)
    add("i64-2^40", [(2 ** 40 + rng.integers(-3, 4, s), None) for s in (2000, 32, 33, 1, 2, 3)], np.int64)
    add("u64-2^40", [(2 ** 40 + rng.integers(0, 7, s), None) for s in (1500, 5, 1, 2)], np.uint64)
    add("i32-small", [(rng.integers(-50, 50, s), None) for s in (31, 32, 1, 2, 700)], np.int32)
    # nulls: a random mask, a group with one valid value, a group with two, a group with none
    add("f64-nulls", [(1e8 + rng.standard_normal(s), rng.random(s) >= 0.2) for s in (2000, 40, 9)]
        + [(1e8 + rng.standard_normal(4), [False, True, False, False]), (1e8 + rng.standard_normal(5), [True, False, False, True, False]),
           (rng.standard_normal(6), np.zeros(6, bool))], np.float64)
    # non-finite values: x - mean is NaN for every row of such a group
    add("f64-nonfinite", [(np.array([1.0, np.inf, 2.0]), None), (np.array([np.nan, 1.0]), None), (np.array([-np.inf, np.inf]), None),
                          (np.array([np.inf]), None), (np.array([3.0, -np.inf, 4.0, 5.0]), [True, True, False, True]),
                          (np.array([1.0, np.nan, 2.0]), [True, False, True]), (rng.standard_normal(40), None)], np.float64)
    return cases


def check_two_pass(res, keys, vals, vmask, what):
    u = X.U64
    for key, r in res.items():
        rows = group_rows(keys, None, key)
        valid = np.ones(len(rows), bool) if vmask is None else vmask[rows]
        xv = vals[rows][valid].astype(np.float64)  # exact: float32 widens, integers here are below 2^53
        n, L = len(xv), len(rows)
        w = f"{what} key={key} n={n}"
        m2, m2_ok = r["m2"]
        assert m2_ok, f"{w}: M2 has no nulls"
        if n == 0:
            assert m2 == 0.0, w
            assert not any(r[k][1] for k in MOMENTS[1:]), w
            continue
        if not np.isfinite(xv).all():
            assert math.isnan(m2), f"{w}: M2 {m2!r}"
            for kind, ddof in DDOF.items():
                v, ok = r[kind]
                assert ok == (n > ddof), f"{w} {kind}"
                if ok:
                    assert math.isnan(v), f"{w} {kind}: {v!r}"
            continue
        k = X.k_segmented(L)
        delta = X.mean_bound(k + 1, u, X.abs_sum(xv), X.exact_sum(xv), n, u)
        X.check(m2, *X.two_pass_bounds(k, xv, delta, 0)[:2], "m2 " + w)
        assert m2 >= 0, f"{w}: M2 {m2!r}"
        for kind, ddof in DDOF.items():
            v, ok = r[kind]
            _, _, var, bv, std, bs = X.two_pass_bounds(k, xv, delta, ddof)
            assert ok == (var is not None), f"{w} {kind}: valid {ok}"
            if not ok:
                continue
            assert v >= 0 and not math.isnan(v), f"{w} {kind}: {v!r}"
            if kind.startswith("var"):
                X.check(v, var, bv, f"{kind} {w}")
            else:
                X.check(v, std, bs, f"{kind} {w}")


@pytest.fixture(scope="module")
def moment_results(plc):
    """Every case down every way into the sort path, and once down the hash path:
    'median' - the moments requested next to MEDIAN (which only the sort path has);
    'sorted' - keys declared sorted (Sorted.YES), rows given in key order;
    'forced' - B2_GROUPBY_SORT=1 in a separate process;
    'hash'   - the moments alone, which the hash path serves."""
    out = {}
    jobs = []
    for name, keys, vals, valid in moment_cases():
        out[(name, "median")] = run(plc, keys, None, vals, valid, MOMENTS + ["median"])
        o = np.argsort(keys, kind="stable")  # a group's rows keep their order: every route sums the same terms in the same order
        out[(name, "sorted")] = run(plc, keys[o], None, vals[o], None if valid is None else valid[o], MOMENTS, keys_sorted=True)
        out[(name, "hash")] = run(plc, keys, None, vals, valid, MOMENTS)
        jobs.append((keys, None, vals, valid, MOMENTS))
    for (name, *_), r in zip(moment_cases(), run_forced_sort(jobs)):
        out[(name, "forced")] = r
    return out


@pytest.mark.parametrize("name", [c[0] for c in moment_cases()])
def test_moments_two_pass_bound(moment_results, name):
    case = {c[0]: c for c in moment_cases()}[name]
    _, keys, vals, valid = case
    check_two_pass(moment_results[(name, "median")], keys, vals, valid, name)


@pytest.mark.parametrize("name", [c[0] for c in moment_cases()])
def test_moments_agree_across_sort_routes(moment_results, name):
    base = moment_results[(name, "median")]
    for route in ("sorted", "forced"):
        other = moment_results[(name, route)]
        assert sorted(other) == sorted(base), route
        for key in base:
            for kind in MOMENTS:
                (a, aok), (b, bok) = base[key][kind], other[key][kind]
                assert aok == bok and (not aok or same_bits(a, b)), f"{name} {route} key={key} {kind}: {b!r} vs {a!r} next to MEDIAN"


def test_moments_hash_path_keeps_the_one_pass_formula(moment_results):
    """Without MEDIAN / NUNIQUE / NTH_ELEMENT and with unsorted keys the hash path runs, and it computes sumsq - sum^2 / n as
    the reference's hash path does: held to that formula's bound, which the large-mean groups need. Float values only: for
    integers the reference squares and sums in INT64, which wraps near 2^40 (the one-pass oracle pins that elsewhere)."""
    for name, keys, vals, valid in moment_cases():
        if vals.dtype.kind != "f":
            continue
        res = moment_results[(name, "hash")]
        for key, r in res.items():
            rows = group_rows(keys, None, key)
            xv = vals[rows] if valid is None else vals[rows][valid[rows]]
            xv = xv.astype(np.float64)
            if not len(xv) or not np.isfinite(xv).all():
                continue
            X.check(r["m2"][0], X.exact_m2(xv), X.m2_bound(X.k_hash_group(len(xv)), xv), f"hash {name} key={key}")

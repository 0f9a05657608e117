"""Randomised differential test of the kernels against the oracle, on the CPU emulator (tests/emu).

  python scripts/emu_fuzz.py [--seconds 120] [--seed 0]

Small random tables (sizes around tile / warp / word boundaries, sliced views with odd offsets, nulls, NaN / -0, wide
and multi-column keys, every join kind and aggregation) through sort, join, groupby, scan / reduce / segmented reduce,
segmented sort, rank and top-k. A development aid, not part of the test suite (it never touches a GPU)."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.chdir(ROOT)

# --mode selects an opt-in path for the whole run (the switches are read by the library, some of them only once)
_MODES = {"default": {}, "carry": {"B2_SORT_CARRY": "1"}, "radix": {"B2_JOIN_RADIX_ROWS": "1"}, "portion": {"B2_SORT_PORTION": "6144"},
          "pgb": {"B2_GROUPBY_PARTITION_ROWS": "1", "B2_GROUPBY_EST": "1", "B2_GROUPBY_EST_MIN": "1"},
          "pgbcap": {"B2_GROUPBY_PARTITION_ROWS": "1", "B2_GROUPBY_EST": "1", "B2_GROUPBY_EST_MIN": "1", "B2_GROUPBY_EST_CAP": "48"},
          "pgbhist": {"B2_GROUPBY_PARTITION_ROWS": "1", "B2_GROUPBY_EST": "0"},
          "fix0": {"B2_SORT_HYBRID_MIN": "0", "B2_SORT_FIX_FAST": "0"}, "fix1": {"B2_SORT_HYBRID_MIN": "0", "B2_SORT_FIX_FAST": "1"}}
for _i, _a in enumerate(sys.argv):
    if _a == "--mode" and _i + 1 < len(sys.argv):
        os.environ.update(_MODES[sys.argv[_i + 1]])

from tests.emu.harness import install  # noqa: E402

install()
import numpy as np  # noqa: E402

import cudf_b200.pylibcudf as plc  # noqa: E402
from oracle import sort as osort  # noqa: E402
from tests.helpers import assert_columns_equal  # noqa: E402
from tests.impls import OracleImpl, PlcImpl, sort_groups  # noqa: E402

cu, o = PlcImpl(plc), OracleImpl()
DTYPES = [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.int64, np.uint64, np.float32, np.float64, np.bool_]
SIZES = [0, 1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1000, 2047, 2048, 2049, 4095, 4096, 4097, 6143, 6144, 6145, 12289, 20011]


def rnd_col(rng, n, dtype, null_frac, card):
    if dtype == np.bool_:
        v = rng.random(n) < 0.5
    elif np.dtype(dtype).kind == "f":
        v = rng.integers(-card, card, n).astype(dtype) / 2
        if n:
            v[rng.random(n) < 0.03] = np.nan
            v[rng.random(n) < 0.03] = -0.0
            v[rng.random(n) < 0.01] = np.inf
    else:
        info = np.iinfo(dtype)
        lo, hi = max(info.min, -card), min(info.max, card)
        v = rng.integers(lo, hi + 1, n).astype(dtype)
        if n and rng.random() < 0.2:
            v[rng.random(n) < 0.05] = info.max
            v[rng.random(n) < 0.05] = info.min
    m = None
    if null_frac > 0:
        m = rng.random(n) >= null_frac
    return v, m


def sliced(rng, col):
    """the same column as a view into a larger buffer with a random offset (bit offsets not multiple of 32)"""
    v, m = col
    pre, post = int(rng.integers(0, 70)), int(rng.integers(0, 40))
    big = np.concatenate([np.zeros(pre, v.dtype), v, np.zeros(post, v.dtype)])
    bm = None if m is None else np.concatenate([np.ones(pre, bool), m, np.ones(post, bool)])
    c = plc.Column.from_numpy(big, bm)
    return c.slice(pre, pre + len(v))


def fuzz_sort(rng):
    n = int(rng.choice(SIZES))
    ncol = int(rng.integers(1, 4))
    cols = [rnd_col(rng, n, DTYPES[rng.integers(len(DTYPES))], float(rng.choice([0, 0, 0.1, 0.6])), int(rng.choice([3, 50, 10**6]))) for _ in range(ncol)]
    order = [int(rng.integers(2)) for _ in range(ncol)]
    prec = [int(rng.integers(2)) for _ in range(ncol)]
    use_slices = rng.random() < 0.5
    pc = [sliced(rng, c) if use_slices else plc.Column.from_numpy(*c) for c in cols]
    got = plc.sorting.sorted_order(plc.Table(pc), order, prec).to_numpy()[0]
    exp = osort.sorted_order(cols, order, prec)
    if ncol == 1:  # the unstable API may order ties freely only for the comparator path; the LSD sort is stable
        assert np.array_equal(got, exp), ("sorted_order", n, [c[0].dtype for c in cols], order, prec, use_slices)
    else:
        assert np.array_equal(got, exp), ("sorted_order multi", n, [c[0].dtype for c in cols], order, prec, use_slices)
    vdt = [np.int32, np.int64, np.float64][int(rng.integers(3))]
    vals = (rng.integers(0, 1 << 30, n).astype(vdt), None)
    g = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(*vals)]), plc.Table(pc), order, prec).columns()[0].to_numpy()[0]
    assert np.array_equal(g, vals[0][exp]), ("sort_by_key", n, vdt)
    if ncol == 1:
        t = plc.Table([pc[0]])
        g, gm = plc.sorting.sort_by_key(t, t, order, prec).columns()[0].to_numpy()       # aliased values = keys
        e, em = osort.sort_by_key([cols[0]], [cols[0]], order, prec)[0]
        ok = np.ones(n, bool) if em is None else np.asarray(em, bool)
        assert np.array_equal(np.asarray(g)[ok].view(np.uint8), np.asarray(e)[ok].view(np.uint8)), ("aliased sort_by_key", n, cols[0][0].dtype)
        g, gm = plc.sorting.sort(t, order, prec).columns()[0].to_numpy()
        assert np.array_equal(np.asarray(g)[ok].view(np.uint8), np.asarray(e)[ok].view(np.uint8)), ("sort", n, cols[0][0].dtype)


def fuzz_join(rng):
    nl, nr = int(rng.choice(SIZES[:20])), int(rng.choice(SIZES[:20]))
    ncol = int(rng.integers(1, 4))
    dts = [DTYPES[rng.integers(len(DTYPES))] for _ in range(ncol)]
    card = int(rng.choice([2, 20, 300]))
    nf = float(rng.choice([0, 0, 0.2]))
    l = [rnd_col(rng, nl, d, nf, card) for d in dts]
    r = [rnd_col(rng, nr, d, nf, card) for d in dts]
    for kind in ("inner_join", "left_join", "full_join"):
        for ne in (0, 1):
            exp = getattr(o, kind)(l, r, ne)
            if len(exp[0]) > 3_000_000:
                continue
            got = getattr(cu, kind)(l, r, ne)
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (kind, ne, nl, nr, dts, card, nf)
    if nl and nr:
        bounds = sorted(rng.integers(0, nl + 1, 2).tolist())
        for kind in ("inner", "left", "full"):
            exp = getattr(o, f"{kind}_join")(l, r, 0)
            if len(exp[0]) <= 3_000_000:
                got = cu.partitioned_join(l, r, 0, kind, bounds)
                assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), ("partitioned", kind, nl, nr, dts)


def fuzz_groupby(rng):
    n = int(rng.choice(SIZES))
    nk = int(rng.integers(1, 3))
    kd = [DTYPES[rng.integers(len(DTYPES))] for _ in range(nk)]
    keys = [rnd_col(rng, n, d, float(rng.choice([0, 0.1])), int(rng.choice([2, 40, 5000]))) for d in kd]
    vd = DTYPES[rng.integers(len(DTYPES) - 1)]
    vals = rnd_col(rng, n, vd, float(rng.choice([0, 0.3])), 200)
    if np.dtype(vd).kind == "f" and n:
        vals = (np.nan_to_num(vals[0], nan=1.0, posinf=2.0), vals[1])
    kinds = ["sum", "min", "max", "count", "count_all", "mean", "sum_of_squares", "var", "std0", "m2", "argmin", "argmax"]
    if np.dtype(vd).kind != "f":
        kinds.append("product")  # float products depend on the multiplication order
    inc = bool(rng.integers(2))
    gk, gr = sort_groups(*cu.groupby(keys, [(vals, kinds)], include_nulls=inc))
    ek, er = sort_groups(*o.groupby(keys, [(vals, kinds)], include_nulls=inc))
    for a, b in zip(gk, ek):
        assert_columns_equal(a, b, what="keys")
    for j, kind in enumerate(kinds):
        g, e = gr[0][j], er[0][j]
        assert np.asarray(g[0]).dtype == np.asarray(e[0]).dtype, (kind, vd)
        gm = np.ones(len(g[0]), bool) if g[1] is None else np.asarray(g[1], bool)
        em = np.ones(len(e[0]), bool) if e[1] is None else np.asarray(e[1], bool)
        assert np.array_equal(gm, em), (kind, vd, kd, n)
        if np.asarray(e[0]).dtype.kind == "f":
            np.testing.assert_allclose(np.asarray(g[0], np.float64)[em], np.asarray(e[0], np.float64)[em], rtol=2e-4, atol=1e-2,
                                       err_msg=str((kind, vd, kd, n)))
        else:
            assert np.array_equal(np.asarray(g[0])[em], np.asarray(e[0])[em]), (kind, vd, kd, n)


def fuzz_reduce_scan(rng):
    n = int(rng.choice(SIZES))
    dt = DTYPES[rng.integers(len(DTYPES) - 1)]
    col = rnd_col(rng, n, dt, float(rng.choice([0, 0.2, 1.0])), 100)
    if np.dtype(dt).kind == "f" and n:
        col = (np.nan_to_num(col[0], nan=1.0, posinf=2.0), col[1])
    for kind in ("sum", "min", "max"):
        for inclusive in (True, False):
            for include in (False, True):
                g, e = cu.scan(col, kind, inclusive, include), o.scan(col, kind, inclusive, include)
                assert_columns_equal(g, e, rtol=1e-6 if np.dtype(dt).kind == "f" else 0.0, what=f"scan {kind} {dt} n={n}")
    if n:
        nseg = int(rng.integers(1, 40))
        offs = np.sort(rng.integers(0, n + 1, nseg + 1)).astype(np.int32)
        odt = np.float64 if np.dtype(dt).kind == "f" else np.int64
        for kind in ("sum", "min", "max"):
            od = odt if kind == "sum" else dt
            g, e = cu.segmented_reduce(col, offs, kind, od), o.segmented_reduce(col, offs, kind, od)
            assert_columns_equal(g, e, rtol=1e-6 if np.dtype(dt).kind == "f" else 0.0, what=f"segmented {kind} {dt} n={n}")


def fuzz_seg_rank(rng):
    n = int(rng.choice(SIZES[:18]))
    dt = DTYPES[rng.integers(len(DTYPES) - 1)]
    col = rnd_col(rng, n, dt, float(rng.choice([0, 0.2])), int(rng.choice([3, 100])))
    if n:
        offs = np.sort(rng.integers(0, n + 1, int(rng.integers(0, 12)))).astype(np.int32)
        keys = [col, (np.arange(n, dtype=np.int32), None)]
    if n:
        order0 = int(rng.integers(2))
        exp = osort.segmented_sorted_order(keys, offs, [order0, 0], None)
        got = plc.sorting.segmented_sorted_order(plc.Table([plc.Column.from_numpy(*c) for c in keys]), plc.Column.from_numpy(offs), [order0, 0],
                                                 []).to_numpy()[0]
        assert np.array_equal(got, exp), ("segmented_sorted_order", n, dt, order0, offs.tolist())
        # top-k: any k rows whose multiset of values equals the oracle's
        k = int(rng.integers(0, n + 3))
        tk_order = int(rng.integers(2))
        gv, gm = plc.sorting.top_k(plc.Column.from_numpy(*col), k, tk_order).to_numpy()
        ev, em = osort.top_k(col, k, tk_order)
        canon = lambda v, m: sorted((bool(a), (float(b) if b == b else float("inf")) if a else 0.0)
                                    for a, b in zip(np.ones(len(v), bool) if m is None else np.asarray(m, bool), np.asarray(v, np.float64)))
        assert canon(gv, gm) == canon(ev, em), ("top_k", n, dt, k, tk_order)
        # cudf::partition through the pylibcudf twin: stable partition by an explicit map
        P = int(rng.integers(1, 40))
        pmap = rng.integers(0, P, n).astype(np.int32)
        out, poffs = plc.partitioning.partition(plc.Table([plc.Column.from_numpy(np.arange(n, dtype=np.int64))]), plc.Column.from_numpy(pmap), P)
        assert np.array_equal(out.columns()[0].to_numpy()[0], np.argsort(pmap, kind="stable")), ("partition", n, P)
        assert poffs == np.concatenate([[0], np.cumsum(np.bincount(pmap, minlength=P))]).tolist()  # P + 1 offsets (partitioning.hpp:58-101)
    for method in range(5):
        order, policy, nprec = int(rng.integers(2)), int(rng.integers(2)), int(rng.integers(2))
        pct = bool(rng.integers(2))
        g = plc.sorting.rank(plc.Column.from_numpy(*col), method, order, policy, nprec, pct).to_numpy()
        e = osort.rank(col, method, order, policy, nprec, pct)
        em = np.ones(n, bool) if e[1] is None else np.asarray(e[1], bool)
        np.testing.assert_allclose(np.asarray(g[0], np.float64)[em], np.asarray(e[0], np.float64)[em], rtol=1e-12,
                                   err_msg=str(("rank", method, dt, n, order, policy, nprec, pct)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--mode", default="default", choices=sorted(_MODES))
    ap.add_argument("--only", default="", help="comma-separated subset of: sort,join,groupby,reduce_scan,seg_rank")
    a = ap.parse_args()
    rng = np.random.default_rng(a.seed)
    fns = [fuzz_sort, fuzz_join, fuzz_groupby, fuzz_reduce_scan, fuzz_seg_rank]
    if a.only:
        fns = [f for f in fns if f.__name__[5:] in a.only.split(",")]
    counts = {f.__name__: 0 for f in fns}
    t0 = time.time()
    it = 0
    while time.time() - t0 < a.seconds:
        f = fns[it % len(fns)]
        state = rng.bit_generator.state
        try:
            f(rng)
        except Exception:
            print(f"FAILED in {f.__name__} at iteration {it} (seed {a.seed}); generator state: {state['state']}", flush=True)
            raise
        counts[f.__name__] += 1
        it += 1
    print("FUZZ_OK", counts, flush=True)


if __name__ == "__main__":
    main()

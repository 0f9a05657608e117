"""Floating-point accuracy of reduce, scan, segmented_reduce, the groupby aggregations (hash, partitioned and sort-based paths)
and the grouped scan: each result is checked against an exact reference within a bound derived from the kernel
(tests/exact_ref.py), on the inputs where summation goes wrong: cancellation, wide dynamic range, subnormals, overflow, NaN
and +-inf, tile-boundary sizes and sliced views (unaligned addresses, bit offsets that are not a multiple of 32).

MIN / MAX rank NaN above +inf whatever its sign: MIN is NaN only when every valid value is NaN, MAX as soon as one is,
ARGMIN / ARGMAX pick the first row holding that value, and -0.0 ties with +0.0 (either sign is accepted where they tie)."""
import math
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from oracle import groupby as ogb
from oracle import reduce as ored
from tests import exact_ref as X
from tests.impls import KINDS, PlcImpl

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLOATS = [np.float32, np.float64]
OFFSETS = [0, 1, 3, 7, 45]  # 45: a bit offset past the first mask word that is not a multiple of 32


def sms() -> int:
    """SMs of the device the reduce grid is sized for (the kernel emulator reports an H100 SXM's 132)."""
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


# ---- inputs -------------------------------------------------------------------------------------------------------
def gen(rng, kind, n, dt):
    dt = np.dtype(dt)
    if kind == "normal":
        x = rng.standard_normal(n) * 10
    elif kind == "cancel":  # x, -x pairs plus small noise: the exact sum is tiny next to sum(|x|)
        h = rng.standard_normal(n // 2 + 1) * 1e3
        x = np.concatenate([h, -h])[:n] + rng.standard_normal(n) * 1e-3
        x = x[rng.permutation(n)]
    elif kind == "wide":
        lo, hi = (-30, 30) if dt == np.float64 else (-6, 6)
        x = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(lo, hi, n)
    elif kind == "subnormal":  # sums of subnormals are exact in any order: the result must be bit-exact
        x = rng.integers(-1000, 1000, n) * float(np.finfo(dt).smallest_subnormal)
    else:
        raise ValueError(kind)
    return x.astype(dt)


def with_specials(rng, x, frac=0.02):
    x = x.copy()
    n = len(x)
    for v in (np.nan, -np.nan, np.inf, -np.inf):
        x[rng.random(n) < frac / 4] = v
    return x


# ---- calls (views at a row offset: same values at an unaligned address and a shifted bit offset) ----------------------
def column(plc, v, m=None, off=0):
    if not off:
        return plc.Column.from_numpy(v, m)
    pv = np.concatenate([np.full(off, 7, v.dtype), v])
    pm = None if m is None else np.concatenate([np.zeros(off, bool), m])
    return plc.Column.from_numpy(pv, pm).slice(off, off + len(v))


def agg(plc, name):
    return PlcImpl(plc)._agg(name)


def reduce_(plc, v, m, kind, od, off=0):
    out = plc.reduce.reduce(column(plc, v, m, off), agg(plc, kind), plc.DataType.from_numpy(od))
    val, ok = out._get()
    assert ok
    return val


def scan_(plc, v, m, kind, inclusive=True, off=0):
    return plc.reduce.scan(column(plc, v, m, off), agg(plc, kind), plc.reduce.ScanType.INCLUSIVE if inclusive else plc.reduce.ScanType.EXCLUSIVE,
                           plc.NullPolicy.EXCLUDE).to_numpy()


def segred_(plc, v, m, offsets, kind, od, off=0):
    o = plc.Column.from_numpy(np.asarray(offsets, np.int32))
    return plc.reduce.segmented_reduce(column(plc, v, m, off), o, agg(plc, kind), plc.DataType.from_numpy(od), plc.NullPolicy.EXCLUDE).to_numpy()


def groupby_(plc, keys, v, m, kinds, off=0):
    """-> (keys ascending, [(values, valid | None)] per kind in that order)."""
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_numpy(keys)]))
    k, res = gb.aggregate([plc.groupby.GroupByRequest(column(plc, v, m, off), [agg(plc, x) for x in kinds])])
    gk = k.columns()[0].to_numpy()[0]
    order = np.argsort(gk, kind="stable")
    return gk[order], [(c.to_numpy()[0][order], None if c.to_numpy()[1] is None else c.to_numpy()[1][order]) for c in res[0].columns()]


def groupby_scan_(plc, keys, v, m, kinds, off=0):
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_numpy(keys)]))
    k, res = gb.scan([plc.groupby.GroupByRequest(column(plc, v, m, off), [agg(plc, x) for x in kinds])])
    return k.columns()[0].to_numpy()[0], [c.to_numpy() for c in res[0].columns()]


_WORKER = r"""
import os, pickle, sys
sys.path.insert(0, '.')
import torch
if os.environ.get('B2_EMU_RUN') == '1' and not torch.cuda.is_available():
    from tests.emu.harness import install
    install()
import cudf_b200.pylibcudf as plc
from tests.test_float_accuracy_gpu import groupby_
with open(sys.argv[1], 'rb') as f:
    jobs = pickle.load(f)
with open(sys.argv[2], 'wb') as f:
    pickle.dump([groupby_(plc, *job) for job in jobs], f)
print('WORKER_OK')
"""


def groupby_in_subprocess(jobs, env_extra):
    """groupby_ over `jobs` in a fresh process with the path-selecting environment (those switches are read once per process)."""
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.pkl"), os.path.join(d, "out.pkl")
        with open(src, "wb") as f:
            pickle.dump(jobs, f)
        r = subprocess.run([sys.executable, "-c", _WORKER, src, dst], capture_output=True, text=True, env=dict(os.environ, **env_extra),
                           cwd=ROOT, timeout=1800)
        assert "WORKER_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
        with open(dst, "rb") as f:
            return pickle.load(f)


# ---- value checks -------------------------------------------------------------------------------------------------
def same_value(got, exp):
    """MIN / MAX results: equal as numbers (-0.0 == +0.0) or both NaN."""
    got, exp = float(got), float(exp)
    return got == exp or (math.isnan(got) and math.isnan(exp))


def check_sum(got, x, k, u, u_out, what):
    sp = X.special_sum(x)
    if sp is not None:
        X.check(got, sp, 0.0, what)
        return
    X.check(got, X.exact_sum(x), X.sum_bound(k, u, X.abs_sum(x), X.exact_sum(x), u_out), what)


def check_mean(got, x, k, u, u_out, what):
    sp = X.special_sum(x)
    if sp is not None:
        X.check(got, sp, 0.0, what)
        return
    s = X.exact_sum(x)
    X.check(got, s / len(x), X.mean_bound(k, u, X.abs_sum(x), s, len(x), u_out), what)


def min_max_exp(x):
    x = np.asarray(x, np.float64)
    return np.fmin.reduce(x), np.maximum.reduce(x)


# ---- the MIN / MAX contract on small known inputs --------------------------------------------------------------------
@pytest.mark.parametrize("dt", FLOATS)
def test_min_max_nan_rule_known_answers(plc, dt):
    nan, inf = np.nan, np.inf
    f = lambda *a: np.array(a, dt)
    assert math.isnan(reduce_(plc, f(nan, nan, nan), None, "min", dt))
    assert math.isnan(reduce_(plc, f(nan, nan, nan), None, "max", dt))
    assert reduce_(plc, f(nan, 2, -inf, nan), None, "min", dt) == -inf
    assert math.isnan(reduce_(plc, f(1, -nan, inf), None, "max", dt))
    assert reduce_(plc, f(inf, -nan), None, "min", dt) == inf
    x = f(nan, 1, 0.5, 2, nan, -1)
    for off in (0, 3):
        got = scan_(plc, x, None, "min", True, off)[0]
        assert np.array_equal(got, f(nan, 1, 0.5, 0.5, 0.5, -1), equal_nan=True), got
        got = scan_(plc, x, None, "max", True, off)[0]
        assert np.isnan(got).all(), got
        got = scan_(plc, x, None, "min", False, off)[0]  # an empty prefix is +inf, the reference's identity
        assert np.array_equal(got, f(inf, nan, 1, 0.5, 0.5, 0.5), equal_nan=True), got
        got = scan_(plc, x, None, "max", False, off)[0]
        assert got[0] == -inf and np.isnan(got[1:]).all(), got
    # leading nulls: the first valid row of an exclusive MIN scan sees an empty prefix
    v, ok = scan_(plc, f(nan, nan, 3, nan), np.array([False, True, True, True]), "min", False)
    assert ok.tolist() == [False, True, True, True] and v[1] == inf and math.isnan(v[2]) and v[3] == 3
    seg_x, seg_o = f(nan, nan, 5, nan, -nan, 2, 1), [0, 2, 4, 7]
    for off in (0, 7):
        mn = segred_(plc, seg_x, None, seg_o, "min", dt, off)[0]
        mx = segred_(plc, seg_x, None, seg_o, "max", dt, off)[0]
        assert math.isnan(mn[0]) and mn[1] == 5 and mn[2] == 1, mn
        assert np.isnan(mx).all(), mx
    keys = np.array([0, 0, 0, 1, 1, 2, 2], np.int32)
    k, ((mn, _), (mx, _)) = groupby_scan_(plc, keys, f(nan, 3, 1, -nan, -nan, 2, nan), None, ["min", "max"])
    assert np.array_equal(mn, f(nan, 3, 1, nan, nan, 2, 2), equal_nan=True), mn
    assert np.array_equal(mx, f(nan, nan, nan, nan, nan, 2, nan), equal_nan=True), mx
    keys = np.array([0, 0, 1, 1, 2, 2, 3, 3], np.int64)
    vals = f(-nan, 1, nan, 1, -0.0, 0.0, nan, -nan)
    k, res = groupby_(plc, keys, vals, None, ["min", "max", "argmin", "argmax"])
    assert np.array_equal(res[0][0], f(1, 1, 0, nan), equal_nan=True) and np.array_equal(res[1][0], f(nan, nan, 0, nan), equal_nan=True), res
    assert res[2][0].tolist() == [1, 3, 4, 6] and res[3][0].tolist() == [0, 2, 4, 6], res


# ---- reduce -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", FLOATS)
@pytest.mark.parametrize("kind", ["normal", "cancel", "wide", "subnormal"])
def test_reduce_sum_mean_bound(plc, dt, kind):
    rng = np.random.default_rng(101)
    u = X.unit_roundoff(dt)
    for n in (1, 2, 4097, 3 * 4096 + 5):  # 4097: just above one block's share of elements
        x = gen(rng, kind, n + 50, dt)
        m = rng.random(n + 50) >= 0.1
        for off in OFFSETS[: 3 if n > 4097 else 5]:
            xs = x[off: off + n]
            for mask in (None, m[off: off + n]):
                if mask is not None and not mask.any():
                    continue
                xv = xs if mask is None else xs[mask]
                k = X.k_reduce(n, sms())
                what = f"{kind} {np.dtype(dt)} n={n} off={off} nulls={mask is not None}"
                got = reduce_(plc, xs, mask, "sum", dt, off)
                if kind == "subnormal":
                    assert got == X.exact_sum(xv), what  # exact in any order: catches flush-to-zero
                check_sum(got, xv, k, u, u, "sum " + what)
                check_sum(reduce_(plc, xs, mask, "sum", np.float64, off), xv, k, X.U64, X.U64, "sum->f64 " + what)
                check_mean(reduce_(plc, xs, mask, "mean", np.float64, off), xv, k, X.U64, X.U64, "mean " + what)
                mn, mx = min_max_exp(xv)
                assert same_value(reduce_(plc, xs, mask, "min", dt, off), mn) and same_value(reduce_(plc, xs, mask, "max", dt, off), mx), what


def test_reduce_one_wave_grid(plc):
    """Just above the element count one wave of blocks (8 per SM) covers: every thread folds more than its 16 elements."""
    rng = np.random.default_rng(102)
    n = 4096 * 8 * sms() + 3
    x = gen(rng, "cancel", n, np.float64)
    check_sum(reduce_(plc, x, None, "sum", np.float64, 1), x, X.k_reduce(n, sms()), X.U64, X.U64, "one wave")


@pytest.mark.parametrize("dt", FLOATS)
def test_reduce_specials(plc, dt):
    rng = np.random.default_rng(103)
    big = np.finfo(dt).max / 2
    x = np.full(4, big, dt)  # every order overflows
    assert reduce_(plc, x, None, "sum", dt) == np.inf and reduce_(plc, -x, None, "sum", dt) == -np.inf
    assert math.isnan(reduce_(plc, np.array([np.inf, 1, -np.inf], dt), None, "sum", dt))
    for n in (5, 4097):
        base = gen(rng, "normal", n, dt)
        for put in ([np.nan], [-np.nan], [np.inf], [-np.inf], [np.inf, -np.inf], [np.nan, np.inf]):
            x = base.copy()
            x[rng.choice(n, len(put), replace=False)] = put
            for mask in (None, rng.random(n) >= 0.2):
                xv = x if mask is None else x[mask]
                if not len(xv):
                    continue
                what = f"{put} n={n} nulls={mask is not None}"
                k, u = X.k_reduce(n, sms()), X.unit_roundoff(dt)  # (a special may sit under a null)
                check_sum(reduce_(plc, x, mask, "sum", dt, 3), xv, k, u, u, what)
                check_mean(reduce_(plc, x, mask, "mean", np.float64, 3), xv, k, X.U64, X.U64, what)
                mn, mx = min_max_exp(xv)
                assert same_value(reduce_(plc, x, mask, "min", dt, 3), mn) and same_value(reduce_(plc, x, mask, "max", dt, 3), mx), what


def test_reduce_mean_of_int64(plc):
    """MEAN of int64 accumulates in float64: each value is rounded once on load (k + 1)."""
    rng = np.random.default_rng(104)
    for n in (1, 4097, 20_001):
        x = rng.integers(-(2 ** 62), 2 ** 62, n + 7)
        for off in (0, 3):
            xs = x[off: off + n]
            ints = [int(a) for a in xs]
            exact = sum(ints) / n
            l1 = float(sum(abs(a) for a in ints))
            k = X.k_reduce(n, sms()) + 1
            X.check(reduce_(plc, xs, None, "mean", np.float64, off), exact, (2 * k * X.U64 * l1) / n + X.U64 * abs(exact), f"n={n} off={off}")


# ---- scan ---------------------------------------------------------------------------------------------------------
SCAN_WIDTHS = {1: np.int8, 2: np.int16, 4: np.float32, 8: np.float64}


@pytest.mark.parametrize("itemsize", [1, 2, 4, 8])
def test_scan_tile_boundaries(plc, itemsize):
    """Sizes around the scan tile of each element width, aligned and sliced, with and without nulls. Integer sums wrap
    exactly like numpy's, so a lost or doubled element fails bit-exactly; float sums are held to the bound."""
    rng = np.random.default_rng(110 + itemsize)
    dt = np.dtype(SCAN_WIDTHS[itemsize])
    tile = X.scan_tile(itemsize)
    for n in (1, tile - 1, tile, tile + 1, 3 * tile + 5):
        full = gen(rng, "cancel", n + 7, dt) if dt.kind == "f" else rng.integers(-100, 100, n + 7).astype(dt)
        fm = rng.random(n + 7) >= 0.05
        for off, nulls in ((0, False), (1, False), (7, True), (3, True)):
            x, m = full[off: off + n], (fm[off: off + n] if nulls else None)
            what = f"{dt} n={n} off={off} nulls={nulls}"
            v, ok = scan_(plc, x, m, "sum", True, off)
            valid = np.ones(n, bool) if m is None else m
            assert np.array_equal(np.ones(n, bool) if ok is None else ok, valid), what
            xz = np.where(valid, x, 0).astype(dt)
            if dt.kind != "f":
                assert np.array_equal(v[valid], np.cumsum(xz, dtype=dt)[valid]), what
            else:
                err, exact, l1 = X.prefix_errors(v, xz)
                u = X.unit_roundoff(dt)
                bound = np.array([X.sum_bound(X.k_scan(i, itemsize), u, l1[i], exact[i], u) for i in range(n)])
                bad = np.nonzero((err > bound) & valid)[0]
                assert len(bad) == 0, f"{what}: first row over the bound {bad[:5]}, err {err[bad[:5]]}, bound {bound[bad[:5]]}"
            for kind, ufunc in (("min", np.fmin), ("max", np.maximum)):
                xs = x.copy()
                if dt.kind == "f":
                    xs[rng.random(n) < 0.01] = np.nan
                got = scan_(plc, xs, m, kind, True, off)[0]
                fill = np.nan if (dt.kind == "f" and kind == "min") else ored._identity(ored.MIN if kind == "min" else ored.MAX, dt)
                exp = ufunc.accumulate(np.where(valid, xs, fill).astype(dt))
                assert np.array_equal(got[valid], exp[valid], equal_nan=True), f"{kind} {what}"


@pytest.mark.parametrize("dt", FLOATS)
@pytest.mark.parametrize("kind", ["wide", "subnormal"])
def test_scan_sum_inputs(plc, dt, kind):
    rng = np.random.default_rng(120)
    n = 2 * X.scan_tile(np.dtype(dt).itemsize) + 3
    x = gen(rng, kind, n, dt)
    v = scan_(plc, x, None, "sum", True, 1)[0]
    err, exact, l1 = X.prefix_errors(v, x)
    if kind == "subnormal":
        assert not err.any()
        return
    u = X.unit_roundoff(dt)
    assert all(err[i] <= X.sum_bound(X.k_scan(i, np.dtype(dt).itemsize), u, l1[i], exact[i], u) for i in range(n))
    xs = x.copy()
    xs[n // 2] = np.inf
    xs[n // 2 + 5] = -np.inf
    v = scan_(plc, xs, None, "sum", True)[0]
    assert np.isposinf(v[n // 2: n // 2 + 5]).all() and np.isnan(v[n // 2 + 5:]).all()


# ---- segmented reduce ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", FLOATS)
@pytest.mark.parametrize("kind", ["cancel", "wide", "subnormal", "specials"])
def test_segmented_reduce_bound(plc, dt, kind):
    rng = np.random.default_rng(130)
    lengths = [0, 1, 31, 32, 33, 0, 5000, 2, 64, 1]
    n = sum(lengths)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    full = gen(rng, "normal" if kind == "specials" else kind, n + 7, dt)
    if kind == "specials":
        full = with_specials(rng, full, 0.2)
    fm = rng.random(n + 7) >= 0.1
    u_same = X.unit_roundoff(dt)
    for off in (0, 1, 7):
        for nulls in (False, True):
            x, m = full[off: off + n], (fm[off: off + n] if nulls else None)
            res = {(k, od): segred_(plc, x, m, offsets, k, od, off) for k, od in
                   (("sum", dt), ("sum", np.float64), ("mean", np.float64), ("min", dt), ("max", dt))}
            for s, L in enumerate(lengths):
                sl = slice(offsets[s], offsets[s + 1])
                xv = x[sl] if m is None else x[sl][m[sl]]
                what = f"{kind} {np.dtype(dt)} seg={s} len={L} off={off} nulls={nulls}"
                for key, (v, ok) in res.items():
                    assert bool(ok[s]) == (len(xv) > 0), what
                if not len(xv):
                    continue
                k = X.k_segmented(L)
                got = res[("sum", dt)][0][s]
                if kind == "subnormal":
                    assert got == X.exact_sum(xv), what
                check_sum(got, xv, k, u_same, u_same, "sum " + what)
                check_sum(res[("sum", np.float64)][0][s], xv, k, X.U64, X.U64, "sum->f64 " + what)
                check_mean(res[("mean", np.float64)][0][s], xv, k, X.U64, X.U64, "mean " + what)
                mn, mx = min_max_exp(xv)
                assert same_value(res[("min", dt)][0][s], mn) and same_value(res[("max", dt)][0][s], mx), what


def test_segmented_mean_of_int64(plc):
    rng = np.random.default_rng(131)
    lengths = [1, 33, 4000]
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    x = rng.integers(-(2 ** 62), 2 ** 62, sum(lengths) + 3)
    v, _ = segred_(plc, x[3:], None, offsets, "mean", np.float64, 3)
    for s, L in enumerate(lengths):
        ints = [int(a) for a in x[3:][offsets[s]: offsets[s + 1]]]
        exact = sum(ints) / L
        k = X.k_segmented(L) + 1
        X.check(v[s], exact, 2 * k * X.U64 * float(sum(abs(a) for a in ints)) / L + X.U64 * abs(exact), f"seg {s}")


# ---- groupby: every path on the same data ---------------------------------------------------------------------------
HASH_KINDS = ["sum", "mean", "min", "max", "argmin", "argmax", "m2", "var", "std", "count"]
SORT_KINDS = ["sum", "mean", "min", "max", "m2", "var", "std", "count"]
PART_KINDS = ["sum", "min", "max", "mean", "count"]  # the partitioned path: one 8-byte integer key, at most 3 data ops, no nulls


def _groupby_cases():
    rng = np.random.default_rng(140)
    cases = []
    for dt in FLOATS:
        for kind in ("cancel", "wide", "subnormal", "specials"):
            sizes = [1, 2, 3, 31, 33, 700, 3000] + list(rng.integers(1, 40, 30))
            keys = np.repeat(np.arange(len(sizes), dtype=np.int64) * 7919 - 50_000, sizes)
            n = len(keys)
            perm = rng.permutation(n)
            keys = keys[perm]
            x = gen(rng, "normal" if kind == "specials" else kind, n, dt)
            if kind == "specials":
                x = with_specials(rng, x, 0.05)
            for nulls in (False, True):
                m = (rng.random(n) >= 0.1) if nulls else None
                # values viewed from row 3 / 7 of a longer column: unaligned data, and a mask read at a bit offset
                cases.append((f"{kind}-{np.dtype(dt)}-nulls={nulls}", keys, x, m, 7 if nulls else 3))
    # the NaN rule on tiny groups; padded past the partitioned path's row threshold
    keys = np.concatenate([np.repeat(np.arange(8, dtype=np.int64), 2), np.arange(100, 164, dtype=np.int64)])
    nan = np.nan
    for dt in FLOATS:
        v = np.concatenate([np.array([-nan, 1, nan, 1, nan, -nan, -0.0, 0.0, np.inf, nan, -np.inf, nan, 0.0, -0.0, np.inf, -np.inf], dt),
                            np.arange(64, dtype=dt)])
        cases.append((f"nan-rule-{np.dtype(dt)}", keys, v, None, 0))
    # a large mean and a small spread: the one-pass M2 formula cancels, and the bound says by how much
    keys = rng.integers(0, 4, 4000).astype(np.int64)
    cases.append(("large-mean", keys, 1e8 + rng.standard_normal(4000), None, 0))
    # int64 values: MEAN in float64
    keys = rng.integers(0, 9, 5000).astype(np.int64)
    cases.append(("int64-mean", keys, rng.integers(-(2 ** 52), 2 ** 52, 5000), None, 0))
    return cases


@pytest.fixture(scope="module")
def groupby_results(plc):
    cases = _groupby_cases()
    out = {}
    for path, kinds, env in (("hash", HASH_KINDS, None), ("sort", SORT_KINDS, {"B2_GROUPBY_SORT": "1"}),
                             ("partitioned", PART_KINDS, {"B2_GROUPBY_PARTITION_ROWS": "64"}),
                             ("partitioned-spill", PART_KINDS, {"B2_GROUPBY_PARTITION_ROWS": "64", "B2_GROUPBY_SMEM_SLOTS": "16"})):
        sel = [c for c in cases if not path.startswith("partitioned") or c[3] is None]
        jobs = [(c[1], c[2], c[3], kinds if np.asarray(c[2]).dtype.kind == "f" else ["sum", "mean", "count"], c[4]) for c in sel]
        res = [groupby_(plc, *j) for j in jobs] if env is None else groupby_in_subprocess(jobs, env)
        for c, j, r in zip(sel, jobs, res):
            out[(path, c[0])] = (c, j[3], r)
    return out


def _k_path(path, count):
    """Longest addition chain behind a group's SUM / MEAN (and, on the hash and partitioned paths, the one-pass M2's SUM and
    SUM_OF_SQUARES): atomics land in any order there; the sort path reduces each group with segmented_reduce, whose MEAN also
    rounds each value on its way to float64 (+1)."""
    return X.k_hash_group(count) if path != "sort" else X.k_segmented(count) + 1


def _two_pass(rows, xv, ddof):
    """The sort path's two-pass bounds for a group of `rows` rows (nulls included: segmented_reduce walks them all) whose valid
    values are xv: the MEAN to within mean_bound, the squared deviations summed by segmented_reduce."""
    k = X.k_segmented(rows)
    delta = X.mean_bound(k + 1, X.U64, X.abs_sum(xv), X.exact_sum(xv), len(xv), X.U64)
    return X.two_pass_bounds(k, xv, delta, ddof)


@pytest.mark.parametrize("path", ["hash", "sort", "partitioned", "partitioned-spill"])
def test_groupby_bounds(groupby_results, path):
    seen = 0
    for (p, name), (case, kinds, (gk, res)) in groupby_results.items():
        if p != path:
            continue
        seen += 1
        _, keys, x, m, _ = case
        uk = np.unique(keys)
        assert np.array_equal(gk, uk), name
        is_int = np.asarray(x).dtype.kind == "i"
        for gi, key in enumerate(uk):
            sel = keys == key
            if m is not None:
                sel &= m
            xv = np.asarray(x)[sel]
            r = {kind: (v[gi], True if ok is None else bool(ok[gi])) for kind, (v, ok) in zip(kinds, res)}
            what = f"{path} {name} key={key} count={len(xv)}"
            assert r["count"][0] == len(xv), what
            if not len(xv):
                assert not any(ok for kind, (v, ok) in r.items() if kind not in ("count", "m2")), what  # M2 has no null mask
                continue
            k = _k_path(path, len(xv))
            if is_int:
                ints = [int(a) for a in xv]
                assert r["sum"][0] == sum(ints), what
                exact = sum(ints) / len(ints)
                X.check(r["mean"][0], exact, (2 * (k + 1) * X.U64 * float(sum(abs(a) for a in ints))) / len(ints) + X.U64 * abs(exact), what)
                continue
            dt = np.asarray(x).dtype
            # hash / partitioned: float32 sums accumulate in float64; sort: segmented_reduce in the column's type
            u_sum = X.unit_roundoff(dt) if path == "sort" else X.U64
            check_sum(r["sum"][0], xv, k, u_sum, X.unit_roundoff(dt), "sum " + what)
            check_mean(r["mean"][0], xv, k, X.U64, X.U64, "mean " + what)
            if "subnormal" in name:
                assert r["sum"][0] == X.exact_sum(xv), what
            if "m2" in r:
                finite = np.isfinite(xv).all()
                if not finite:
                    assert math.isnan(r["m2"][0]), what
                elif path == "sort":  # two passes: never negative
                    m2, bm, var, bv, std, bs = _two_pass(int((keys == key).sum()), xv.astype(np.float64), 1)
                    assert r["m2"][0] >= 0, what
                    X.check(r["m2"][0], m2, bm, "m2 " + what)
                else:
                    X.check(r["m2"][0], X.exact_m2(xv), X.m2_bound(k, xv), "m2 " + what)
                assert r["var"][1] == (len(xv) > 1) and r["std"][1] == (len(xv) > 1), what
                if len(xv) > 1:
                    if not finite:
                        assert math.isnan(r["var"][0]) and math.isnan(r["std"][0]), what
                    elif path == "sort":
                        X.check(r["var"][0], var, bv, "var " + what)
                        X.check(r["std"][0], std, bs, "std " + what)
                    else:
                        var, bv, std, bs = X.var_std_bounds(k, xv, 1)
                        X.check(r["var"][0], var, bv, "var " + what)
                        if math.isnan(r["std"][0]):
                            # the formula's variance may come out negative, and its square root is NaN as in the reference
                            assert r["var"][0] < 0 and var - bv < 0, what
                        else:
                            X.check(r["std"][0], std, bs, "std " + what)
    assert seen


def test_groupby_large_mean_small_spread_matches_the_one_pass_formula(groupby_results):
    """The hash path's M2 = sumsq - sum^2 / n (the reference's hash formula) loses most of its digits here: it stays within
    that formula's bound and no tighter claim is made. The sort path takes two passes, as the reference's sort path does, and
    is held to that algorithm's bound, which is many times tighter."""
    for path in ("hash", "sort"):
        case, kinds, (gk, res) = groupby_results[(path, "large-mean")]
        _, keys, x, _, _ = case
        m2 = res[kinds.index("m2")][0]
        for gi, key in enumerate(gk):
            xv = x[keys == key]
            one_pass = X.m2_bound(_k_path(path, len(xv)), xv)
            assert one_pass > 1e-3 * X.exact_m2(xv)  # the one-pass formula cannot promise better than ~0.1 % here
            if path == "hash":
                X.check(m2[gi], X.exact_m2(xv), one_pass, f"{path} key={key}")
            else:
                exact, bound = _two_pass(len(xv), xv, 0)[:2]
                assert bound < 1e-9 * exact
                X.check(m2[gi], exact, bound, f"{path} key={key}")


def test_groupby_min_max_arg_agree_across_paths(groupby_results):
    """MIN / MAX bit-equal (as numbers) on every path that supports them, equal to the rule; ARGMIN / ARGMAX (hash path) point at
    the first row holding that value."""
    names = sorted({name for (_, name) in groupby_results})
    for name in names:
        case, _, _ = groupby_results[("hash", name)]
        _, keys, x, m, _ = case
        if np.asarray(x).dtype.kind != "f":
            continue
        uk = np.unique(keys)
        for path in ("hash", "sort", "partitioned", "partitioned-spill"):
            if (path, name) not in groupby_results:
                continue
            _, kinds, (gk, res) = groupby_results[(path, name)]
            r = dict(zip(kinds, res))
            for gi, key in enumerate(uk):
                sel = keys == key
                if m is not None:
                    sel &= m
                if not sel.any():
                    continue
                mn, mx = min_max_exp(x[sel])
                what = f"{path} {name} key={key}"
                assert same_value(r["min"][0][gi], mn) and same_value(r["max"][0][gi], mx), what
                if path == "hash":
                    rows = np.nonzero(sel)[0]
                    for kind, ext in (("argmin", mn), ("argmax", mx)):
                        first = rows[[same_value(v, ext) for v in x[rows]].index(True)]
                        assert r[kind][0][gi] == first, f"{kind} {what}: row {r[kind][0][gi]}, expected {first}"


def test_groupby_oracle_follows_the_rule(groupby_results):
    """The oracle (which pins types and validity for the other suites) computes the same MIN / MAX / ARGMIN / ARGMAX."""
    for (path, name), (case, kinds, (gk, res)) in groupby_results.items():
        if path != "hash" or not name.startswith(("nan-rule", "specials")):
            continue
        _, keys, x, m, _ = case
        ek, er = ogb.aggregate([(keys, None)], [((x, m), [KINDS[k] for k in ("min", "max", "argmin", "argmax")])])
        r = dict(zip(kinds, res))
        for j, kind in enumerate(("min", "max", "argmin", "argmax")):
            ev, em = er[0][j]
            ok = np.ones(len(ev), bool) if em is None else em
            assert all(same_value(a, b) for a, b in zip(r[kind][0][ok], ev[ok])), f"{kind} {name}"


# ---- grouped scan -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", FLOATS)
@pytest.mark.parametrize("kind", ["cancel", "wide", "specials"])
def test_groupby_scan_bound(plc, dt, kind):
    rng = np.random.default_rng(150)
    sizes = [1, 2, 33, 2100, 5000] + list(rng.integers(1, 20, 20))
    keys = np.repeat(np.arange(len(sizes), dtype=np.int32), sizes)
    keys = keys[rng.permutation(len(keys))]
    n = len(keys)
    full = gen(rng, "normal" if kind == "specials" else kind, n + 7, dt)
    if kind == "specials":
        full = with_specials(rng, full, 0.05)
    fm = rng.random(n + 7) >= 0.1
    u_out = X.unit_roundoff(dt)
    for off, nulls in ((0, False), (7, True)):
        x, m = full[off: off + n], (fm[off: off + n] if nulls else None)
        gk, ((s, sm), (mn, _), (mx, _)) = groupby_scan_(plc, keys, x, m, ["sum", "min", "max"], off)
        ek, er = ogb.scan([(keys, None)], [((x, m), [0, 3, 4])])
        assert np.array_equal(gk, ek[0][0])
        valid = np.ones(n, bool) if m is None else m[np.argsort(keys, kind="stable")]
        assert np.array_equal(np.ones(n, bool) if sm is None else sm, valid)
        for j, got in ((1, mn), (2, mx)):
            assert all(same_value(a, b) for a, b in zip(got[valid], er[0][j][0][valid])), f"{'min' if j == 1 else 'max'} off={off}"
        xs = x[np.argsort(keys, kind="stable")]
        starts = np.concatenate([[0], np.cumsum(np.bincount(keys))])
        for g in range(len(sizes)):
            b, e = starts[g], starts[g + 1]
            vg = valid[b:e]
            xg = np.where(vg, xs[b:e], 0).astype(dt)
            what = f"{kind} {np.dtype(dt)} group={g} off={off}"
            if not np.isfinite(xg).all():
                # rows from the first NaN / inf on: NaN, +inf or -inf exactly
                for i in np.nonzero(vg & ~np.isfinite(np.cumsum(np.abs(xg.astype(np.float64)))))[0]:
                    X.check(s[b + i], X.special_sum(xg[: i + 1]), 0.0, what)
                continue
            err, exact, l1 = X.prefix_errors(s[b:e].astype(np.float64), xg)
            # float32 values run in float64 and are rounded once into the output type
            bound = np.array([X.sum_bound(X.k_grouped_scan(i), X.U64, l1[i], exact[i], u_out) for i in range(e - b)])
            bad = np.nonzero((err > bound) & vg)[0]
            assert len(bad) == 0, f"{what}: rows {bad[:5]} err {err[bad[:5]]} bound {bound[bad[:5]]}"

"""Integer reduce, scan, segmented_reduce, groupby aggregations (hash, partitioned and sort-based paths) and the grouped scan over
each type's whole value range, against the exact references of tests/int_ref.py.

Values are drawn where integer kernels go wrong: uniformly over the whole range, pinned at min, min + 1, -1, 0, 1, max - 1 and
max, unsigned values with the top bit set, int64 values near +-2^62 / +-2^63 (sums that wrap once or several times), values
above 2^53 (whose conversion to double rounds) and runs whose product overflows. Every result is compared bit for bit, except
reduce / segmented_reduce MEAN, whose float sum depends on the order and is held to the bound of tests/exact_ref.py.
Under B2_EMU_RUN=1 without a device the cases run on the kernel emulator at reduced sizes."""
import math
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from tests import exact_ref as X
from tests import int_ref as R
from tests.impls import PlcImpl

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
TYPES = INTS + [np.bool_]


def _emulated() -> bool:
    if os.environ.get("B2_EMU_RUN") != "1":
        return False
    import torch

    return not torch.cuda.is_available()


EMU = _emulated()
BIG = 40_003 if EMU else 1_000_003  # past the multi-block fold of reduce_kernel either way
NAME = lambda d: np.dtype(d).name


def sms() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


# ---- inputs -----------------------------------------------------------------------------------------------------------
def pinned(dt):
    lo, hi = R.bounds(dt)
    return sorted({lo, lo + 1, max(lo, -1), 0, 1, hi - 1, hi})


def gen(rng, dt, n, pattern):
    """n values of dt. pattern: uniform | pinned | top (unsigned top bit set; signed: the negative half) | wrap (int64 near
    +-2^62 / +-2^63, above 2^53) | product (small factors with a few large ones: products overflow) | mixed (all of these)."""
    dt = np.dtype(dt)
    if dt == np.bool_:
        return rng.random(n) < (0.5 if pattern != "product" else 0.97)
    lo, hi = R.bounds(dt)
    bits = dt.itemsize * 8
    if pattern == "uniform":
        return rng.integers(lo, hi, n, dtype=dt, endpoint=True)
    if pattern == "pinned":
        return np.array(pinned(dt), dtype=object)[rng.integers(0, len(pinned(dt)), n)].astype(dt)
    if pattern == "top":
        return rng.integers(1 << (bits - 1), hi, n, dtype=dt, endpoint=True) if lo == 0 else rng.integers(lo, -1, n, dtype=dt, endpoint=True)
    if pattern == "wrap":
        if bits < 64:
            return gen(rng, dt, n, "top")
        c = rng.integers(0, 5, n)
        off = rng.integers(0, 1 << 20, n)
        base = np.array([2 ** 62, 2 ** 63 - 2 ** 20, 2 ** 53 + 1, 2 ** 62 + 2 ** 61, 2 ** 63 - 2 ** 21], dtype=object)
        v = base[c] + off.astype(object)
        if lo < 0:
            v = np.where(rng.random(n) < 0.35, -v, v)
        else:
            v = v + np.where(rng.random(n) < 0.5, 2 ** 63 - 2 ** 21, 0)
        return v.astype(dt)
    if pattern == "product":
        v = rng.integers(max(lo, -3), min(hi, 3), n, endpoint=True).astype(dt)
        v[v == 0] = 2
        big = rng.random(n) < 0.02
        v[big] = rng.integers(lo, hi, int(big.sum()), dtype=dt, endpoint=True)
        return v
    parts = [gen(rng, dt, n, p) for p in ("uniform", "pinned", "top", "wrap", "product")]
    return np.choose(rng.integers(0, 5, n), parts).astype(dt)


def column(plc, v, m=None, off=0):
    """The values as a view starting at row `off` of a longer column (unaligned data, mask read at a bit offset)."""
    if not off:
        return plc.Column.from_numpy(v, m)
    pv = np.concatenate([np.ones(off, v.dtype), v])
    pm = None if m is None else np.concatenate([np.zeros(off, bool), m])
    return plc.Column.from_numpy(pv, pm).slice(off, off + len(v))


def agg(plc, name):
    return PlcImpl(plc)._agg(name)


def same(got, exp):
    """Bit-exact equality of a device value with a reference value (Python int / float / bool)."""
    if isinstance(exp, bool):
        return bool(got) == exp
    if isinstance(exp, float):
        g = float(got)
        return g == exp and math.copysign(1.0, g) == math.copysign(1.0, exp)
    return int(got) == exp


def out_types(dt):
    """Output types of SUM / PRODUCT: the input type, INT64, UINT64, a narrower integer, FLOAT64, FLOAT32."""
    narrow = np.uint8 if np.dtype(dt) == np.int8 else np.int8
    return list(dict.fromkeys([np.dtype(x) for x in (dt, np.int64, np.uint64, narrow, np.float64, np.float32)]))


def inits(rng, dt):
    """No initial value, a valid one at the type's extreme, a null one."""
    lo, hi = R.bounds(dt)
    v = hi if np.dtype(dt).kind != "i" else lo
    return [None, (v if np.dtype(dt) != np.bool_ else True, True), (0, False)]


def masks(rng, n):
    """(valid | None, offset): no nulls; no nulls at an unaligned offset; nulls at a bit offset not a multiple of 32."""
    return [(None, 0), (None, 3), (rng.random(n) >= 0.3, 45)]


# ---- reduce -----------------------------------------------------------------------------------------------------------
def check_reduce(plc, v, m, off, kinds, outs, init_list, what):
    col = column(plc, v, m, off)
    xs = R.ints(v, m)
    for kind in kinds:
        for od in (outs if kind in ("sum", "product") else [v.dtype]):
            for init in (init_list if kind != "mean" else [None]):
                s = None if init is None else plc.Scalar.from_py(init[0], col.type(), valid=init[1])
                if kind == "mean":
                    for fd in (np.float64, np.float32):
                        out = plc.reduce.reduce(col, agg(plc, "mean"), plc.DataType.from_numpy(fd))
                        got, ok = out._get()
                        w = f"{what} mean -> {np.dtype(fd)}"
                        assert ok == bool(xs), w
                        if xs:
                            terms = [R.to_float(a, fd) for a in xs]
                            u = X.unit_roundoff(fd)
                            ex = X.exact_sum(terms)
                            X.check(got, ex / len(xs), X.mean_bound(X.k_reduce(len(v), sms()), u, X.abs_sum(terms), ex, len(xs), u), w)
                    continue
                out = plc.reduce.reduce(col, agg(plc, kind), plc.DataType.from_numpy(od), s)
                got, ok = out._get()
                exp, eok = R.reduce_ints(xs, v.dtype, R.__dict__[kind.upper()], od, init)
                w = f"{what} {kind} -> {np.dtype(od)} init={init}"
                assert ok == eok, f"{w}: valid {ok}"
                if eok:
                    assert same(got, exp), f"{w}: got {got!r}, expected {exp!r}"


@pytest.mark.parametrize("dt", TYPES, ids=NAME)
def test_reduce(plc, dt):
    rng = np.random.default_rng(400 + np.dtype(dt).num)
    kinds = ["sum", "product", "min", "max", "mean"]
    outs = out_types(dt)
    for n in (1, 31, 4097):
        for pattern in ("mixed", "wrap", "product", "pinned"):
            v = gen(rng, dt, n, pattern)
            for m, off in masks(rng, n):
                check_reduce(plc, v, m, off, kinds, outs, inits(rng, dt), f"{NAME(dt)} n={n} {pattern} off={off} nulls={m is not None}")
    # the multi-block fold; a single value; an all-null column
    for pattern in ("mixed",):
        v = gen(rng, dt, BIG, pattern)
        for m, off in ((None, 0), (rng.random(BIG) >= 0.5, 45)):
            check_reduce(plc, v, m, off, kinds, outs, [None], f"{NAME(dt)} n={BIG} {pattern} off={off}")
    v = gen(rng, dt, 40, "mixed")
    check_reduce(plc, v, np.zeros(40, bool), 5, kinds, outs, inits(rng, dt), f"{NAME(dt)} all null")


def test_reduce_known_answers(plc):
    """SUM of UINT64 [2^63, 1] to FLOAT64 accumulates in int64 as the reference does: -2^63 + 1, converted."""
    col = plc.Column.from_numpy(np.array([2 ** 63, 1], np.uint64))
    for od, exp in ((np.float64, -9.223372036854776e18), (np.float32, -9.223372036854776e18), (np.uint64, 2 ** 63 + 1),
                    (np.int64, -(2 ** 63) + 1)):
        got, ok = plc.reduce.reduce(col, agg(plc, "sum"), plc.DataType.from_numpy(od))._get()
        assert ok and same(got, exp), (od, got, exp)


# ---- scan -------------------------------------------------------------------------------------------------------------
def scan_sizes(dt):
    t = X.scan_tile(np.dtype(dt).itemsize)
    return [1, 33, t - 1, t, t + 1, 2 * t + 3]


@pytest.mark.parametrize("dt", TYPES, ids=NAME)
def test_scan(plc, dt):
    rng = np.random.default_rng(500 + np.dtype(dt).num)
    for n in scan_sizes(dt):
        v = gen(rng, dt, n, "mixed" if n < 100 else ("wrap", "product", "mixed")[n % 3])
        nm = rng.random(n) >= 0.1
        nm[: min(n, 40)] = True  # INCLUDE: a few valid rows before the first null
        for m, off in ((None, 0), (None, 3), (nm, 45)):
            col = column(plc, v, m, off)
            for kind in ("sum", "product", "min", "max"):
                for inclusive in (True, False):
                    for include in (False, True):
                        out = plc.reduce.scan(col, agg(plc, kind), plc.reduce.ScanType.INCLUSIVE if inclusive else plc.reduce.ScanType.EXCLUSIVE,
                                              plc.NullPolicy.INCLUDE if include else plc.NullPolicy.EXCLUDE)
                        gv, gm = out.to_numpy()
                        exp, em = R.scan(v, m, getattr(R, kind.upper()), inclusive, include)
                        w = f"{NAME(dt)} n={n} off={off} {kind} {'incl' if inclusive else 'excl'} {'INCLUDE' if include else 'EXCLUDE'}"
                        assert (gm is None) == (em is None) or (em is None and gm.all()), f"{w}: mask"
                        if em is not None:
                            assert np.array_equal(gm, np.array(em, bool)), f"{w}: mask"
                        gl = gv.tolist()
                        for i, e in enumerate(exp):
                            if e is not None and not same(gl[i], e):
                                raise AssertionError(f"{w}: row {i}: got {gl[i]!r}, expected {e!r}")


# ---- segmented_reduce -------------------------------------------------------------------------------------------------
SEG_LENGTHS = [0, 1, 31, 32, 33, 1000, 0, 2, 1, 64, 0, 3, 33, 7]


@pytest.mark.parametrize("dt", TYPES, ids=NAME)
def test_segmented_reduce(plc, dt):
    rng = np.random.default_rng(600 + np.dtype(dt).num)
    offsets = np.concatenate([[0], np.cumsum(SEG_LENGTHS)]).astype(np.int32)
    n = int(offsets[-1])
    oc = plc.Column.from_numpy(offsets)
    for pattern in ("mixed", "wrap", "product"):
        v = gen(rng, dt, n, pattern)
        nm = rng.random(n) >= 0.3
        nm[offsets[3]: offsets[4]] = False  # a segment with no valid value
        for m, off in ((None, 0), (nm, 45)):
            col = column(plc, v, m, off)
            for kind in ("sum", "product", "min", "max", "mean"):
                for od in (out_types(dt) if kind in ("sum", "product") else [v.dtype] if kind != "mean" else [np.dtype(np.float64), np.dtype(np.float32)]):
                    for include in (False, True):
                        for init in (inits(rng, dt) if kind != "mean" else [None]):
                            s = None if init is None else plc.Scalar.from_py(init[0], col.type(), valid=init[1])
                            out = plc.reduce.segmented_reduce(col, oc, agg(plc, kind), plc.DataType.from_numpy(od),
                                                              plc.NullPolicy.INCLUDE if include else plc.NullPolicy.EXCLUDE, s)
                            gv, gm = out.to_numpy()
                            w = f"{NAME(dt)} {pattern} off={off} {kind} -> {np.dtype(od)} include={include} init={init}"
                            if kind == "mean":
                                exp = R.segmented_reduce(v, m, offsets.tolist(), R.SUM, np.int64, include)
                                for g, (b, e) in enumerate(zip(offsets[:-1], offsets[1:])):
                                    xs = R.ints(v[b:e], None if m is None else m[b:e])
                                    ok = exp[g][1] and len(xs) > 0
                                    assert bool(gm[g]) == exp[g][1], f"{w} segment {g}: valid"
                                    if ok:
                                        terms = [R.to_float(a, od) for a in xs]
                                        u = X.unit_roundoff(od)
                                        ex = X.exact_sum(terms)
                                        X.check(gv[g], ex / len(xs), X.mean_bound(X.k_segmented(e - b) + 1, u, X.abs_sum(terms), ex, len(xs), u),
                                                f"{w} segment {g}")
                                continue
                            exp = R.segmented_reduce(v, m, offsets.tolist(), getattr(R, kind.upper()), od, include, init)
                            for g, (e, eok) in enumerate(exp):
                                assert bool(gm[g]) == eok, f"{w} segment {g}: valid {gm[g]}"
                                if eok:
                                    assert same(gv[g].item(), e), f"{w} segment {g}: got {gv[g]!r}, expected {e!r}"


# ---- groupby ----------------------------------------------------------------------------------------------------------
GB_KINDS = ["sum", "product", "min", "max", "mean", "sum_of_squares", "count", "argmin", "argmax"]


def run_groupby(plc, keys, kmask, vals, vmask, kinds, off=0, include_nulls=False, keys_sorted=False):
    """One groupby aggregate -> {key (None for the null key): {kind: (value, valid)}}, values as Python scalars."""
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_numpy(keys, kmask)]), plc.NullPolicy.INCLUDE if include_nulls else plc.NullPolicy.EXCLUDE,
                             plc.Sorted.YES if keys_sorted else plc.Sorted.NO)
    k, res = gb.aggregate([plc.groupby.GroupByRequest(column(plc, vals, vmask, off), [agg(plc, x) for x in kinds])])
    kv, km = k.columns()[0].to_numpy()
    if kv.dtype.kind == "m":
        kv = kv.view(np.int64)
    cols = [c.to_numpy() for c in res[0].columns()]
    out = {}
    for g, key in enumerate(kv.tolist()):
        key = None if (km is not None and not km[g]) else key
        assert key not in out, f"group {key} returned twice"
        out[key] = {kind: (v[g].item(), True if m is None else bool(m[g])) for kind, (v, m) in zip(kinds, cols)}
    return out


def check_groups(res, keys, kmask, vals, vmask, kinds, what, include_nulls=False):
    groups = R.group_rows(keys, kmask, include_nulls)
    assert sorted(res, key=repr) == sorted(groups, key=repr), f"{what}: group keys"
    prep = R.prepare(vals, vmask)
    for key, rows in groups.items():
        for kind in kinds:
            got, ok = res[key][kind]
            exp, eok = R.group_agg(vals, vmask, rows, kind, prep)
            w = f"{what} key={key} {kind} rows={len(rows)}"
            if kind in ("count", "count_all"):
                assert got == exp, f"{w}: got {got}, expected {exp}"
                continue
            assert ok == eok, f"{w}: valid {ok}"
            if not eok:
                continue
            if kind in ("argmin", "argmax"):
                assert got in exp, f"{w}: row {got} does not hold the extreme (rows {exp[:5]})"
            else:
                assert same(got, exp), f"{w}: got {got!r}, expected {exp!r}"


def gb_input(rng, dt, pattern, sizes):
    """Shuffled rows of groups of the given sizes (int64 keys), their values, and a value mask with an all-null group."""
    keys = np.repeat(np.arange(len(sizes), dtype=np.int64) * 7919 - 100_000, sizes)
    p = rng.permutation(len(keys))
    keys = keys[p]
    vals = gen(rng, dt, len(keys), pattern)
    vm = rng.random(len(keys)) >= 0.25
    vm[keys == keys[0]] = False
    return keys, vals, vm


GB_SIZES = [1, 2, 3, 31, 33, 700, 5, 64, 2, 1, 4, 9, 100, 17]


@pytest.mark.parametrize("dt", TYPES, ids=NAME)
def test_hash_groupby(plc, dt):
    rng = np.random.default_rng(700 + np.dtype(dt).num)
    for pattern in ("mixed", "wrap", "product", "uniform"):
        keys, vals, vm = gb_input(rng, dt, pattern, GB_SIZES)
        for m, off in ((None, 0), (vm, 45)):
            res = run_groupby(plc, keys, None, vals, m, GB_KINDS, off)
            check_groups(res, keys, None, vals, m, GB_KINDS, f"{NAME(dt)} {pattern} off={off} nulls={m is not None}")


def test_hash_groupby_duration(plc):
    """MIN / MAX of a duration column (integer storage) at the int64 extremes."""
    rng = np.random.default_rng(710)
    keys, vals, vm = gb_input(rng, np.int64, "mixed", GB_SIZES)
    d = vals.view("m8[ns]")
    for m in (None, vm):
        res = run_groupby(plc, keys, None, d, m, ["min", "max", "count"])
        check_groups(res, keys, None, vals, m, ["min", "max", "count"], f"duration nulls={m is not None}")


@pytest.mark.parametrize("kdt", [np.int64, np.uint64, np.int8, np.uint16], ids=NAME)
def test_hash_groupby_extreme_keys(plc, kdt):
    """Keys at INT64_MIN, -1, UINT64_MAX and the ends of INT8 / UINT16, with nullable keys under EXCLUDE and INCLUDE."""
    rng = np.random.default_rng(720)
    lo, hi = R.bounds(kdt)
    kv = sorted({lo, lo + 1, max(lo, -1), 0, 1, hi - 1, hi})
    n = 3000
    keys = np.array(kv, dtype=object)[rng.integers(0, len(kv), n)].astype(kdt)
    kmask = rng.random(n) >= 0.1
    vals = gen(rng, np.int64, n, "mixed")
    vm = rng.random(n) >= 0.2
    kinds = ["sum", "min", "max", "mean", "count", "argmax"]
    for km in (None, kmask):
        for inc in (False, True):
            res = run_groupby(plc, keys, km, vals, vm, kinds, include_nulls=inc)
            check_groups(res, keys, km, vals, vm, kinds, f"keys {NAME(kdt)} nullable={km is not None} include={inc}", include_nulls=inc)


# ---- paths forced in a separate process (environment switches read once per process) ------------------------------------
_WORKER = r"""
import os, pickle, sys
sys.path.insert(0, '.')
import torch
if os.environ.get('B2_EMU_RUN') == '1' and not torch.cuda.is_available():
    from tests.emu.harness import install
    install()
import cudf_b200.pylibcudf as plc
from tests.test_integer_extremes_gpu import run_groupby
with open(sys.argv[1], 'rb') as f:
    jobs = pickle.load(f)
with open(sys.argv[2], 'wb') as f:
    pickle.dump([run_groupby(plc, *job) for job in jobs], f)
print('WORKER_OK')
"""


def run_forced(jobs, env):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.pkl"), os.path.join(d, "out.pkl")
        with open(src, "wb") as f:
            pickle.dump(jobs, f)
        r = subprocess.run([sys.executable, "-c", _WORKER, src, dst], capture_output=True, text=True, env=dict(os.environ, **env), cwd=ROOT,
                           timeout=1800)
        assert "WORKER_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
        with open(dst, "rb") as f:
            return pickle.load(f)


PGB_KINDS = ["sum", "min", "max", "mean", "count"]


@pytest.mark.parametrize("est", ["0", "1"])
def test_partitioned_groupby(est):
    """groupby.cu::pgb_agg_kernel, forced with B2_GROUPBY_PARTITION_ROWS=1 (est: the histogram-free partition pass). UINT32
    values >= 2^31 must not be sign-extended on their way into the 8-byte accumulator (pgb_value_bits)."""
    rng = np.random.default_rng(800)
    n, G = (5000, 300) if EMU else (60_000, 2000)
    jobs, cases = [], []
    for dt in (np.int32, np.uint32, np.int64, np.uint64):
        for pattern in ("mixed", "wrap", "top"):
            keys = rng.integers(0, G, n).astype(np.int64) * 1_000_003 - 5
            keys[:7] = [np.iinfo(np.int64).min, -1, 0, 1, np.iinfo(np.int64).max, -2, 2]
            vals = gen(rng, dt, n, pattern)
            jobs.append((keys, None, vals, None, PGB_KINDS))
            cases.append((keys, vals, f"{NAME(dt)} {pattern}"))
    env = dict(B2_GROUPBY_PARTITION_ROWS="1", B2_GROUPBY_EST=est, B2_GROUPBY_EST_MIN="1")
    for (keys, vals, what), res in zip(cases, run_forced(jobs, env)):
        check_groups(res, keys, None, vals, None, PGB_KINDS, f"partitioned est={est} {what}")


SORT_KINDS = ["sum", "product", "min", "max", "mean", "count"]


def m2_small(vals, valid, rows):
    """Sort-path M2 of a group of at most two valid values, where it does not depend on the order of the sum: the MEAN is
    double(INT64 SUM) / count, then (double(x) - mean)^2 summed (group_m2.cu)."""
    mean, ok = R.group_agg(vals, valid, rows, "mean")
    if not ok:
        return 0.0
    xs = [R.to_float(a, np.float64) for a in R.ints(vals[rows], None if valid is None else valid[rows])]
    t = [(x - mean) * (x - mean) for x in xs]
    return t[0] + t[1] if len(t) == 2 else t[0]


@pytest.mark.parametrize("dt", TYPES, ids=NAME)
def test_sort_groupby(plc, dt):
    """The sort-based path, reached with B2_GROUPBY_SORT=1 and by adding MEDIAN to the request, agrees bit for bit with the
    reference and with the hash path; M2 of groups with one or two values is exact too."""
    rng = np.random.default_rng(900 + np.dtype(dt).num)
    jobs, cases = [], []
    for pattern in ("mixed", "wrap", "product", "uniform"):
        keys, vals, vm = gb_input(rng, dt, pattern, GB_SIZES)
        for m, off in ((None, 0), (vm, 45)):
            cases.append((keys, vals, m, off, f"{NAME(dt)} {pattern} off={off} nulls={m is not None}"))
            jobs.append((keys, None, vals, m, SORT_KINDS + ["m2"], off))
    forced = run_forced(jobs, dict(B2_GROUPBY_SORT="1"))
    for (keys, vals, m, off, what), fres in zip(cases, forced):
        hres = run_groupby(plc, keys, None, vals, m, SORT_KINDS, off)
        mres = run_groupby(plc, keys, None, vals, m, SORT_KINDS + ["m2", "median"], off)
        for route, res in (("hash", hres), ("forced sort", fres), ("sort next to MEDIAN", mres)):
            check_groups(res, keys, None, vals, m, SORT_KINDS, f"{route} {what}")
            for key in hres:
                for kind in SORT_KINDS:
                    a, b = hres[key][kind], res[key][kind]
                    assert a[1] == b[1] and (not a[1] or same(b[0], a[0])), f"{route} {what} key={key} {kind}: {b} vs hash {a}"
        for route, res in (("forced sort", fres), ("sort next to MEDIAN", mres)):
            for key, rows in R.group_rows(keys).items():
                nv = len(rows) if m is None else int(m[rows].sum())
                if nv <= 2:
                    assert same(res[key]["m2"][0], m2_small(vals, m, rows)), f"{route} {what} key={key} m2: {res[key]['m2'][0]!r}"


# ---- grouped scan -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", INTS, ids=NAME)
def test_grouped_scan(plc, dt):
    rng = np.random.default_rng(1000 + np.dtype(dt).num)
    kinds = ["sum", "min", "max", "count"]
    for pattern in ("mixed", "wrap"):
        keys, vals, vm = gb_input(rng, dt, pattern, GB_SIZES + [3000])
        for m, off in ((None, 0), (vm, 45)):
            gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_numpy(keys)]))
            k, res = gb.scan([plc.groupby.GroupByRequest(column(plc, vals, m, off), [agg(plc, x) for x in kinds])])
            order = np.argsort(keys, kind="stable")
            assert np.array_equal(k.columns()[0].to_numpy()[0], keys[order])
            for kind, c in zip(kinds, res[0].columns()):
                gv, gm = c.to_numpy()
                gl = gv.tolist()
                w = f"{NAME(dt)} {pattern} off={off} {kind}"
                pos = 0
                prep = R.prepare(vals, m)
                for key, rows in sorted(R.group_rows(keys).items()):
                    for r, e in zip(rows, R.group_scan(vals, m, rows, kind, prep)):
                        if e is None:
                            assert gm is not None and not gm[pos], f"{w} key={key} row {r}: not null"
                        else:
                            assert gm is None or gm[pos], f"{w} key={key} row {r}: null"
                            assert same(gl[pos], e), f"{w} key={key} row {r}: got {gl[pos]!r}, expected {e!r}"
                        pos += 1

"""GPU parity on seeded random inputs: CUDA path (through the C ABI) vs the oracle, bit-exact for indices and
integer aggregates, relative tolerance for floating-point reductions (written in each test)."""
import numpy as np
import pytest

from oracle import groupby as ogb
from oracle import join as ojoin
from oracle import reduce as ored
from tests.helpers import assert_columns_equal
from tests.impls import OracleImpl, PlcImpl, sort_groups

pytestmark = pytest.mark.gpu

F64_RTOL = 1e-6   # north_star tolerance for float reductions
F32_RTOL = 2e-4   # float32 accumulations (atomics / tree order differ from the float64 oracle)


@pytest.fixture
def cu(plc):
    return PlcImpl(plc)


def rnd_col(rng, n, dtype, null_frac=0.0, lo=-50, hi=50):
    dt = np.dtype(dtype)
    if dt == np.bool_:
        v = rng.integers(0, 2, n).astype(bool)
    elif dt.kind == "f":
        v = (rng.standard_normal(n) * 10).astype(dt)
    elif dt.kind == "u":
        v = rng.integers(0, hi, n).astype(dt)
    else:
        v = rng.integers(max(lo, np.iinfo(dt).min), min(hi, np.iinfo(dt).max), n).astype(dt)
    m = None
    if null_frac > 0:
        m = rng.random(n) >= null_frac
    return v, m


# ---- join ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64, np.uint32, np.uint64, np.float32, np.float64, np.bool_])
@pytest.mark.parametrize("kind", ["inner_join", "left_join", "full_join"])
def test_join_random_single_key(cu, dtype, kind):
    rng = np.random.default_rng(42)
    sizes = [(1, 1, 0.0), (100, 37, 0.0), (1000, 1000, 0.2), (20_000, 5_000, 0.1), (5_000, 60_000, 0.0)]
    if np.dtype(dtype) == np.bool_:
        sizes = sizes[:3]  # two distinct keys: the output is ~n*m/2 pairs, keep it small
    for nl, nr, nf in sizes:
        l = [rnd_col(rng, nl, dtype, nf, -30, 30)]
        r = [rnd_col(rng, nr, dtype, nf, -30, 30)]
        for ne in (0, 1):
            got = getattr(cu, kind)(l, r, ne)
            exp = getattr(ojoin, kind)(l, r, ne)
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), f"{kind} {np.dtype(dtype)} {nl}x{nr} ne={ne}"


def test_join_multi_key(cu):
    rng = np.random.default_rng(43)
    for n in (500, 30_000):
        l = [rnd_col(rng, n, np.int32, 0.1, 0, 20), rnd_col(rng, n, np.int16, 0.1, 0, 5), rnd_col(rng, n, np.int8, 0.0, 0, 3)]
        r = [rnd_col(rng, n // 2, np.int32, 0.1, 0, 20), rnd_col(rng, n // 2, np.int16, 0.1, 0, 5), rnd_col(rng, n // 2, np.int8, 0.0, 0, 3)]
        for ne in (0, 1):
            got = cu.inner_join(l, r, ne)
            exp = ojoin.inner_join(l, r, ne)
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])


def test_wide_keys_join_and_groupby(plc):
    """Keys wider than 8 bytes: the table holds a hash of the row and confirms it against the key columns."""
    cu, o = PlcImpl(plc), OracleImpl()
    rng = np.random.default_rng(91)
    # join: (int64, int64 with nulls) and (int32, float64 with NaN / -0, int64)
    for nl, nr in [(1, 1), (20_000, 7_000), (3_000, 50_000)]:
        l = [(rng.integers(0, 40, nl).astype(np.int64), None), (rng.integers(0, 30, nl).astype(np.int64), rng.random(nl) < 0.9)]
        r = [(rng.integers(0, 40, nr).astype(np.int64), None), (rng.integers(0, 30, nr).astype(np.int64), rng.random(nr) < 0.9)]
        for kind in ("inner_join", "left_join", "full_join"):
            for ne in (0, 1):
                got, exp = getattr(cu, kind)(l, r, ne), getattr(o, kind)(l, r, ne)
                assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (nl, nr, kind, ne)
        assert cu.inner_join_size(l, r) == o.inner_join_size(l, r)
    # sliced views of both sides (offsets not a multiple of 32): row ids count from the start of the view
    (lb, le), (rb, re) = (5, 2_990), (37, 49_000)
    lt = plc.Table([plc.Column.from_numpy(v, m).slice(lb, le) for v, m in l])
    rt = plc.Table([plc.Column.from_numpy(v, m).slice(rb, re) for v, m in r])
    ls = [(v[lb:le], None if m is None else m[lb:le]) for v, m in l]
    rs = [(v[rb:re], None if m is None else m[rb:re]) for v, m in r]
    for kind in ("inner_join", "left_join", "full_join"):
        for ne in (0, 1):
            res = getattr(plc.join, kind)(lt, rt, ne)
            got = ojoin.canonical(res[0].to_numpy()[0], res[1].to_numpy()[0])
            exp = getattr(o, kind)(ls, rs, ne)
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), ("sliced", kind, ne)
    f = np.array([0.0, -0.0, np.nan, 1.5, np.nan, 2.0])
    l = [(np.arange(6, dtype=np.int32) % 2, None), (f, None), (np.arange(6, dtype=np.int64) % 2, None)]
    r = [(np.array([0, 1, 0, 1], np.int32), None), (np.array([-0.0, np.nan, np.nan, 1.5]), None), (np.array([0, 1, 0, 1], np.int64), None)]
    got, exp = cu.inner_join(l, r), o.inner_join(l, r)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
    # groupby aggregate + scan on (int64, int64) keys
    n = 60_000
    keys = [(rng.integers(0, 50, n).astype(np.int64), None), (rng.integers(-20, 20, n).astype(np.int64), rng.random(n) < 0.95)]
    vals = (rng.integers(-1000, 1000, n).astype(np.int32), rng.random(n) < 0.8)
    kinds = ["sum", "min", "max", "count", "count_all"]
    for inc in (False, True):
        gk, gr = sort_groups(*cu.groupby(keys, [(vals, kinds)], include_nulls=inc))
        ek, er = sort_groups(*o.groupby(keys, [(vals, kinds)], include_nulls=inc))
        for a, b in zip(gk, ek):
            assert_columns_equal(a, b, what="keys")
        for j, kind in enumerate(kinds):
            assert_columns_equal(gr[0][j], er[0][j], what=kind)
    nn = [(keys[0][0], None), (keys[1][0], None)]
    gk, gr = cu.groupby_scan(nn, [(vals, ["sum", "count"])])
    ek, er = o.groupby_scan(nn, [(vals, ["sum", "count"])])
    for a, b in zip(gk, ek):
        assert_columns_equal(a, b, what="scan keys")
    for j in range(2):
        assert_columns_equal(gr[0][j], er[0][j], what=f"scan {j}")


def test_hash_join_object_reuse_and_errors(plc):
    rng = np.random.default_rng(44)
    build = (rng.integers(0, 1000, 50_000).astype(np.int64), None)
    hj = plc.join.HashJoin(plc.Table([plc.Column.from_numpy(build[0])]), plc.NullEquality.EQUAL)
    for n in (9, 5, 3, 40_000):  # HashJoinSequentialProbes (join_tests.cpp:2040-2123): build once, probe many
        probe = (rng.integers(0, 1500, n).astype(np.int64), None)
        pt = plc.Table([plc.Column.from_numpy(probe[0])])
        l, r = hj.inner_join(pt)
        got = ojoin.canonical(l.to_numpy()[0], r.to_numpy()[0])
        exp = ojoin.inner_join([probe], [build])
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
        assert hj.inner_join_size(pt) == len(exp[0])
        assert hj.left_join_size(pt) == len(ojoin.left_join([probe], [build])[0])
        assert hj.full_join_size(pt) == len(ojoin.full_join([probe], [build])[0])
    t = plc.Table([plc.Column.from_numpy(np.array([3, 1, 2, 0, 3], np.int32))])
    for lf in (-0.1, 0.0, 1.5):  # InvalidLoadFactor (join_tests.cpp:346-366) -> std::invalid_argument
        with pytest.raises(ValueError):
            plc.join.HashJoin(t, plc.NullEquality.EQUAL, has_nulls=False, load_factor=lf)
    # load_factor 1.0 is legal (join_tests.cpp:346-366 rejects only <= 0 and > 1): a power-of-two build must not fill the table
    for nb in (16, 1024):
        b = np.arange(nb, dtype=np.int64)
        hj1 = plc.join.HashJoin(plc.Table([plc.Column.from_numpy(b)]), plc.NullEquality.EQUAL, has_nulls=False, load_factor=1.0)
        pr = np.array([0, nb - 1, nb, -5, 7], np.int64)
        l, r = hj1.inner_join(plc.Table([plc.Column.from_numpy(pr)]))
        got = ojoin.canonical(l.to_numpy()[0], r.to_numpy()[0])
        exp = ojoin.inner_join([(pr, None)], [(b, None)])
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
    with pytest.raises(TypeError):  # cudf::data_type_error: mismatched key types
        plc.join.inner_join(t, plc.Table([plc.Column.from_numpy(np.array([1.0, 2.0]))]), plc.NullEquality.EQUAL)
    with pytest.raises(ValueError):  # std::invalid_argument: column count mismatch
        plc.join.inner_join(t, plc.Table([t.columns()[0], t.columns()[0]]), plc.NullEquality.EQUAL)
    # nullable_join::NO rejects a probe table with nulls (hash_join.cu:53-55)
    hj2 = plc.join.HashJoin(t, plc.NullEquality.EQUAL, has_nulls=False)
    with pytest.raises(ValueError):
        hj2.inner_join(plc.Table([plc.Column.from_numpy(np.array([1, 2], np.int32), np.array([True, False]))]))


def test_join_benchmark_shape_properties(plc):
    """BASELINE config 3 shape at 2^24 rows: 10 % of probe rows match exactly once."""
    import ctypes as C

    import torch

    from cudf_b200 import _lib

    n = 1 << 24
    rk = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(rk.data_ptr()), n, 0x5EED0002, 0, 0, 0, _lib.stream_arg(None)))
    sel = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(sel.data_ptr()), n, 0x5EED0005, 0, 2, n, _lib.stream_arg(None)))
    u = torch.empty(n, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(u.data_ptr()), n, 0x5EED0005, 1 << 40, 1, 0, _lib.stream_arg(None)))
    fresh = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(fresh.data_ptr()), n, 0x5EED0001, 1 << 41, 0, 0, _lib.stream_arg(None)))
    hit = u < 0.10
    lk = torch.where(hit, rk[sel], fresh)
    l, r = plc.join.inner_join(plc.Table([plc.Column.from_torch(lk)]), plc.Table([plc.Column.from_torch(rk)]), plc.NullEquality.EQUAL)
    li, ri = l.to_torch().long(), r.to_torch().long()
    assert li.numel() >= int(hit.sum())  # every selected probe row matches (>= because of 64-bit collisions ~ 0)
    assert bool((lk[li] == rk[ri]).all())
    assert abs(li.numel() / n - 0.10) < 0.005


# ---- groupby --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kdtype", [np.int8, np.int32, np.int64, np.uint16, np.float64])
@pytest.mark.parametrize("vdtype", [np.int8, np.int32, np.int64, np.uint32, np.float32, np.float64])
def test_groupby_random(cu, kdtype, vdtype):
    rng = np.random.default_rng(7)
    o = OracleImpl()
    for n, ng, nf in [(1, 1, 0.0), (1000, 13, 0.0), (50_000, 700, 0.15), (200_000, 100_000, 0.05)]:
        ng = min(ng, 100) if np.dtype(kdtype).itemsize == 1 else ng
        keys = [(rng.integers(0, ng, n).astype(kdtype), (rng.random(n) >= nf) if nf else None)]
        vals = rnd_col(rng, n, vdtype, nf)
        kinds = ["sum", "min", "max", "count", "count_all", "mean"]
        for inc in (False, True):
            gk, gr = sort_groups(*cu.groupby(keys, [(vals, kinds)], include_nulls=inc))
            ek, er = sort_groups(*o.groupby(keys, [(vals, kinds)], include_nulls=inc))
            assert_columns_equal(gk[0], ek[0], what="keys")
            for j, kind in enumerate(kinds):
                rtol = 0.0
                if np.dtype(vdtype).kind == "f" or kind == "mean":
                    rtol = F32_RTOL if np.dtype(vdtype) == np.float32 else F64_RTOL
                g, e = gr[0][j], er[0][j]
                assert np.asarray(g[0]).dtype == np.asarray(e[0]).dtype, f"{kind}: {np.asarray(g[0]).dtype} vs {np.asarray(e[0]).dtype}"
                if rtol and kind in ("sum", "mean"):
                    # sums of mixed-sign values: compare with an absolute floor scaled by the group's L1 mass
                    gm = np.ones(len(g[0]), bool) if g[1] is None else np.asarray(g[1])
                    em = np.ones(len(e[0]), bool) if e[1] is None else np.asarray(e[1])
                    assert np.array_equal(gm, em)
                    np.testing.assert_allclose(np.asarray(g[0], np.float64)[em], np.asarray(e[0], np.float64)[em], rtol=rtol, atol=rtol * 1e3)
                else:
                    assert_columns_equal(g, e, rtol=rtol, what=f"{kind} n={n}")


def test_groupby_multi_request_multi_key(cu):
    rng = np.random.default_rng(8)
    o = OracleImpl()
    n = 80_000
    keys = [rnd_col(rng, n, np.int32, 0.05, 0, 30), rnd_col(rng, n, np.int16, 0.0, 0, 4)]
    reqs = [(rnd_col(rng, n, np.float64, 0.3), ["sum", "mean"]), (rnd_col(rng, n, np.int32, 0.0), ["count", "max"]),
            (rnd_col(rng, n, np.int64, 0.5), ["count", "count_all"])]
    gk, gr = sort_groups(*cu.groupby(keys, reqs))
    ek, er = sort_groups(*o.groupby(keys, reqs))
    for a, b in zip(gk, ek):
        assert_columns_equal(a, b, what="keys")
    for q in range(len(reqs)):
        for j in range(len(reqs[q][1])):
            assert_columns_equal(gr[q][j], er[q][j], rtol=F64_RTOL, what=f"req {q} agg {j}")


def test_groupby_grows_table(cu):
    """More groups than the initial L2-sized table holds: exercises the overflow -> regrow path."""
    rng = np.random.default_rng(9)
    n = 3_000_000
    keys = [(rng.integers(0, 2_500_000, n).astype(np.int64), None)]
    vals = (rng.integers(0, 100, n).astype(np.int32), None)
    gk, gr = sort_groups(*cu.groupby(keys, [(vals, ["sum", "count"])]))
    uk, inv = np.unique(keys[0][0], return_inverse=True)
    assert np.array_equal(gk[0][0], uk)
    assert np.array_equal(gr[0][0][0], np.bincount(inv, weights=vals[0]).astype(np.int64))
    assert np.array_equal(gr[0][1][0], np.bincount(inv).astype(np.int32))


def test_groupby_errors(plc):
    k = plc.Table([plc.Column.from_numpy(np.array([1, 2, 3], np.int32))])
    gb = plc.groupby.GroupBy(k)
    with pytest.raises(RuntimeError):  # cudf::logic_error: size mismatch (groupby.cu:226-230)
        gb.aggregate([plc.groupby.GroupByRequest(plc.Column.from_numpy(np.array([1, 2], np.int32)), [plc.aggregation.sum()])])


@pytest.mark.parametrize("vdtype", [np.int16, np.int64, np.float64])
def test_groupby_scan_random(cu, vdtype):
    rng = np.random.default_rng(10)
    o = OracleImpl()
    for n, ng, nf in [(10, 3, 0.0), (5000, 40, 0.2), (100_000, 3000, 0.1)]:
        keys = [(rng.integers(0, ng, n).astype(np.int32), (rng.random(n) >= nf / 2) if nf else None)]
        vals = rnd_col(rng, n, vdtype, nf)
        kinds = ["sum", "min", "max", "count"]
        gk, gr = cu.groupby_scan(keys, [(vals, kinds)])
        ek, er = o.groupby_scan(keys, [(vals, kinds)])
        assert_columns_equal(gk[0], ek[0], what="scan keys")
        for j, kind in enumerate(kinds):
            assert_columns_equal(gr[0][j], er[0][j], rtol=F64_RTOL if np.dtype(vdtype).kind == "f" else 0.0, what=f"scan {kind} n={n}")


# ---- reduce / scan / segmented reduce ---------------------------------------------------------------------
ALL_NUM = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64]


@pytest.mark.parametrize("dtype", ALL_NUM + [np.bool_])
def test_reduce_random(cu, dtype):
    rng = np.random.default_rng(11)
    for n, nf in [(1, 0.0), (33, 0.3), (4097, 0.0), (1_000_003, 0.1)]:
        col = rnd_col(rng, n, dtype, nf, -100, 100)
        for kind in ("sum", "min", "max", "product", "mean"):
            outs = [dtype]
            if kind in ("sum", "product"):
                outs += [np.int64 if np.dtype(dtype).kind in "iub" else np.float64]
            if kind == "mean":
                outs = [np.float64, np.float32]
            if kind == "product" and n > 33:
                continue  # overflows / inf everywhere: nothing to pin
            for od in outs:
                g = cu.reduce(col, kind, od)
                e = ored.reduce(col[0], col[1], {"sum": 0, "product": 2, "min": 3, "max": 4, "mean": 10}[kind], od)
                assert g[1] == e[1], f"{kind} valid n={n}"
                if e[1]:
                    if np.dtype(od).kind == "f":
                        rtol = F32_RTOL if (np.dtype(od) == np.float32 or np.dtype(dtype) == np.float32) else F64_RTOL
                        np.testing.assert_allclose(float(g[0]), float(e[0]), rtol=rtol, atol=rtol * 1e3, err_msg=f"{kind} {np.dtype(dtype)}->{np.dtype(od)} n={n}")
                    else:
                        assert g[0] == e[0], f"{kind} {np.dtype(dtype)}->{np.dtype(od)} n={n}: {g[0]} vs {e[0]}"


@pytest.mark.parametrize("dtype", ALL_NUM)
def test_scan_random(cu, dtype):
    rng = np.random.default_rng(12)
    for n, nf in [(1, 0.0), (31, 0.0), (4096, 0.3), (4097, 0.0), (300_001, 0.05)]:
        col = rnd_col(rng, n, dtype, nf, -5, 5)
        for kind in ("sum", "min", "max"):
            for inclusive in (True, False):
                for include in (False, True):
                    g = cu.scan(col, kind, inclusive, include)
                    e = ored.scan(col[0], col[1], {"sum": 0, "min": 3, "max": 4}[kind], inclusive, 1 if include else 0)
                    rtol = 0.0
                    if np.dtype(dtype).kind == "f" and kind == "sum":
                        rtol = F32_RTOL if np.dtype(dtype) == np.float32 else F64_RTOL
                    if rtol:
                        gm = np.ones(n, bool) if g[1] is None else np.asarray(g[1])
                        em = np.ones(n, bool) if e[1] is None else np.asarray(e[1])
                        assert np.array_equal(gm, em)
                        np.testing.assert_allclose(np.asarray(g[0], np.float64)[em], np.asarray(e[0], np.float64)[em], rtol=rtol, atol=rtol * 100)
                    else:
                        assert_columns_equal(g, e, what=f"scan {kind} incl={inclusive} include={include} n={n} {np.dtype(dtype)}")
        for kind in ("count", "count_all"):
            g = cu.scan(col, kind, True, False)
            e = ored.scan(col[0], col[1], 5 if kind == "count" else 6, True, 0)
            assert_columns_equal(g, e, what=f"count scan {kind}")


@pytest.mark.parametrize("dtype", [np.int8, np.int32, np.int64, np.uint32, np.float32, np.float64])
def test_segmented_reduce_random(cu, dtype):
    rng = np.random.default_rng(13)
    n = 20_000
    for nf in (0.0, 0.2):
        col = rnd_col(rng, n, dtype, nf, -20, 20)
        cuts = np.sort(rng.integers(0, n, 300))
        offsets = np.concatenate([[0], cuts, [n]]).astype(np.int32)
        for kind in ("sum", "min", "max", "mean"):
            for include in (False, True):
                od = np.float64 if kind == "mean" else dtype
                g = cu.segmented_reduce(col, offsets, kind, od, include)
                e = ored.segmented_reduce(col[0], col[1], offsets, {"sum": 0, "min": 3, "max": 4, "mean": 10}[kind], od, 1 if include else 0)
                rtol = 0.0
                if np.dtype(od).kind == "f":
                    rtol = F32_RTOL if np.dtype(dtype) == np.float32 else F64_RTOL
                gm, em = np.asarray(g[1]), np.asarray(e[1])
                assert np.array_equal(gm, em), f"validity {kind} include={include}"
                if rtol:
                    np.testing.assert_allclose(np.asarray(g[0], np.float64)[em], np.asarray(e[0], np.float64)[em], rtol=rtol, atol=rtol * 100)
                else:
                    assert np.array_equal(np.asarray(g[0])[em], np.asarray(e[0])[em]), f"{kind} include={include}"


def test_gather_and_masks(plc):
    # gather_tests.cpp:44-250 semantics: negative wrap, NULLIFY, mask gather; bitmask_tests: counts, and, copy with offsets
    rng = np.random.default_rng(14)
    from oracle import bitmask as obm
    from oracle import sort as osort

    n = 10_000
    src = [rnd_col(rng, n, np.int64, 0.3), rnd_col(rng, n, np.int8, 0.0), rnd_col(rng, n, np.float32, 0.5)]
    gm = rng.integers(-n, n, 7777).astype(np.int32)
    t = plc.Table([plc.Column.from_numpy(v, m) for v, m in src])
    out = plc.copying.gather(t, plc.Column.from_numpy(gm), plc.OutOfBoundsPolicy.DONT_CHECK)
    exp = osort.gather(src, gm)
    for c, e in zip(out.columns(), exp):
        assert_columns_equal(c.to_numpy(), e, what="gather")
        assert c.null_count() == (0 if e[1] is None else int((~e[1]).sum()))
    gm2 = rng.integers(-2 * n, 2 * n, 5000).astype(np.int32)
    out = plc.copying.gather(t, plc.Column.from_numpy(gm2), plc.OutOfBoundsPolicy.NULLIFY)
    exp = osort.gather(src, gm2, nullify_oob=True)
    for c, e in zip(out.columns(), exp):
        assert_columns_equal(c.to_numpy(), e, what="gather nullify")
    # null masks
    cols = [plc.Column.from_numpy(v, m) for v, m in src]
    buf, nulls = plc.null_mask.bitmask_and(cols)
    ev, en = obm.bitmask_and([m for _, m in src], n)
    assert nulls == en and np.array_equal(buf.to_numpy_bits(n), ev)
    sl = cols[0].slice(37, 9000)
    cp = plc.null_mask.copy_bitmask(sl)
    assert np.array_equal(cp.to_numpy_bits(9000 - 37), src[0][1][37:9000])
    assert plc.null_mask.null_count(cols[0]._mask, 5, 7777) == int((~src[0][1][5:7777]).sum())
    m = plc.null_mask.create_null_mask(1000, plc.MaskState.ALL_VALID)
    plc.null_mask.set_null_mask(m.ptr, 13, 700, False)
    bits = m.to_numpy_bits(1000)
    assert bits[:13].all() and not bits[13:700].any() and bits[700:].all()
    assert plc.null_mask.bitmask_allocation_size_bytes(1000) == 128


def test_partition(plc):
    """b2_partition: stable range / hash partition (sharded-path bucket step)."""
    import torch

    from cudf_b200.sharded import CudaOps

    ops = CudaOps()
    rng = np.random.default_rng(15)
    for n in (1, 4095, 4096, 4097, 300_001):
        keys = rng.integers(-1000, 1000, n)
        pay = rng.integers(0, 1 << 30, n).astype(np.int32)
        kt, pt = torch.from_numpy(keys).cuda(), torch.from_numpy(pay).cuda()
        for P in (1, 2, 8, 13):
            spl = np.sort(rng.integers(-1000, 1000, P - 1))
            cols, offs = ops.partition([kt, pt], kt, 0, torch.from_numpy(spl).cuda() if P > 1 else None, P)
            b = np.searchsorted(spl, keys, side="right")
            order = np.argsort(b, kind="stable")
            assert offs == np.concatenate([[0], np.cumsum(np.bincount(b, minlength=P))]).tolist()
            assert np.array_equal(cols[0].cpu().numpy(), keys[order]) and np.array_equal(cols[1].cpu().numpy(), pay[order])
            cols, offs = ops.partition([kt, pt], kt, 1, None, P)
            got_k, got_p = cols[0].cpu().numpy(), cols[1].cpu().numpy()
            # hash mode: same multiset, every bucket holds whole key classes, stable inside a bucket
            assert offs[-1] == n and np.array_equal(np.sort(got_k), np.sort(keys))
            seen = {}
            for bi in range(P):
                for k in np.unique(got_k[offs[bi]:offs[bi + 1]]):
                    assert seen.setdefault(int(k), bi) == bi
    # nullable payload goes through the gather fallback
    n = 10_000
    keys = rng.integers(0, 100, n)
    vals = rng.standard_normal(n)
    valid = rng.random(n) < 0.5
    tbl = plc.Table([plc.Column.from_numpy(keys), plc.Column.from_numpy(vals, valid)])
    import ctypes as C

    from cudf_b200 import _lib

    out = C.c_void_p()
    offs = (C.c_int32 * 5)()
    tv, kv = tbl._view(), tbl.columns()[0]._view()
    _lib.check(_lib.lib.b2_partition(C.byref(tv), C.byref(kv), 1, None, 4, _lib.stream_arg(None), C.byref(out), offs))
    res = plc.Table._from_handle(out.value)
    gk = res.columns()[0].to_numpy()[0]
    gv, gm = res.columns()[1].to_numpy()
    assert np.array_equal(np.sort(gk), np.sort(keys)) and int(gm.sum()) == int(valid.sum())
    assert res.columns()[1].null_count() == int((~valid).sum())


def test_join_hash_table_small(cu):
    """Inner / left / full joins on the hash table: one key column of four types (int32 with nulls) at three size ratios
    under both null equalities, and a packed int32 + int16 key."""
    rng = np.random.default_rng(77)
    for dtype in (np.int64, np.int32, np.float64, np.int8):
        for nl, nr in [(1000, 700), (50_000, 20_000), (300, 90_000)]:
            hi = 100 if dtype == np.int8 else 5000
            l = [(rng.integers(0, hi, nl).astype(dtype), rng.random(nl) < 0.9 if dtype == np.int32 else None)]
            r = [(rng.integers(0, hi, nr).astype(dtype), None)]
            for kind in ("inner_join", "left_join", "full_join"):
                for ne in (0, 1):
                    got = getattr(cu, kind)(l, r, ne)
                    exp = getattr(ojoin, kind)(l, r, ne)
                    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (dtype, nl, nr, kind, ne)
    l = [(rng.integers(0, 50, 20000).astype(np.int32), None), (rng.integers(0, 9, 20000).astype(np.int16), None)]
    r = [(rng.integers(0, 50, 9000).astype(np.int32), None), (rng.integers(0, 9, 9000).astype(np.int16), None)]
    got = cu.inner_join(l, r)
    exp = ojoin.inner_join(l, r)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])

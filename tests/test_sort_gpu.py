"""GPU parity: CUDA radix sort (through the C ABI / pylibcudf-named shim) vs golden vectors and the oracle."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import sort as osort
from tests.golden import sort_cases as G
from tests.helpers import ALL_DTYPES, assert_columns_equal, make_col, to_plc_column, to_plc_table

pytestmark = pytest.mark.gpu

TYPED = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64]
SIZES = [1, 2, 31, 32, 33, 64, 65, 1000, 6143, 6144, 6145, 100_003, (1 << 20) + 7]


def rand_values(rng, n, dtype, small=False):
    dt = np.dtype(dtype)
    if dt == np.bool_:
        return rng.integers(0, 2, n).astype(bool)
    if dt.kind == "f":
        v = rng.standard_normal(n).astype(dt) * (3 if small else 1e6)
        if small:
            v = np.round(v)
        if n > 8:
            pos = rng.integers(0, n, max(1, n // 16))
            v[pos] = rng.choice(np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0], dtype=dt), len(pos))
        return v
    info = np.iinfo(dt)
    if small:
        return rng.integers(max(info.min, -5), min(info.max, 5) + 1, n).astype(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


@pytest.mark.parametrize("case", G.SORTED_ORDER_CASES, ids=lambda c: c["name"])
@pytest.mark.parametrize("dtype", TYPED + [np.bool_])
def test_sorted_order_golden(plc, case, dtype):
    if dtype == np.bool_ and case["skip_bool"]:
        pytest.skip("not pinned by the reference for bool")
    cols = [make_col(v, dtype if k == "T" else np.int32) for v, k in case["cols"]]
    tbl = to_plc_table(plc, cols)
    for fn in (plc.sorting.sorted_order, plc.sorting.stable_sorted_order):
        got = fn(tbl, case["order"], case["nulls"])
        assert got.type().id() == plc.TypeId.INT32 and got.null_count() == 0
        assert got.to_numpy()[0].tolist() == case["expected"], case["cite"]
    # run_sort_test (sort_test.cpp:25-41): sort and sort_by_key give the gathered table
    exp_tbl = osort.gather(cols, case["expected"])
    for res in (plc.sorting.sort(tbl, case["order"], case["nulls"]), plc.sorting.sort_by_key(tbl, tbl, case["order"], case["nulls"])):
        for c, e in zip(res.columns(), exp_tbl):
            assert_columns_equal(c.to_numpy(), e, what=case["name"])


def test_inf_nan_golden(plc):
    col = (np.array(G.INF_NAN["values"], dtype=np.float64), None)
    tbl = to_plc_table(plc, [col])
    assert plc.sorting.sorted_order(tbl, [], []).to_numpy()[0].tolist() == G.INF_NAN["expected"]
    assert plc.sorting.stable_sorted_order(tbl, [], []).to_numpy()[0].tolist() == G.INF_NAN["expected"]
    assert plc.sorting.sorted_order(tbl, [1], []).to_numpy()[0].tolist() == osort.sorted_order([col], [1]).tolist()


@pytest.mark.parametrize("dtype", TYPED)
def test_sliced_columns_golden(plc, dtype):
    c1 = make_col(G.SLICED["col1"], np.int32)
    c2 = make_col(G.SLICED["col2"], dtype)
    p1, p2 = to_plc_column(plc, c1), to_plc_column(plc, c2)
    got = plc.sorting.sorted_order(plc.Table([p1, p2]), [0, 0], [])
    assert got.to_numpy()[0].tolist() == G.SLICED["expected"]
    k = G.SLICED["split"]
    s1 = p1.slice(k, p1.size())
    got = plc.sorting.sorted_order(plc.Table([s1, s1]), [0, 0], [])
    assert got.to_numpy()[0].tolist() == G.SLICED["expected_sliced"]


def test_errors(plc):
    c = to_plc_column(plc, make_col([1, 2, 3], np.int32))
    t2 = plc.Table([c, c])
    with pytest.raises(RuntimeError):  # cudf::logic_error (sort_test.cpp:667-698)
        plc.sorting.sorted_order(t2, [0], [])
    with pytest.raises(RuntimeError):
        plc.sorting.sorted_order(t2, [0, 0], [1])
    with pytest.raises(RuntimeError):  # sort_test.cpp:962-978
        plc.sorting.sort_by_key(plc.Table([to_plc_column(plc, make_col([1, 2], np.int32))]), plc.Table([c]), [], [])
    empty = plc.Table([plc.Column.from_numpy(np.empty(0, np.int32))])
    got = plc.sorting.sorted_order(empty, [], [])
    assert got.size() == 0 and got.type().id() == plc.TypeId.INT32
    assert plc.sorting.sort(empty, [], []).num_rows() == 0


@pytest.mark.parametrize("dtype", ALL_DTYPES)
@pytest.mark.parametrize("order", [0, 1])
def test_single_column_random(plc, dtype, order):
    rng = np.random.default_rng(1234 + order)
    for n in SIZES:
        for small in (False, True):
            v = rand_values(rng, n, dtype, small)
            col = (v, None)
            got = plc.sorting.sorted_order(to_plc_table(plc, [col]), [order], []).to_numpy()[0]
            exp = osort.sorted_order([col], [order])
            assert np.array_equal(got, exp), f"{np.dtype(dtype)} n={n} small={small} order={order}"


@pytest.mark.parametrize("dtype", [np.int8, np.int32, np.int64, np.uint16, np.uint64, np.float32, np.float64, np.bool_])
@pytest.mark.parametrize("order,nprec", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_single_column_nullable_random(plc, dtype, order, nprec):
    rng = np.random.default_rng(99)
    for n in [1, 33, 2047, 2048, 2049, 70_001, (1 << 20) + 5]:
        v = rand_values(rng, n, dtype, small=(n % 2 == 1))
        valid = rng.random(n) < 0.7
        if n > 1:
            valid[rng.integers(0, n)] = False
        col = (v, valid)
        got = plc.sorting.sorted_order(to_plc_table(plc, [col]), [order], [nprec]).to_numpy()[0]
        exp = osort.sorted_order([col], [order], [nprec])
        assert np.array_equal(got, exp), f"{np.dtype(dtype)} n={n}"
    # all-null and sliced (offset not a multiple of 32)
    n = 5000
    v = rand_values(rng, n, dtype)
    valid = rng.random(n) < 0.5
    full = to_plc_column(plc, (v, valid))
    for b, e in [(0, n), (7, n - 3), (33, 4097), (100, 101)]:
        sl = full.slice(b, e)
        got = plc.sorting.sorted_order(plc.Table([sl]), [order], [nprec]).to_numpy()[0]
        exp = osort.sorted_order([(v[b:e], valid[b:e])], [order], [nprec])
        assert np.array_equal(got, exp), f"slice {b}:{e}"
    allnull = (v, np.zeros(n, bool))
    got = plc.sorting.sorted_order(to_plc_table(plc, [allnull]), [order], [nprec]).to_numpy()[0]
    assert np.array_equal(got, np.arange(n))


@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint32, np.uint64, np.bool_])
@pytest.mark.parametrize("order", [0, 1])
def test_keys_only_sort(plc, dtype, order):
    """cudf::sort single non-null column fast path (sort_radix.cu:151-161)."""
    rng = np.random.default_rng(5)
    for n in [1, 100, 6144, 250_001]:
        v = rand_values(rng, n, dtype, small=(n == 100))
        got = plc.sorting.sort(to_plc_table(plc, [(v, None)]), [order], []).columns()[0].to_numpy()[0]
        exp = np.sort(v.astype(np.uint8) if v.dtype == np.bool_ else v, kind="stable")
        if order:
            exp = exp[::-1]
        assert np.array_equal(got.astype(exp.dtype), exp)


def test_multi_column_random(plc):
    rng = np.random.default_rng(7)
    for n in [10, 1000, 50_001]:
        cols = [
            (rng.integers(0, 4, n).astype(np.int32), rng.random(n) < 0.9),
            (rand_values(rng, n, np.float64, small=True), None),
            (rng.integers(0, 3, n).astype(np.int8), rng.random(n) < 0.8),
            (rng.integers(-2, 2, n).astype(np.int64), None),
        ]
        for order, nprec in [([0, 1, 0, 1], [1, 0, 0, 1]), ([1, 1, 1, 0], [0, 0, 1, 1]), ([0, 0, 0, 0], [])]:
            got = plc.sorting.stable_sorted_order(to_plc_table(plc, cols), order, nprec).to_numpy()[0]
            exp = osort.sorted_order(cols, order, nprec)
            assert np.array_equal(got, exp), f"n={n} order={order}"


def test_sort_by_key_payload(plc):
    rng = np.random.default_rng(11)
    n = 100_000
    keys = [(rng.integers(-1000, 1000, n).astype(np.int64), None)]
    vals = [(rng.standard_normal(n), rng.random(n) < 0.5), (rng.integers(0, 100, n).astype(np.int16), None), keys[0]]
    got = plc.sorting.sort_by_key(to_plc_table(plc, vals), to_plc_table(plc, keys), [0], [])
    exp = osort.sort_by_key(vals, keys, [0])
    for c, e in zip(got.columns(), exp):
        assert_columns_equal(c.to_numpy(), e)
    assert got.columns()[0].null_count() == int((~vals[0][1]).sum())


def test_sort_by_key_carry_payload(plc):
    """One non-null payload column carried through the passes (no row ids, no gather) for key / value type pairs at the
    6144-row tile edge."""
    rng = np.random.default_rng(5)
    for n in (1, 33, 6144, 6145, 200_003):
        for kdt in (np.int64, np.int32, np.uint16, np.float64):
            for vdt in (np.int64, np.float64, np.int32, np.float32):
                keys = (rng.standard_normal(n) * 50).astype(kdt)
                vals = rng.integers(0, 1 << 30, n).astype(vdt)
                for order in ((0, 1) if np.dtype(kdt).kind != "f" else (0,)):
                    got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([plc.Column.from_numpy(keys)]), [order], [])
                    exp = osort.sort_by_key([(vals, None)], [(keys, None)], [order])[0][0]
                    assert np.array_equal(got.columns()[0].to_numpy()[0], exp), (n, kdt, vdt, order)


def test_sort_by_key_aliased_column(plc):
    """sort_by_key(T, T): the values and the keys are the same column."""
    rng = np.random.default_rng(11)
    for n in (1, 33, 6145, 200_003, 3_000_001):
        for dt in (np.int64, np.int32, np.uint16, np.int8, np.uint64):
            keys = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
            for order in (0, 1):
                c = plc.Column.from_numpy(keys)
                got = plc.sorting.sort_by_key(plc.Table([c]), plc.Table([c]), [order], []).columns()[0].to_numpy()[0]
                exp = np.sort(keys, kind="stable")
                if order == 1:
                    exp = exp[::-1]
                assert np.array_equal(got, exp), (n, dt, order)


def test_sortedness_property_large(plc):
    """Size-independent properties at 2^26 rows: permutation, non-decreasing keys, stable ties."""
    import torch

    n = 1 << 26
    from cudf_b200 import _lib
    import ctypes as C

    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(keys.data_ptr()), n, 0x5EED0001, 0, 2, 1 << 20, _lib.stream_arg(None)))
    col = plc.Column.from_torch(keys)
    order = plc.sorting.sorted_order(plc.Table([col]), [0], []).to_torch().long()
    sk = keys[order]
    assert bool((sk[1:] >= sk[:-1]).all())
    ties = sk[1:] == sk[:-1]
    assert bool((order[1:][ties] > order[:-1][ties]).all())
    assert int(order.sum()) == n * (n - 1) // 2
    assert int(torch.bincount(order, minlength=n).max()) == 1


def test_portion_path():
    """N > portion limit: per-portion digit bases (exercised with a tiny portion via B2_SORT_PORTION)."""
    code = r"""
import numpy as np, sys
sys.path.insert(0, '.')
import cudf_b200.pylibcudf as plc
from oracle import sort as osort
rng = np.random.default_rng(3)
for n in [50_000, 200_003]:
    for dt in (np.int64, np.int16, np.float32):
        v = (rng.standard_normal(n) * 100).astype(dt)
        for order in (0, 1):
            got = plc.sorting.sorted_order(plc.Table([plc.Column.from_numpy(v)]), [order], []).to_numpy()[0]
            assert np.array_equal(got, osort.sorted_order([(v, None)], [order])), (n, dt, order)
        got = plc.sorting.sort(plc.Table([plc.Column.from_numpy(v)]), [0], []).columns()[0].to_numpy()[0]
        assert np.array_equal(got, np.sort(v))
print('PORTION_OK')
"""
    env = dict(os.environ, B2_SORT_PORTION="20000")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=os.path.dirname(os.path.dirname(__file__)))
    assert "PORTION_OK" in r.stdout, r.stdout + r.stderr

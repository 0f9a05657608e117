"""tests/int_ref.py on hand-computed answers, and the numpy oracle (oracle/reduce.py, oracle/groupby.py) against it on the
generated full-range cases of tests/test_integer_extremes_gpu.py."""
import math

import numpy as np
import pytest

from oracle import groupby as ogb
from oracle import reduce as ored
from tests import exact_ref as X
from tests import int_ref as R
from tests.impls import KINDS
from tests.test_integer_extremes_gpu import GB_SIZES, INTS, TYPES, gb_input, gen, inits, m2_small, out_types, same

T63 = 2 ** 63


def test_conversions_round_once():
    assert R.to_float(2 ** 53 + 1, np.float64) == 2.0 ** 53            # a tie: to even
    assert R.to_float(2 ** 53 + 3, np.float64) == 2.0 ** 53 + 4
    assert R.to_float(2 ** 24 + 1, np.float32) == 2.0 ** 24
    assert R.to_float(T63 - 1, np.float32) == 2.0 ** 63
    assert R.to_float(-(T63), np.float64) == -(2.0 ** 63)
    # int -> double -> float32 would round to a float32 tie and then to even (2^60); one rounding goes up
    x = 2 ** 60 + 2 ** 36 + 1
    assert float(np.float32(float(x))) == 2.0 ** 60
    assert R.to_float(x, np.float32) == 2.0 ** 60 + 2.0 ** 37
    assert R.wrap(T63, np.int64) == -T63 and R.wrap(-1, np.uint64) == 2 ** 64 - 1 and R.wrap(300, np.int8) == 44


def test_reduce_known_answers():
    u64 = np.array([T63, 1], np.uint64)
    assert R.reduce(u64, None, R.SUM, np.float64) == (-9.223372036854776e18, True)   # int64 accumulator: -2^63 + 1
    assert R.reduce(u64, None, R.SUM, np.float32) == (-9.223372036854776e18, True)
    assert R.reduce(u64, None, R.SUM, np.uint64) == (T63 + 1, True)
    assert R.reduce(u64, None, R.SUM, np.int64) == (-T63 + 1, True)
    u8 = np.array([200, 100], np.uint8)
    assert R.reduce(u8, None, R.SUM, np.uint8) == (44, True)
    assert R.reduce(u8, None, R.SUM, np.int64) == (300, True)
    assert R.reduce(u8, None, R.SUM, np.float32) == (300.0, True)
    assert R.reduce(np.array([2 ** 32, 2 ** 31], np.uint64), None, R.PRODUCT, np.float64) == (-9.223372036854776e18, True)
    assert R.reduce(np.array([2 ** 31, 2], np.uint32), None, R.PRODUCT, np.float64) == (4294967296.0, True)
    assert R.reduce(np.array([2 ** 31, 2], np.uint32), None, R.PRODUCT, np.uint32) == (0, True)
    assert R.reduce(np.array([127, 1], np.int8), None, R.SUM, np.int8) == (-128, True)
    assert R.reduce(np.array([127, 1], np.int8), None, R.SUM, np.int64) == (128, True)
    assert R.reduce(np.array([1], np.uint64), None, R.SUM, np.float64, (2 ** 64 - 1, True)) == (0.0, True)
    assert R.reduce(np.array([1], np.uint64), None, R.SUM, np.uint64, (2 ** 64 - 1, True)) == (0, True)
    assert R.reduce(np.array([5], np.int32), None, R.SUM, np.int32, (1, False))[1] is False  # a null initial value: a null result
    assert R.reduce(np.array([5], np.int32), [False], R.SUM, np.int32) == (None, False)
    assert R.reduce(np.array([3, -7, 2], np.int64), [True, False, True], R.MIN, np.int64) == (2, True)
    assert R.reduce(np.array([True] * 300), None, R.SUM, np.bool_) == (True, True)
    assert R.reduce(np.array([True] * 300), None, R.SUM, np.int64) == (300, True)
    assert R.mean_terms(np.array([2 ** 53 + 1, 1], np.int64), None, np.float64) == [2.0 ** 53, 1.0]


def test_scan_and_segmented_known_answers():
    assert R.scan(np.array([200, 100, 0], np.uint8), None, R.SUM) == ([200, 44, 44], None)
    assert R.scan(np.array([200, 100, 0], np.uint8), None, R.SUM, inclusive=False) == ([0, 200, 44], None)
    assert R.scan(np.array([5, 1, 3], np.int8), [True, False, True], R.MIN, True, True) == ([5, None, None], [True, False, False])
    assert R.scan(np.array([5, 1, 3], np.int8), [True, False, True], R.MAX, False, False) == ([-128, None, 5], [True, False, True])
    assert R.scan(np.array([True] * 300), None, R.SUM)[0][-1] is True
    v = np.array([T63, 1, 7, 2 ** 64 - 1], np.uint64)
    assert R.segmented_reduce(v, None, [0, 2, 2, 4], R.SUM, np.float64) == [(-9.223372036854776e18, True), (None, False), (6.0, True)]
    assert R.segmented_reduce(v, [True, True, False, True], [0, 2, 4], R.MAX, np.uint64, True) == [(T63, True), (None, False)]
    assert R.segmented_reduce(v, None, [0, 0, 1], R.SUM, np.uint64, init=(5, True)) == [(5, True), (T63 + 5, True)]


def test_groupby_known_answers():
    i64 = np.array([T63 - 1, T63 - 1, 3], np.int64)
    assert R.group_agg(i64, None, [0, 1], "sum") == (-2, True)
    assert R.group_agg(i64, None, [0, 1], "mean") == (-1.0, True)
    assert R.group_agg(np.array([T63], np.uint64), None, [0], "mean") == (-9.223372036854776e18, True)
    assert R.group_agg(np.array([T63 + 5], np.uint64), None, [0], "max") == (T63 + 5, True)
    assert R.group_agg(np.array([2 ** 32 + 1], np.uint64), None, [0], "sum_of_squares") == (2 ** 33 + 1, True)
    assert R.group_agg(i64, [False, False, True], [0, 1], "min") == (None, False)
    assert R.group_agg(i64, [False, False, True], [0, 1], "count") == (0, True)
    assert R.group_agg(i64, None, [0, 1, 2], "argmax") == ([0, 1], True)
    assert R.group_scan(np.array([T63 - 1, 1, 4], np.int64), [True, True, False], [0, 1, 2], "sum") == [T63 - 1, -T63, None]
    # a single UINT64 value at or above 2^63: the MEAN is that value minus 2^64, so the sort path's M2 is 2^128
    assert m2_small(np.array([T63], np.uint64), None, [0]) == 2.0 ** 128


# ---- the oracle against the reference ----------------------------------------------------------------------------------
def _mean_ok(got, xs, od, k):
    terms = [R.to_float(a, od) for a in xs]
    ex = X.exact_sum(terms)
    u = X.unit_roundoff(od)
    X.check(got, ex / len(xs), X.mean_bound(k, u, X.abs_sum(terms), ex, len(xs), u))


@pytest.mark.parametrize("dt", TYPES, ids=lambda d: np.dtype(d).name)
def test_oracle_reduce_agrees(dt):
    rng = np.random.default_rng(30 + np.dtype(dt).num)
    for n, pattern in ((1, "mixed"), (31, "wrap"), (300, "product"), (4097, "mixed")):
        v = gen(rng, dt, n, pattern)
        for m in (None, rng.random(n) >= 0.3):
            xs = R.ints(v, m)
            for kind in ("sum", "product", "min", "max"):
                for od in (out_types(dt) if kind in ("sum", "product") else [v.dtype]):
                    for init in inits(rng, dt):
                        oinit = None if init is None else (np.asarray(init[0]).astype(dt)[()], init[1])
                        got, ok = ored.reduce(v, m, KINDS[kind], od, oinit)
                        exp, eok = R.reduce_ints(xs, dt, kind, od, init)
                        assert ok == eok
                        assert not eok or same(got, exp), f"{np.dtype(dt)} n={n} {kind} -> {np.dtype(od)} init={init}: {got!r} vs {exp!r}"
            for od in (np.float64, np.float32):
                got, ok = ored.reduce(v, m, KINDS["mean"], od)
                if xs:
                    _mean_ok(got, xs, od, n)
            for kind in ("sum", "product", "min", "max"):
                for inclusive in (True, False):
                    for inc in (False, True):
                        gv, gm = ored.scan(v, m, KINDS[kind], inclusive, 1 if inc else 0)
                        ev, em = R.scan(v, m, kind, inclusive, inc)
                        assert (gm is None) == (em is None) and (em is None or np.array_equal(gm, em))
                        assert all(e is None or same(g, e) for g, e in zip(gv.tolist(), ev)), f"scan {kind} {inclusive} {inc}"


@pytest.mark.parametrize("dt", TYPES, ids=lambda d: np.dtype(d).name)
def test_oracle_segmented_reduce_agrees(dt):
    rng = np.random.default_rng(40 + np.dtype(dt).num)
    offsets = [0, 0, 1, 32, 65, 1065, 1066, 1066, 1099]
    v = gen(rng, dt, offsets[-1], "mixed")
    for m in (None, rng.random(len(v)) >= 0.3):
        for kind in ("sum", "product", "min", "max"):
            for od in (out_types(dt) if kind in ("sum", "product") else [v.dtype]):
                for inc in (False, True):
                    for init in inits(rng, dt):
                        oinit = None if init is None else (np.asarray(init[0]).astype(dt)[()], init[1])
                        gv, gm = ored.segmented_reduce(v, m, offsets, KINDS[kind], od, 1 if inc else 0, oinit)
                        exp = R.segmented_reduce(v, m, offsets, kind, od, inc, init)
                        for g, (e, eok) in enumerate(exp):
                            assert bool(gm[g]) == eok
                            assert not eok or same(gv[g].item(), e), f"{np.dtype(dt)} {kind} -> {np.dtype(od)} seg {g}: {gv[g]!r} vs {e!r}"


@pytest.mark.parametrize("dt", TYPES, ids=lambda d: np.dtype(d).name)
def test_oracle_groupby_agrees(dt):
    rng = np.random.default_rng(50 + np.dtype(dt).num)
    kinds = ["sum", "product", "min", "max", "mean", "sum_of_squares", "count", "argmin", "argmax"]
    for pattern in ("mixed", "wrap", "product"):
        keys, vals, vm = gb_input(rng, dt, pattern, GB_SIZES)
        for m in (None, vm):
            for sort_path in (False, True):
                ks = kinds + (["m2"] if sort_path else [])
                (okeys,), (res,) = ogb.aggregate([(keys, None)], [((vals, m), [KINDS[k] for k in ks])], sort_path=sort_path)
                groups = R.group_rows(keys)
                for g, key in enumerate(okeys[0].tolist()):
                    rows = groups[key]
                    for kind, (ov, om) in zip(ks, res):
                        w = f"{np.dtype(dt)} {pattern} sort_path={sort_path} key={key} {kind}"
                        if kind == "m2":
                            nv = len(rows) if m is None else int(m[rows].sum())
                            assert nv > 2 or same(ov[g].item(), m2_small(vals, m, rows)), f"{w}: {ov[g]!r}"
                            continue
                        exp, eok = R.group_agg(vals, m, rows, kind)
                        ok = True if om is None else bool(om[g])
                        if kind in ("count", "count_all"):
                            assert ov[g] == exp, w
                            continue
                        assert ok == eok, w
                        if eok:
                            assert (ov[g] in exp) if kind.startswith("arg") else same(ov[g].item(), exp), f"{w}: {ov[g]!r} vs {exp!r}"
        if dt != np.bool_:
            (okeys,), (res,) = ogb.scan([(keys, None)], [((vals, vm), [KINDS[k] for k in ("sum", "min", "max", "count")])])
            pos = 0
            for key, rows in sorted(R.group_rows(keys).items()):
                for kind, (ov, om) in zip(("sum", "min", "max", "count"), res):
                    for j, e in enumerate(R.group_scan(vals, vm, rows, kind)):
                        assert e is None or same(ov[pos + j].item(), e), f"grouped scan {kind} key={key}"
                pos += len(rows)

"""Stream compaction (apply_boolean_mask / apply_deletion_mask, drop_nulls, drop_nans, unique, distinct, stable_distinct,
distinct_indices) through the C ABI and the ctypes twin, against the reference's known answers (tests/golden) and the
numpy oracle. Filters, unique and stable_distinct must match in order; distinct is compared after canonical sorting."""
import itertools

import numpy as np
import pytest

from oracle import stream_compaction as osc
from tests.golden.stream_compaction_cases import CASES
from tests.helpers import assert_columns_equal, make_col
from tests.test_stream_compaction_oracle import check_case, run_case

pytestmark = pytest.mark.gpu

TILE = 8192  # rows per compaction tile (stream_compaction.cu CP_TILE)
SIZES = (0, 1, 31, TILE - 1, TILE, TILE + 1, 3 * TILE + 77)
DTYPES = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64, np.bool_]


def _table(plc, cols):
    return plc.Table([plc.Column.from_numpy(v, m) for v, m in cols])


def _got(t):
    return [c.to_numpy() for c in t.columns()]


def _check(got, exp, what):
    assert len(got) == len(exp), what
    for j, (g, e) in enumerate(zip(got, exp)):
        assert_columns_equal(g, e, what=f"{what} col {j}")


def _rand_col(rng, n, dt, null_frac=0.0, card=None):
    dt = np.dtype(dt)
    if dt == np.bool_:
        v = rng.random(n) < 0.5
    elif dt.kind == "f":
        v = (rng.integers(0, card or 1000, n) - (card or 1000) // 2).astype(dt) * dt.type(0.5)
        v[rng.random(n) < 0.05] = np.nan
        v[rng.random(n) < 0.05] = -0.0
    else:
        info = np.iinfo(dt)
        hi = min(int(info.max), card or int(info.max))
        v = rng.integers(max(int(info.min), -hi) if card else int(info.min), hi, n, endpoint=True, dtype=np.int64 if dt != np.uint64 else np.uint64).astype(dt)
    m = (rng.random(n) >= null_frac) if null_frac else None
    return v, m


def _case_cols(spec):
    return [make_col(vals, dt) for vals, dt in spec]


class _Ops:
    """The binding's stream_compaction with the golden cases' integer enums."""

    def __init__(self, plc):
        self.sc, self.plc = plc.stream_compaction, plc

    def __getattr__(self, name):
        return getattr(self.sc, name)

    def unique(self, t, keys, keep, ne):
        return self.sc.unique(t, keys, self.sc.DuplicateKeepOption(keep), self.plc.NullEquality(ne))

    def distinct(self, t, keys, keep, ne, nan):
        return self.sc.distinct(t, keys, self.sc.DuplicateKeepOption(keep), self.plc.NullEquality(ne), self.plc.NanEquality(nan))

    def stable_distinct(self, t, keys, keep, ne, nan):
        return self.sc.stable_distinct(t, keys, self.sc.DuplicateKeepOption(keep), self.plc.NullEquality(ne), self.plc.NanEquality(nan))


@pytest.mark.parametrize("case", CASES, ids=[c["src"] for c in CASES])
def test_golden(plc, case):
    got, exp = run_case(case, _Ops(plc), lambda cols: _table(plc, cols), lambda m: plc.Column.from_numpy(*m))
    check_case(case, _got(got), exp)


@pytest.mark.parametrize("dt", DTYPES, ids=[np.dtype(d).name for d in DTYPES])
def test_boolean_and_deletion_mask(plc, dt):
    rng = np.random.default_rng(11)
    sc = plc.stream_compaction
    for n in SIZES:
        cols = [_rand_col(rng, n, dt, 0.3), _rand_col(rng, n, np.int64)]
        for frac, mask_nulls in ((0.5, 0.0), (0.5, 0.2), (1.0, 0.0), (0.0, 0.0), (0.5, 1.0)):
            mv = rng.random(n) < frac
            mm = (rng.random(n) >= mask_nulls) if mask_nulls else None
            t, mcol = _table(plc, cols), plc.Column.from_numpy(mv, mm)
            if n == 0:
                assert sc.apply_boolean_mask(t, mcol).num_rows() == 0
                continue
            _check(_got(sc.apply_boolean_mask(t, mcol)), osc.apply_boolean_mask(cols, (mv, mm)), (n, frac, mask_nulls))
            _check(_got(sc.apply_deletion_mask(t, mcol)), osc.apply_boolean_mask(cols, (mv, mm), True), (n, frac, mask_nulls, "del"))


def test_sliced_inputs(plc):
    """Views whose offsets are not multiples of 32 for the data, the mask's values and both validity masks."""
    rng = np.random.default_rng(12)
    sc = plc.stream_compaction
    n = 2 * TILE + 333
    v, vm = _rand_col(rng, n, np.float64, 0.3)
    mv, mm = rng.random(n) < 0.5, rng.random(n) >= 0.2
    for a, b in ((0, n), (5, n - 3), (37, 37 + TILE), (101, 1000)):
        col = plc.Column.from_numpy(v, vm).slice(a, b)
        mcol = plc.Column.from_numpy(mv, mm).slice(a, b)
        cols = [(v[a:b], vm[a:b])]
        _check(_got(sc.apply_boolean_mask(plc.Table([col]), mcol)), osc.apply_boolean_mask(cols, (mv[a:b], mm[a:b])), (a, b))
        _check(_got(sc.drop_nulls(plc.Table([col]), [0])), osc.drop_nulls(cols, [0]), (a, b, "nulls"))
        _check(_got(sc.drop_nans(plc.Table([col]), [0])), osc.drop_nans(cols, [0]), (a, b, "nans"))
        _check(_got(sc.unique(plc.Table([col]), [0], sc.DuplicateKeepOption.KEEP_NONE, plc.NullEquality.EQUAL)),
               osc.unique(cols, [0], osc.KEEP_NONE), (a, b, "unique"))
        _check(_got(sc.stable_distinct(plc.Table([col]), [0], sc.DuplicateKeepOption.KEEP_LAST, plc.NullEquality.EQUAL,
                                       plc.NanEquality.ALL_EQUAL)), osc.stable_distinct(cols, [0], osc.KEEP_LAST), (a, b, "distinct"))


def test_drop_nulls_and_nans(plc):
    rng = np.random.default_rng(13)
    sc = plc.stream_compaction
    for n in SIZES:
        cols = [_rand_col(rng, n, np.float32, 0.2), _rand_col(rng, n, np.int16, 0.4), _rand_col(rng, n, np.float64, 0.1),
                _rand_col(rng, n, np.int64)]
        t = _table(plc, cols)
        for keys in ([0], [0, 1], [1, 2, 3], [3], []):
            for thr in (None, 0, 1, 2, 3):
                _check(_got(sc.drop_nulls(t, keys, thr)), osc.drop_nulls(cols, keys, thr), (n, keys, thr))
        for keys in ([0], [0, 2], [2]):
            for thr in (None, 0, 1, 2):
                _check(_got(sc.drop_nans(t, keys, thr)), osc.drop_nans(cols, keys, thr), (n, keys, thr, "nan"))


KEEPS = (0, 1, 2, 3)


def _sorted_rows(cols):
    """Rows in a canonical order (for distinct, whose output order is unspecified)."""
    if not cols or len(cols[0][0]) == 0:
        return cols
    keys = []
    for v, m in cols:
        valid = np.ones(len(v), bool) if m is None else m
        x = np.where(valid, np.nan_to_num(np.asarray(v, dtype=np.float64), nan=np.inf), -np.inf)
        keys += [x, valid]
    order = np.lexsort(keys[::-1])
    return osc.gather(cols, order)


def _key_sets(plc):
    rng = np.random.default_rng(14)
    n = 2 * TILE + 501
    packed = [_rand_col(rng, n, np.int32, 0.1, card=40), _rand_col(rng, n, np.float32, 0.1, card=8)]   # 8 bytes
    wide = [_rand_col(rng, n, np.int64, 0.1, card=30), _rand_col(rng, n, np.float64, 0.1, card=6)]      # 16 bytes
    eight = [_rand_col(rng, n, dt, 0.05, card=2) for dt in (np.int8, np.uint8, np.bool_, np.int16, np.float32, np.int32,
                                                            np.float64, np.uint16)]
    # one-column packed keys of 1, 2 and 8 bytes (pack_row), the float64 one with NaN and -0
    singles = [[_rand_col(rng, n, dt, 0.1, card=6)] for dt in (np.int8, np.bool_, np.int16, np.float64)]
    for cols in (packed, wide, eight, *singles):  # sorted copies make unique remove real runs
        order = np.lexsort([np.nan_to_num(c[0].astype(np.float64)) for c in cols][::-1])
        yield [(v[order], None if m is None else m[order]) for v, m in cols] + [(np.arange(n, dtype=np.int64), None)]


def test_unique_all_options(plc):
    sc = plc.stream_compaction
    for cols in _key_sets(plc):
        t, keys = _table(plc, cols), list(range(len(cols) - 1))
        for keep, ne in itertools.product(KEEPS, (0, 1)):
            got = sc.unique(t, keys, sc.DuplicateKeepOption(keep), plc.NullEquality(ne))
            _check(_got(got), osc.unique(cols, keys, keep, ne), (len(keys), keep, ne))


def test_distinct_all_options(plc):
    sc = plc.stream_compaction
    for cols in _key_sets(plc):
        t, keys = _table(plc, cols), list(range(len(cols) - 1))
        kcols = cols[:-1]
        for keep, ne, nan in itertools.product(KEEPS, (0, 1), (0, 1)):
            args = (sc.DuplicateKeepOption(keep), plc.NullEquality(ne), plc.NanEquality(nan))
            stable = _got(sc.stable_distinct(t, keys, *args))
            unordered = _got(sc.distinct(t, keys, *args))
            exp = osc.stable_distinct(cols, keys, keep, ne, nan)
            what = (len(keys), keep, ne, nan)
            if keep == osc.KEEP_ANY:  # any row of each set: the key rows match as a set, the row ids are in order
                _check(_sorted_rows(stable[:-1]), _sorted_rows(exp[:-1]), what)
                assert np.all(np.diff(stable[-1][0]) > 0), what
            else:
                _check(stable, exp, what)
                idx = plc.stream_compaction.distinct_indices(_table(plc, kcols), *args).to_numpy()[0]
                assert np.array_equal(idx, osc.distinct_indices(kcols, keep, ne, nan)), what
            _check(_sorted_rows(unordered[:-1]), _sorted_rows(stable[:-1]), what)


def test_empty_and_degenerate(plc):
    sc = plc.stream_compaction
    K = sc.DuplicateKeepOption
    empty = plc.Table([plc.Column.from_numpy(np.zeros(0, np.int32))])
    none_ = plc.Table([])
    two = _table(plc, [(np.array([1, 1, 2], np.int64), None)])
    for fn in (sc.distinct, sc.stable_distinct):
        assert fn(none_, [5], K.KEEP_ANY, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL).num_columns() == 0
        assert fn(empty, [0], K.KEEP_ANY, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL).num_rows() == 0
        out = fn(two, [], K.KEEP_ANY, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL)
        assert out.num_rows() == 0 and out.num_columns() == 1
    assert sc.unique(two, [], K.KEEP_FIRST, plc.NullEquality.EQUAL).num_rows() == 0
    assert sc.distinct_indices(none_, K.KEEP_ANY, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL).size() == 0
    out = sc.apply_boolean_mask(two, plc.Column.from_numpy(np.zeros(0, np.bool_)))
    assert out.num_rows() == 0 and out.num_columns() == 1
    assert sc.drop_nulls(two, []).num_rows() == 3 and sc.drop_nans(two, []).num_rows() == 3
    # no nulls in the keys: a copy
    _check(_got(sc.drop_nulls(two, [0])), [(np.array([1, 1, 2]), None)], "copy")


def test_errors(plc):
    sc = plc.stream_compaction
    K = sc.DuplicateKeepOption
    t = _table(plc, [(np.arange(10, dtype=np.int64), None), (np.arange(10, dtype=np.float64), None)])
    with pytest.raises(RuntimeError):  # mask not BOOL8
        sc.apply_boolean_mask(t, plc.Column.from_numpy(np.ones(10, np.int8)))
    with pytest.raises(RuntimeError):  # size mismatch
        sc.apply_boolean_mask(t, plc.Column.from_numpy(np.ones(9, np.bool_)))
    with pytest.raises(RuntimeError):  # non-float key
        sc.drop_nans(t, [0])
    for bad in ([2], [-1]):
        with pytest.raises(IndexError):
            sc.drop_nulls(t, bad)
        with pytest.raises(IndexError):
            sc.unique(t, bad, K.KEEP_FIRST, plc.NullEquality.EQUAL)
        with pytest.raises(IndexError):
            sc.distinct(t, bad, K.KEEP_FIRST, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL)
    wide = plc.Table([plc.Column.from_numpy(np.arange(10, dtype=np.int32)) for _ in range(9)])
    with pytest.raises(ValueError):  # more than 8 key columns
        sc.distinct(wide, list(range(9)), K.KEEP_FIRST, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL)
    with pytest.raises(ValueError):
        sc.unique(t, [0], 7, plc.NullEquality.EQUAL)


def test_distinct_table_growth(plc):
    """More than 3e6 distinct keys: the L2-sized initial table (2^21 slots) overflows and grows x8 before the rerun."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs the device (too large for the emulator)")
    sc = plc.stream_compaction
    n, card = 8_000_000, 3_500_000
    rng = np.random.default_rng(15)
    k = rng.integers(0, card, n).astype(np.int64)
    t = plc.Table([plc.Column.from_numpy(k)])
    for keep in (sc.DuplicateKeepOption.KEEP_ANY, sc.DuplicateKeepOption.KEEP_FIRST):
        got = sc.distinct(t, [0], keep, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL).columns()[0].to_numpy()[0]
        assert np.array_equal(np.sort(got), np.unique(k))
    idx = sc.distinct_indices(t, sc.DuplicateKeepOption.KEEP_LAST, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL).to_numpy()[0]
    _, last = np.unique(k[::-1], return_index=True)
    assert np.array_equal(idx, np.sort(n - 1 - last).astype(np.int32))

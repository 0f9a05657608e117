"""Left semi / anti join (cudf::filtered_join; pylibcudf's FilteredJoin / left_semi_join / left_anti_join) through the C ABI
and the ctypes twin, against the reference's known answers (tests/golden/semi_anti_join_cases.py) and the oracle
(tests/semi_anti_oracle.py). Results are compared exactly, order included: both joins return ascending left indices.

The parity cases are functions of (plc, small): tests/test_emu_semi_anti_join.py runs them at reduced sizes on the kernel
emulator, this file at full size on the GPU."""
import numpy as np
import pytest

from tests import semi_anti_oracle as osa
from tests.golden.semi_anti_join_cases import CASES, INVALID_LOAD_FACTORS
from tests.test_semi_anti_join_oracle import case_cols

pytestmark = pytest.mark.gpu

TILE = 8192  # rows per compaction tile (compact.cuh CP_TILE)
INT_DTYPES = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
CHRONO = ["datetime64[D]", "datetime64[s]", "datetime64[ms]", "datetime64[us]", "datetime64[ns]",
          "timedelta64[D]", "timedelta64[s]", "timedelta64[ms]", "timedelta64[us]", "timedelta64[ns]"]


def _table(plc, cols):
    return plc.Table([plc.Column.from_numpy(v, m) for v, m in cols])


def _ids(col):
    assert col.type().id() == col.type().id().INT32
    return col.to_numpy()[0]


def check(plc, left, right, ne, what, load_factor=0.5, oracle_left=None, oracle_right=None):
    """FilteredJoin(right).semi_join / anti_join(left) equal the oracle exactly; returns the object for reuse."""
    fj = plc.join.FilteredJoin(_table(plc, right), plc.NullEquality(ne), load_factor)
    lt = _table(plc, left)
    ol, orr = oracle_left or left, oracle_right or right
    exp_s, exp_a = osa.left_semi_join(ol, orr, ne), osa.left_anti_join(ol, orr, ne)
    got_s, got_a = _ids(fj.semi_join(lt)), _ids(fj.anti_join(lt))
    assert np.array_equal(got_s, exp_s), (what, "semi", got_s[:20], exp_s[:20])
    assert np.array_equal(got_a, exp_a), (what, "anti", got_a[:20], exp_a[:20])
    return fj


def _rand(rng, n, dt, card, null_frac=0.0):
    dt = np.dtype(dt)
    if dt == np.bool_:
        v = rng.random(n) < 0.5
    elif dt.kind == "f":
        v = (rng.integers(0, card, n) - card // 2).astype(dt) * dt.type(0.5)
    else:
        info = np.iinfo(dt)
        lo = max(int(info.min), -(card // 2)) if info.min < 0 else 0
        v = (rng.integers(0, card, n) + lo).astype(dt)
    return v, ((rng.random(n) >= null_frac) if null_frac else None)


# ---- parity cases ------------------------------------------------------------------------------------------------------
def case_key_types(plc, small):
    """Every fixed-width type as a one-column key, with and without nulls: packed keys of 1, 2, 4 and 8 bytes."""
    rng = np.random.default_rng(31)
    n = 2000 if small else 3 * TILE + 77
    for dt in INT_DTYPES + [np.float32, np.float64, np.bool_]:
        for nf in (0.0, 0.2):
            left, right = [_rand(rng, n, dt, 60, nf)], [_rand(rng, n // 3 + 1, dt, 60, nf)]
            for ne in (0, 1):
                check(plc, left, right, ne, (np.dtype(dt).name, nf, ne))
    for name in CHRONO:
        dt = np.dtype(name)
        base = np.int32 if dt.itemsize == 4 else np.int64
        (lv, lm), (rv, rm) = _rand(rng, n, base, 80, 0.1), _rand(rng, n // 2, base, 80, 0.1)
        for ne in (0, 1):
            check(plc, [(lv.view(dt), lm)], [(rv.view(dt), rm)], ne, (name, ne),
                  oracle_left=[(lv, lm)], oracle_right=[(rv, rm)])


def _bits64(vals):
    return np.array(vals, np.uint64).view(np.float64)


def case_float_keys(plc, small):
    """NaNs with several payloads and both signs equal each other, -0.0 == +0.0, and +-inf."""
    rng = np.random.default_rng(32)
    n = 3000 if small else 50_000
    special64 = np.concatenate([_bits64([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF4000000000abc]),
                                [-0.0, 0.0, np.inf, -np.inf, 1.5, -2.25]])
    special32 = np.concatenate([np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFA00123], np.uint32).view(np.float32),
                                np.array([-0.0, 0.0, np.inf, -np.inf, 1.5, -2.25], np.float32)])
    for sp in (special64, special32):
        for right_sel in (slice(0, 1), slice(4, 5), slice(6, 7), slice(2, 6), slice(None)):
            left = [(rng.choice(sp, n), rng.random(n) >= 0.1)]
            right = [(sp[right_sel].copy(), None)]
            for ne in (0, 1):
                check(plc, left, right, ne, (sp.dtype.name, right_sel, ne))
        # a float key next to an int32 key: 12 bytes (wide) for float64, 8 bytes (packed) for float32
        left = [(rng.choice(sp, n), None), (rng.integers(0, 3, n).astype(np.int32), None)]
        right = [(rng.choice(sp, 50), None), (rng.integers(0, 3, 50).astype(np.int32), None)]
        check(plc, left, right, 0, (sp.dtype.name, "with int32"))


def case_nulls(plc, small):
    """Nulls on either side and on both, under EQUAL and UNEQUAL, and an all-null right table."""
    rng = np.random.default_rng(33)
    n = 2000 if small else 20_000
    for lf, rf in ((0.0, 0.3), (0.3, 0.0), (0.3, 0.3), (0.9, 0.5)):
        left, right = [_rand(rng, n, np.int64, 500, lf)], [_rand(rng, n // 4, np.int64, 500, rf)]
        for ne in (0, 1):
            check(plc, left, right, ne, ("nulls", lf, rf, ne))
    all_null = [(np.zeros(100, np.int64), np.zeros(100, bool))]
    left = [_rand(rng, n, np.int64, 50, 0.2)]
    for ne in (0, 1):
        check(plc, left, all_null, ne, ("all-null right", ne))
        check(plc, [(np.zeros(40, np.int64), np.zeros(40, bool))], all_null, ne, ("all-null both", ne))


def case_multi_column(plc, small):
    """Packed multi-column keys (int32 + int16 + uint8 = 7 bytes) and wide keys (two int64 columns, and 8 columns)."""
    rng = np.random.default_rng(34)
    n = 3000 if small else 2 * TILE + 501
    packed = [(np.int32, 6), (np.int16, 5), (np.uint8, 4)]
    two64 = [(np.int64, 30), (np.int64, 7)]
    eight = [(np.int8, 2), (np.uint8, 2), (np.bool_, 2), (np.int16, 2), (np.float32, 2), (np.int32, 2), (np.float64, 2),
             (np.uint16, 2)]
    for spec in (packed, two64, eight):
        for nf in (0.0, 0.05):
            left = [_rand(rng, n, dt, card, nf) for dt, card in spec]
            right = [_rand(rng, n // 5 + 3, dt, card, nf) for dt, card in spec]
            for ne in (0, 1):
                check(plc, left, right, ne, (len(spec), nf, ne))


def case_sliced(plc, small):
    """Views whose offsets are not multiples of 32, in the data and in the validity masks, on both sides."""
    rng = np.random.default_rng(35)
    n = 3000 if small else 2 * TILE + 333
    (v, m), (v2, m2) = _rand(rng, n, np.int64, 400, 0.2), _rand(rng, n, np.int32, 5, 0.1)
    (rv, rm), (rv2, rm2) = _rand(rng, n // 2, np.int64, 400, 0.2), _rand(rng, n // 2, np.int32, 5, 0.1)
    for (a, b), (c, d) in (((0, n), (3, n // 2)), ((5, n - 3), (37, 200)), ((37, n // 2 + 37), (1, n // 2 - 1))):
        for ne in (0, 1):
            for wide in (False, True):
                lcols = [plc.Column.from_numpy(v, m).slice(a, b)] + ([plc.Column.from_numpy(v2, m2).slice(a, b)] if wide else [])
                rcols = [plc.Column.from_numpy(rv, rm).slice(c, d)] + ([plc.Column.from_numpy(rv2, rm2).slice(c, d)] if wide else [])
                ol = [(v[a:b], m[a:b])] + ([(v2[a:b], m2[a:b])] if wide else [])
                orr = [(rv[c:d], rm[c:d])] + ([(rv2[c:d], rm2[c:d])] if wide else [])
                fj = plc.join.FilteredJoin(plc.Table(rcols), plc.NullEquality(ne))
                got_s, got_a = _ids(fj.semi_join(plc.Table(lcols))), _ids(fj.anti_join(plc.Table(lcols)))
                assert np.array_equal(got_s, osa.left_semi_join(ol, orr, ne)), (a, b, c, d, ne, wide)
                assert np.array_equal(got_a, osa.left_anti_join(ol, orr, ne)), (a, b, c, d, ne, wide)


def case_tile_edges(plc, small):
    """Left sizes around one compaction tile, and more than 32 tiles so the look-back reads past its first window."""
    rng = np.random.default_rng(36)
    sizes = (1, 31, TILE - 1, TILE, TILE + 1, 33 * TILE + 5)
    right = [(rng.integers(0, 1000, 500).astype(np.int64), None)]
    for n in sizes:
        for frac in (0.5, 1.0):  # about half of the rows kept, or every row on one side
            card = 1000 if frac == 0.5 else 500
            left = [(rng.integers(0, card if frac == 0.5 else 1, n).astype(np.int64) + (0 if frac == 0.5 else right[0][0][0]), None)]
            check(plc, left, right, 0, ("tile", n, frac))


def case_right_shapes(plc, small):
    """A duplicate-heavy filter (1e6 rows over 10 keys: one slot per key) and 2^20 distinct keys."""
    rng = np.random.default_rng(37)
    nd, nk, nl = (20_000, 1 << 12, 5000) if small else (1_000_000, 1 << 20, 300_000)
    dup = [(rng.integers(0, 10, nd).astype(np.int64) * 7, None)]
    left = [(rng.integers(0, 140, nl).astype(np.int64), None)]
    check(plc, left, dup, 0, "duplicate-heavy")
    distinct = [(rng.permutation(nk).astype(np.int64) * 3, None)]
    left = [(rng.integers(0, 6 * nk, nl).astype(np.int64), None)]
    check(plc, left, distinct, 0, "distinct")
    # the same shapes as wide keys (int64 + int32)
    check(plc, left + [(np.zeros(nl, np.int32), None)], distinct + [(np.zeros(nk, np.int32), None)], 0, "distinct wide")


def case_empty_inputs(plc, small):
    """Empty and zero-column sides return before any column check (filtered_join.cu:158-186)."""
    e64 = [(np.zeros(0, np.int64), None)]
    three = [(np.array([4, 5, 6], np.int64), None)]
    J = plc.join
    for right in ([], e64):
        fj = J.FilteredJoin(_table(plc, right), plc.NullEquality.EQUAL)
        for left in ([], e64):
            assert _ids(fj.semi_join(_table(plc, left))).size == 0 and _ids(fj.anti_join(_table(plc, left))).size == 0
        assert _ids(fj.semi_join(_table(plc, three))).size == 0
        assert _ids(fj.anti_join(_table(plc, three))).tolist() == [0, 1, 2]
        # an empty right side returns 0..n-1 whatever the left columns are
        assert _ids(fj.anti_join(_table(plc, three + [(np.zeros(3, np.float32), None)]))).tolist() == [0, 1, 2]
    fj = J.FilteredJoin(_table(plc, three), plc.NullEquality.EQUAL)
    for left in ([], e64, [(np.zeros(0, np.int8), None)] * 2):  # an empty left side: empty, even with mismatched columns
        assert _ids(fj.semi_join(_table(plc, left))).size == 0 and _ids(fj.anti_join(_table(plc, left))).size == 0


def case_load_factor(plc, small):
    """(0, 1] is valid; outside it is std::invalid_argument. A tiny factor is capped at 8x the rows' power of two."""
    rng = np.random.default_rng(38)
    right = [(np.arange(1000, dtype=np.int64) * 2, None)]
    left = [(rng.integers(0, 2500, 5000).astype(np.int64), None)]
    for lf in (1.0, 0.999, 0.5, 0.1, 1e-6):
        check(plc, left, right, 0, ("load factor", lf), load_factor=lf)
    n = 10_000 if small else 10_000_000
    big = plc.Table([plc.Column.from_numpy(np.arange(n, dtype=np.int32))])
    fj = plc.join.FilteredJoin(big, plc.NullEquality.EQUAL, 0.004)  # ~2.5e9 slots unless capped
    assert _ids(fj.semi_join(plc.Table([]))).size == 0 and _ids(fj.anti_join(plc.Table([]))).size == 0
    probe = np.array([-1, 0, n - 1, n, 7], np.int32)
    assert _ids(fj.semi_join(plc.Table([plc.Column.from_numpy(probe)]))).tolist() == [1, 2, 4]
    assert _ids(fj.anti_join(plc.Table([plc.Column.from_numpy(probe)]))).tolist() == [0, 3]


def case_object_reuse(plc, small):
    """One object probed with several left tables gives what a fresh object gives; the free functions match it."""
    rng = np.random.default_rng(39)
    right = [_rand(rng, 700, np.int64, 900, 0.1)]
    fj = plc.join.FilteredJoin(_table(plc, right), plc.NullEquality.EQUAL)
    J = plc.join
    for n in (5, 1000, TILE + 3):
        left = [_rand(rng, n, np.int64, 900, 0.1)]
        lt = _table(plc, left)
        s, a = _ids(fj.semi_join(lt)), _ids(fj.anti_join(lt))
        assert np.array_equal(s, osa.left_semi_join(left, right)) and np.array_equal(a, osa.left_anti_join(left, right)), n
        assert np.array_equal(_ids(J.left_semi_join(lt, _table(plc, right), plc.NullEquality.EQUAL)), s), n
        assert np.array_equal(_ids(J.left_anti_join(lt, _table(plc, right), plc.NullEquality.EQUAL)), a), n
        assert np.array_equal(_ids(fj.semi_join(lt)), s), n  # probes do not change the object


def case_errors(plc, small):
    J, EQ = plc.join, plc.NullEquality.EQUAL
    t64 = _table(plc, [(np.arange(10, dtype=np.int64), None)])
    fj = J.FilteredJoin(t64, EQ)
    with pytest.raises(ValueError):  # column count
        fj.semi_join(_table(plc, [(np.arange(4, dtype=np.int64), None)] * 2))
    with pytest.raises(ValueError):  # column type
        fj.anti_join(_table(plc, [(np.arange(4, dtype=np.int32), None)]))
    with pytest.raises(ValueError):
        J.left_semi_join(_table(plc, [(np.arange(4, dtype=np.uint64), None)]), t64, EQ)
    nine = plc.Table([plc.Column.from_numpy(np.arange(10, dtype=np.int8)) for _ in range(9)])
    with pytest.raises(ValueError):  # more than 8 key columns
        J.FilteredJoin(nine, EQ)
    with pytest.raises(ValueError):
        J.FilteredJoin(t64, 2)
    for lf in INVALID_LOAD_FACTORS["load_factors"] + [float("nan")]:
        with pytest.raises(ValueError):
            J.FilteredJoin(_table(plc, case_cols(INVALID_LOAD_FACTORS["right"])), EQ, lf)
    class _StringType:  # cudf::type_id::STRING, not fixed-width
        def id(self):
            return 23

    col = plc.Column.from_numpy(np.arange(10, dtype=np.int64))
    bad = plc.Column(_StringType(), 10, col._data, 0, 0, 0, [col])
    with pytest.raises(TypeError):  # a non-fixed-width column
        J.FilteredJoin(plc.Table([bad]), EQ)
    with pytest.raises(TypeError):
        fj.semi_join(plc.Table([bad]))


PARITY = {f.__name__[5:]: f for f in (case_key_types, case_float_keys, case_nulls, case_multi_column, case_sliced, case_tile_edges,
                                      case_right_shapes, case_empty_inputs, case_load_factor, case_object_reuse, case_errors)}


@pytest.mark.parametrize("case", CASES, ids=[c["src"] for c in CASES])
def test_golden(plc, case):
    fj = plc.join.FilteredJoin(_table(plc, case_cols(case["right"])), plc.NullEquality(case["nulls_equal"]))
    left = _table(plc, case_cols(case["left"]))
    assert _ids(fj.semi_join(left)).tolist() == case["semi"]
    assert _ids(fj.anti_join(left)).tolist() == case["anti"]


@pytest.mark.parametrize("name", list(PARITY))
def test_parity(plc, name):
    PARITY[name](plc, False)


def test_two_streams(plc):
    """One object probed from two CUDA streams at once gives the same results as a probe on one stream."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs CUDA streams")
    rng = np.random.default_rng(40)
    right = [(rng.integers(0, 1 << 22, 1 << 20).astype(np.int64), None)]
    fj = plc.join.FilteredJoin(_table(plc, right), plc.NullEquality.EQUAL)
    lefts = [_table(plc, [(rng.integers(0, 1 << 22, 3_000_000).astype(np.int64), None)]) for _ in range(2)]
    torch.cuda.synchronize()
    ref = [(_ids(fj.semi_join(lt)), _ids(fj.anti_join(lt))) for lt in lefts]
    streams = [torch.cuda.Stream() for _ in range(2)]
    out = [None, None]
    for i in range(2):
        with torch.cuda.stream(streams[i]):
            out[i] = (fj.semi_join(lefts[i], streams[i]), fj.anti_join(lefts[i], streams[i]))
    torch.cuda.synchronize()
    for i in range(2):
        assert np.array_equal(_ids(out[i][0]), ref[i][0]) and np.array_equal(_ids(out[i][1]), ref[i][1]), i

"""Unary operations and casts (cudf::unary_operation, cast, is_supported_cast, is_null / is_valid, is_nan / is_not_nan; pylibcudf's
unary module) through the C ABI and the ctypes twin, against the reference's known answers (tests/golden/unary_cases.py) and the
oracle (tests/unary_oracle.py).

Values are exact, sign of zero included and NaN payloads ignored, at rows that are valid and defined; SIN .. ARCTANH, EXP, LOG and
CBRT on float inputs are held to 4 ulp of the float64 oracle (rounded to float32 for FLOAT32), and an integer-typed result of those
operators must be the truncation of a value within 4 ulp of the oracle's double. The validity, null count and presence of a mask
are exact.

The parity cases are functions of (plc, small): tests/test_emu_unary.py runs them at reduced sizes on the kernel emulator, this
file at full size on the GPU."""
import numpy as np
import pytest

from tests import unary_oracle as ou
from tests.golden.unary_cases import CASES
from tests.test_unary_oracle import golden_input, oracle_of

pytestmark = pytest.mark.gpu

BLOCK = 256  # threads per CTA of unary_kernel


def _dt(plc, t):
    return plc.DataType(plc.TypeId(t))


def _rand(rng, n, t, nulls=0.0):
    """Values of type id t with the type's edge values mixed in; valid None or a bool array with `nulls` of them null."""
    dt = np.dtype(ou.NP[t])
    if dt == np.bool_:
        v = rng.random(n) < 0.5
    elif dt.kind == "f":
        v = (rng.normal(size=n) * 10).astype(dt)
        tiny = np.finfo(dt).smallest_subnormal
        special = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 0.5, -0.5, 1.5, 2.5, -2.5, 1.0, -1.0, 0.999, 3e9, -3e9,
                            tiny, -tiny, 3 * tiny, np.finfo(dt).max, np.finfo(dt).tiny], dt)
        pick = rng.random(n) < 0.2
        v[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    else:
        info = np.iinfo(dt)
        lo = -1000 if info.min < 0 else 0
        v = rng.integers(lo, 1000, n).astype(dt)
        special = np.array([info.min, info.max, 0, 1, info.max // 2 + 1, info.min + 1], dtype=dt)
        if info.min < 0:
            special = np.concatenate([special, np.array([-1], dt)])
        pick = rng.random(n) < 0.1
        v[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
        if ou.is_chrono(t):  # ticks around the epoch and whole units of the coarser types, before and after it
            near = rng.integers(-3 * 86400 * 1000, 3 * 86400 * 1000, n).astype(dt)
            v = np.where(rng.random(n) < 0.5, near, v)
    valid = (rng.random(n) >= nulls) if nulls else None
    return v, valid, t


def _column(plc, col):
    vals, valid, t = col
    return plc.Column.from_numpy(vals, valid, dtype=_dt(plc, t))  # chrono: the storage integers


def _ulps(a, b):
    it = np.int32 if a.dtype == np.float32 else np.int64
    ia, ib = a.view(it).astype(np.int64), b.view(it).astype(np.int64)
    ia = np.where(ia < 0, np.iinfo(it).min - ia, ia)
    ib = np.where(ib < 0, np.iinfo(it).min - ib, ib)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    return np.where(same, 0, np.abs(ia - ib))


def _same_float(g, e):
    return ((g == e) & (np.signbit(g) == np.signbit(e))) | (np.isnan(g) & np.isnan(e))


def compare(got, exp, exp_valid, defined, out_type, nullable, what, inexact=None):
    """got (a plc Column) equals the oracle's (values, valid, defined); `inexact`: (op, input column) of an operator held to 4 ulp."""
    assert int(got.type().id()) == out_type, (what, "type", got.type().id(), out_type)
    gv, gm = got.to_numpy()
    n = len(exp)
    assert got.size() == n, (what, "size")
    assert (gm is not None) == nullable, (what, "mask", gm is not None, nullable)
    valid = np.ones(n, bool) if gm is None else gm
    want_valid = np.ones(n, bool) if exp_valid is None else exp_valid
    assert np.array_equal(valid, want_valid), (what, "validity")
    assert got.null_count() == int((~want_valid).sum()), (what, "null_count")
    cmp = want_valid & defined
    g, e = gv[cmp], exp[cmp]
    if inexact is not None and ou.is_float(inexact[1][2]):
        bad = _ulps(g, e) > 4
    elif inexact is not None:
        op, (iv, _, it) = inexact
        d = ou.math_double(op, iv, it)[cmp]
        slack = 4 * np.spacing(np.abs(d))
        if out_type == ou.BOOL8:
            bad = (g != (d != 0)) & ~(np.abs(d) <= slack)
        else:
            lo, hi = np.trunc(d - slack), np.trunc(d + slack)
            gf = g.astype(np.float64)
            bad = (gf < lo) | (gf > hi)
    elif e.dtype.kind == "f":
        bad = ~_same_float(g, e)
    else:
        bad = g != e
    assert not bad.any(), (what, np.nonzero(cmp)[0][np.nonzero(bad)[0][:5]], g[bad][:5], e[bad][:5])


def check_unary(plc, op, col, what, plc_col=None):
    vals, valid, defined = ou.unary(op, col)
    out_t = ou.output_type(op, col[2]) if len(col[0]) else ou.empty_output_type(op, col[2])
    got = plc.unary.unary_operation(plc_col or _column(plc, col), plc.unary.UnaryOperator(op))
    compare(got, vals, valid, defined, out_t, col[1] is not None and len(col[0]) > 0, what,
            inexact=(op, col) if op in ou.INEXACT_OPS else None)


def check_cast(plc, col, to, what, plc_col=None):
    vals, valid, defined = ou.cast(col, to)
    got = plc.unary.cast(plc_col or _column(plc, col), _dt(plc, to))
    compare(got, vals, valid, defined, to, col[1] is not None and len(col[0]) > 0, what)


def check_predicate(plc, name, col, what, plc_col=None):
    exp = {"is_null": ou.is_null, "is_valid": ou.is_valid, "is_nan": ou.is_nan,
           "is_not_nan": lambda c: ou.is_nan(c, want_nan=False)}[name](col)
    got = getattr(plc.unary, name)(plc_col or _column(plc, col))
    compare(got, exp, None, np.ones(len(exp), bool), ou.BOOL8, False, what)


# ---- parity cases ------------------------------------------------------------------------------------------------------
def case_ops_by_type(plc, small):
    """Every operator over every fixed-width type, nulls on every other pair; unsupported pairs -> RuntimeError."""
    rng = np.random.default_rng(7)
    n = 150 if small else 3 * 32 * BLOCK + 45
    for op in ou.ALL_OPS:
        for i, t in enumerate(ou.FIXED_WIDTH):
            col = _rand(rng, n, t, 0.15 if (op + i) % 2 else 0.0)
            if ou.output_type(op, t) is None:
                with pytest.raises(RuntimeError):
                    plc.unary.unary_operation(_column(plc, col), plc.unary.UnaryOperator(op))
            else:
                check_unary(plc, op, col, (op, t))


def case_cast_matrix(plc, small):
    """Every cast pair of the 21 fixed-width ids, with and without nulls; timestamp <-> numeric -> RuntimeError; decimal
    targets -> TypeError, non-fixed-width targets -> RuntimeError."""
    rng = np.random.default_rng(11)
    n = 120 if small else 2 * 32 * BLOCK * 4 + 17
    for f in ou.FIXED_WIDTH:
        for i, to in enumerate(ou.FIXED_WIDTH):
            col = _rand(rng, n, f, 0.2 if i % 2 else 0.0)
            if ou.is_supported_cast(f, to):
                check_cast(plc, col, to, (f, to))
            else:
                with pytest.raises(RuntimeError):
                    plc.unary.cast(_column(plc, col), _dt(plc, to))
        c = _column(plc, _rand(rng, 5, f))
        for d in ou.DECIMALS:
            with pytest.raises(TypeError):
                plc.unary.cast(c, _dt(plc, d))
        for bad in (0, 22, 23, 24, 28):
            with pytest.raises(RuntimeError):
                plc.unary.cast(c, _dt(plc, bad))


def case_is_supported_cast(plc, small):
    """is_supported_cast over every pair of type ids equals the oracle (decimal pairs: False)."""
    for f in range(ou.NUM_TYPE_IDS):
        for to in range(ou.NUM_TYPE_IDS):
            assert plc.unary.is_supported_cast(_dt(plc, f), _dt(plc, to)) == ou.is_supported_cast(f, to), (f, to)


def case_float_specials(plc, small):
    """Every float operator and float cast on +-0, NaN, +-inf, subnormals, halfway values (RINT) and the type's limits."""
    for t in (ou.FLOAT32, ou.FLOAT64):
        dt = ou.NP[t]
        fi = np.finfo(dt)
        v = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, fi.smallest_subnormal, -fi.smallest_subnormal, fi.tiny, -fi.tiny,
                      fi.max, -fi.max, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 3.5, 4.5, 1e7 + 0.5, 2.0**52 + 1 if t == ou.FLOAT64 else 2.0**23 + 1,
                      1.0, -1.0, 0.99999, 2.0, 1e-300 if t == ou.FLOAT64 else 1e-40, 88.0, 710.0, -745.0, 3.0, 27.0], dt)
        for nulls in (None, np.arange(len(v)) % 3 != 1):
            col = (v, nulls, t)
            for op in ou.ALL_OPS:
                if ou.output_type(op, t) is not None:
                    check_unary(plc, op, col, ("special", t, op))
            for to in ou.NUMERIC + ou.DURATIONS:
                check_cast(plc, col, to, ("special cast", t, to))
            for name in ("is_nan", "is_not_nan"):
                check_predicate(plc, name, col, ("special", name, t))


def case_integer_extremes(plc, small):
    """Integer minima / maxima through every integer operator and cast, and pre-epoch chrono ticks through every unit change."""
    for t in [1, 2, 3, 4, 5, 6, 7, 8]:
        info = np.iinfo(ou.NP[t])
        v = np.array([info.min, info.min + 1, -1 if info.min < 0 else 2, 0, 1, info.max - 1, info.max], ou.NP[t])
        col = (v, None, t)
        for op in ou.ALL_OPS:
            if ou.output_type(op, t) is not None:
                check_unary(plc, op, col, ("extreme", t, op))
        for to in ou.NUMERIC + ou.DURATIONS:
            check_cast(plc, col, to, ("extreme cast", t, to))
    for f in ou.TIMESTAMPS + ou.DURATIONS:
        st = ou.NP[f]
        v = np.array([-1, -86399, -86400, -86401, -1001, -999, 0, 999, 1000, -131968727238, 1674631932929, np.iinfo(st).min,
                      np.iinfo(st).max] if st == np.int64 else [-1, -1528, 0, 17716, np.iinfo(st).min, np.iinfo(st).max], st)
        for to in ou.TIMESTAMPS + ou.DURATIONS + ou.NUMERIC:
            if ou.is_supported_cast(f, to):
                check_cast(plc, (v, None, f), to, ("chrono", f, to))


def case_masks(plc, small):
    """A mask with no nulls still gives the output a mask (copy_bitmask); all-null and all-valid masks; is_null / is_valid."""
    rng = np.random.default_rng(13)
    n = 300 if small else 70_001
    for t, op in [(ou.INT32, ou.NEGATE), (ou.FLOAT64, ou.SQRT), (ou.FLOAT32, ou.SIN), (ou.INT64, ou.BIT_COUNT), (ou.UINT8, ou.NOT)]:
        for valid in (np.ones(n, bool), np.zeros(n, bool), rng.random(n) < 0.5, None):
            col = _rand(rng, n, t)[:1] + (valid, t)
            check_unary(plc, op, col, (t, op, "mask"))
            check_cast(plc, col, ou.FLOAT64 if t != ou.FLOAT64 else ou.INT64, (t, "cast mask"))
            for name in ("is_null", "is_valid"):
                check_predicate(plc, name, col, (t, name))
            if ou.is_float(t):
                for name in ("is_nan", "is_not_nan"):
                    check_predicate(plc, name, col, (t, name))


def case_sliced_views(plc, small):
    """Views at offsets that are not multiples of 32 (nor of the vector width), on the vector and the generic paths."""
    rng = np.random.default_rng(17)
    n = 900 if small else 20_000
    work = [("unary", ou.FLOAT64, ou.SQRT), ("unary", ou.FLOAT32, ou.SIN), ("unary", ou.INT32, ou.NOT), ("unary", ou.INT16, ou.ABS),
            ("cast", ou.INT32, ou.FLOAT64), ("cast", ou.FLOAT64, ou.INT8), ("cast", ou.TIMESTAMP_NS, ou.TIMESTAMP_MS),
            ("cast", ou.TIMESTAMP_S, ou.TIMESTAMP_D), ("cast", ou.UINT16, ou.BOOL8), ("is_null", ou.INT64, None),
            ("is_valid", ou.INT8, None), ("is_nan", ou.FLOAT32, None), ("is_not_nan", ou.FLOAT64, None)]
    for kind, t, arg in work:
        col = _rand(rng, n, t, 0.3)
        full = _column(plc, col)
        for b, m in [(0, n), (1, n - 40), (33, 300), (31, n - 64), (4, 129), (64, n - 100), (7, 0)]:
            sl = (col[0][b:b + m], col[1][b:b + m], t)
            pc = full.slice(b, b + m)
            what = (kind, t, arg, b, m)
            if kind == "unary":
                check_unary(plc, arg, sl, what, plc_col=pc)
            elif kind == "cast":
                check_cast(plc, sl, arg, what, plc_col=pc)
            else:
                check_predicate(plc, kind, sl, what, plc_col=pc)


def case_lengths(plc, small):
    """Lengths around 32-row words, vector tiles (32 x 1 .. 16 rows per warp), 1024-row validity steps and 256-thread blocks."""
    rng = np.random.default_rng(19)
    lengths = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025]
    if not small:
        lengths += [2047, 2048, 2049, 8 * 1024 - 1, 8 * 1024 + 1, 32 * BLOCK * 16 + 3]
    for n in lengths:
        for nulls in (0.0, 0.25):
            check_unary(plc, ou.SQRT, _rand(rng, n, ou.FLOAT64, nulls), (n, "sqrt"))
            check_unary(plc, ou.SIN, _rand(rng, n, ou.FLOAT32, nulls), (n, "sin"))
            check_unary(plc, ou.NEGATE, _rand(rng, n, ou.INT64, nulls), (n, "negate"))
            check_cast(plc, _rand(rng, n, ou.INT8, nulls), ou.FLOAT64, (n, "i8->f64"))
            check_cast(plc, _rand(rng, n, ou.FLOAT64, nulls), ou.INT32, (n, "f64->i32"))
            check_cast(plc, _rand(rng, n, ou.TIMESTAMP_NS, nulls), ou.TIMESTAMP_MS, (n, "ns->ms"))
            check_cast(plc, _rand(rng, n, ou.TIMESTAMP_D, nulls), ou.TIMESTAMP_S, (n, "D->s"))
            check_predicate(plc, "is_null", _rand(rng, n, ou.INT32, nulls or 0.5), (n, "is_null"))
            check_predicate(plc, "is_nan", _rand(rng, n, ou.FLOAT32, nulls), (n, "is_nan"))


def case_empty(plc, small):
    """Empty columns: the output type without a type check (RINT of INT32 is INT32), casts, predicates; the errors that still
    apply (timestamp <-> numeric cast, is_nan of a non-float)."""
    for t in ou.FIXED_WIDTH:
        col = (np.zeros(0, ou.NP[t]), None, t)
        for op in ou.ALL_OPS:
            got = plc.unary.unary_operation(_column(plc, col), plc.unary.UnaryOperator(op))
            assert int(got.type().id()) == ou.empty_output_type(op, t) and got.size() == 0, (t, op)
        for to in ou.FIXED_WIDTH:
            if ou.is_supported_cast(t, to):
                check_cast(plc, col, to, ("empty", t, to))
            else:
                with pytest.raises(RuntimeError):
                    plc.unary.cast(_column(plc, col), _dt(plc, to))
        for name in ("is_null", "is_valid"):
            check_predicate(plc, name, col, ("empty", name, t))
        for name in ("is_nan", "is_not_nan"):
            if ou.is_float(t):
                check_predicate(plc, name, col, ("empty", name, t))
            else:
                with pytest.raises(RuntimeError):
                    getattr(plc.unary, name)(_column(plc, col))


def case_bit_cast(plc, small):
    """bit_cast: a copy of the bits and the mask under the target type; types of different widths -> RuntimeError."""
    rng = np.random.default_rng(23)
    n = 200 if small else 10_007
    for f in ou.FIXED_WIDTH:
        col = _rand(rng, n, f, 0.3)
        c = _column(plc, col).slice(3, n)
        for to in ou.FIXED_WIDTH:
            if np.dtype(ou.NP[f]).itemsize != np.dtype(ou.NP[to]).itemsize:
                with pytest.raises(RuntimeError):
                    plc.unary.bit_cast(c, _dt(plc, to))
                continue
            got = plc.unary.bit_cast(c, _dt(plc, to))
            assert int(got.type().id()) == to and got.null_count() == c.null_count()
            gv, gm = got.to_numpy()
            w = np.dtype(ou.NP[to]).itemsize
            want = col[0][3:].view(np.uint8) if col[0].dtype != np.bool_ else col[0][3:].astype(np.uint8)
            have = gv.view(np.uint8) if gv.dtype != np.bool_ else gv.astype(np.uint8)
            if to == ou.BOOL8 or f == ou.BOOL8:  # BOOL8 reads back as 0 / 1
                want, have = want != 0, have != 0
            assert np.array_equal(have.reshape(-1, w) if w > 1 else have, want.reshape(-1, w) if w > 1 else want), (f, to)
            assert np.array_equal(gm, col[1][3:]), (f, to)
        for d in ou.DECIMALS:
            with pytest.raises(RuntimeError):
                plc.unary.bit_cast(c, _dt(plc, d))


def case_integration(plc, small):
    """With the existing operations: apply_boolean_mask(t, is_valid(c)) == drop_nulls, apply_boolean_mask(t, is_not_nan(c)) ==
    drop_nans, NOT of a binary_operation GREATER, and a binary_operation on a cast result."""
    rng = np.random.default_rng(29)
    n = 1000 if small else 1_000_003
    x = rng.normal(size=n)
    x[rng.random(n) < 0.1] = np.nan
    valid = rng.random(n) >= 0.2
    k = rng.integers(-50, 50, n).astype(np.int32)
    xc, kc = plc.Column.from_numpy(x, valid), plc.Column.from_numpy(k)
    t = plc.Table([xc, kc])
    sc = plc.stream_compaction

    def cols(tbl):
        return [c.to_numpy() for c in tbl.columns()]

    def same(a, b):
        for (av, am), (bv, bm) in zip(cols(a), cols(b)):
            am = np.ones(len(av), bool) if am is None else am
            bm = np.ones(len(bv), bool) if bm is None else bm
            assert np.array_equal(am, bm)
            assert np.array_equal(av[am], bv[bm], equal_nan=av.dtype.kind == "f")

    same(sc.apply_boolean_mask(t, plc.unary.is_valid(xc)), sc.drop_nulls(t, [0], 1))
    same(sc.apply_boolean_mask(t, plc.unary.is_not_nan(xc)), sc.drop_nans(t, [0], 1))
    gt = plc.binaryop.binary_operation(xc, plc.Scalar.from_py(0.5, _dt(plc, ou.FLOAT64)), plc.binaryop.BinaryOperator.GREATER,
                                       _dt(plc, ou.BOOL8))
    notgt = plc.unary.unary_operation(gt, plc.unary.UnaryOperator.NOT)
    gv, gm = notgt.to_numpy()
    assert np.array_equal(gm, valid) and notgt.null_count() == int((~valid).sum())
    assert np.array_equal(gv[valid], ~(x[valid] > 0.5))
    kf = plc.unary.cast(kc, _dt(plc, ou.FLOAT64))
    s = plc.binaryop.binary_operation(kf, xc, plc.binaryop.BinaryOperator.ADD, _dt(plc, ou.FLOAT64))
    sv, sm = s.to_numpy()
    assert np.array_equal(sm, valid)
    assert np.array_equal(sv[valid], k[valid].astype(np.float64) + x[valid], equal_nan=True)


PARITY = {
    "ops by type": case_ops_by_type, "cast matrix": case_cast_matrix, "is_supported_cast": case_is_supported_cast,
    "float specials": case_float_specials, "integer extremes": case_integer_extremes, "masks": case_masks,
    "sliced views": case_sliced_views, "lengths": case_lengths, "empty": case_empty, "bit_cast": case_bit_cast,
    "integration": case_integration,
}


@pytest.mark.parametrize("name", list(PARITY))
def test_parity(plc, name):
    PARITY[name](plc, False)


def test_golden(plc):
    for c in CASES:
        col = golden_input(c)
        pc = _column(plc, col)
        fn = c["fn"]

        def run():
            if fn == "unary":
                return plc.unary.unary_operation(pc, plc.unary.UnaryOperator(c["op"]))
            if fn == "cast":
                out = pc
                for to in (c["to"] if isinstance(c["to"], list) else [c["to"]]):
                    out = plc.unary.cast(out, _dt(plc, to))
                return out
            return getattr(plc.unary, fn)(pc)

        if "raises" in c:
            with pytest.raises({"RuntimeError": RuntimeError, "TypeError": TypeError}[c["raises"]]):
                run()
            continue
        got = run()
        assert int(got.type().id()) == c["expect_type"], c["src"]
        vals, valid, _ = oracle_of(c)
        gv, gm = got.to_numpy()
        gm = np.ones(len(gv), bool) if gm is None else gm
        assert [e is not None for e in c["expect"]] == list(gm), c["src"]
        e = np.array([0 if x is None else x for x in c["expect"]], dtype=np.float64 if gv.dtype.kind == "f" else object).astype(gv.dtype)
        if c.get("approx"):
            assert (_ulps(gv[gm], e[gm]) <= 4).all(), c["src"]
        elif gv.dtype.kind == "f":
            assert ((gv[gm] == e[gm]) | (np.isnan(gv[gm]) & np.isnan(e[gm]))).all(), c["src"]
        else:
            assert np.array_equal(gv[gm], e[gm]), (c["src"], gv, e)

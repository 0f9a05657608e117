"""Replacement (cudf::replace_nulls, replace_nans, find_and_replace_all, clamp, normalize_nans_and_zeros; pylibcudf's replace
module) through the C ABI and the ctypes twin, against the reference's known answers (tests/golden/replace_cases.py) and the
oracle (tests/replace_oracle.py).

Values are exact at valid rows, sign of zero included (normalize_nans_and_zeros: bit for bit, NaN payloads included); the
validity, the null count and the presence of a mask are exact.

The parity cases are functions of (plc, small): tests/test_emu_replace.py runs them at reduced sizes on the kernel emulator, this
file at full size on the GPU."""
import ctypes as C

import numpy as np
import pytest

from tests import replace_oracle as orp
from tests import unary_oracle as ou
from tests.test_unary_gpu import _column, _dt, _rand

pytestmark = pytest.mark.gpu

TILE = 8192  # rows per look-back tile of fill_kernel
S = orp.Scalar
FLOATS = (ou.FLOAT32, ou.FLOAT64)


def _scalar(plc, value, t, valid=True):
    return plc.Scalar.from_py(None if not valid else value, _dt(plc, t))


def _bits(a):
    return a.view(np.uint8) if a.dtype != np.bool_ else a.astype(np.uint8)


def check(got, exp, t, what, bitwise=False):
    vals, valid = exp
    assert int(got.type().id()) == t, (what, "type")
    gv, gm = got.to_numpy()
    n = len(vals)
    assert got.size() == n, (what, "size")
    assert (gm is not None) == (valid is not None), (what, "mask", gm is not None, valid is not None)
    m = np.ones(n, bool) if valid is None else valid
    if gm is not None:
        assert np.array_equal(gm, m), (what, "validity", np.nonzero(gm != m)[0][:5])
    assert got.null_count() == int((~m).sum()), (what, "null_count", got.null_count(), int((~m).sum()))
    g, e = gv[m], vals[m]
    if bitwise:
        assert np.array_equal(_bits(g), _bits(e.astype(g.dtype))), (what, "bits")
    elif g.dtype.kind == "f":
        bad = ~(((g == e) & (np.signbit(g) == np.signbit(e))) | (np.isnan(g) & np.isnan(e)))
        assert not bad.any(), (what, np.nonzero(m)[0][np.nonzero(bad)[0][:5]], g[bad][:5], e[bad][:5])
    else:
        assert np.array_equal(g, e.astype(g.dtype)), (what, np.nonzero(g != e)[0][:5])


def _sliced(plc, col, b, m):
    """(the oracle's view of rows [b, b + m), the plc column slice)."""
    full = _column(plc, col)
    return (col[0][b:b + m], None if col[1] is None else col[1][b:b + m], col[2]), full.slice(b, b + m)


def _policy(plc, p):
    return plc.replace.ReplacePolicy(p)


# ---- parity cases ------------------------------------------------------------------------------------------------------
def case_nulls_by_type(plc, small):
    """replace_nulls with a column (with and without nulls), a scalar (valid and null) and both policies over every type."""
    rng = np.random.default_rng(3)
    n = 300 if small else 3 * TILE + 77
    for i, t in enumerate(ou.FIXED_WIDTH):
        col = _rand(rng, n, t, 0.4)
        for rn in (0.0, 0.3):
            rep = _rand(rng, n, t, rn)
            check(plc.replace.replace_nulls(_column(plc, col), _column(plc, rep)), orp.replace_nulls_column(col, rep), t, (t, "col", rn))
        s = rep[0][0]
        check(plc.replace.replace_nulls(_column(plc, col), _scalar(plc, s, t)), orp.replace_nulls_scalar(col, orp.Scalar(s, True, t)), t, (t, "scalar"))
        check(plc.replace.replace_nulls(_column(plc, col), _scalar(plc, s, t, False)), orp.replace_nulls_scalar(col, orp.Scalar(s, False, t)), t,
              (t, "null scalar"))
        for p in (orp.PRECEDING, orp.FOLLOWING):
            check(plc.replace.replace_nulls(_column(plc, col), _policy(plc, p)), orp.replace_nulls_policy(col, p), t, (t, "policy", p))
        none = (col[0], None, t)
        check(plc.replace.replace_nulls(_column(plc, none), _policy(plc, i % 2)), orp.copy(none), t, (t, "no mask"))


def case_nans_by_type(plc, small):
    """replace_nans with a column (nulls or not) and a scalar (valid or null) on both float types; NaNs under null bits."""
    rng = np.random.default_rng(5)
    n = 300 if small else 3 * 32 * 256 + 13
    for t in FLOATS:
        for nulls in (0.0, 0.3):
            col = _rand(rng, n, t, nulls)
            col[0][rng.random(n) < 0.3] = np.nan
            for rn in (0.0, 0.3):
                rep = _rand(rng, n, t, rn)
                exp = orp.replace_nans(col, rep)
                check(_nans_abi(plc, col, rep), exp, t, (t, "nans col", nulls, rn))
            for sv in (True, False):
                exp = orp.replace_nans(col, orp.Scalar(2.5, sv, t))
                check(_nans_abi(plc, col, _scalar(plc, 2.5, t, sv)), exp, t, (t, "nans scalar", sv))
        # views at offsets that are not multiples of 4 rows: the generic (one row per lane) path for the whole call
        rep = _rand(rng, n + 8, t, 0.3)
        for b, rb in ((1, 3), (5, 2), (33, 7)):
            m = n - 40
            sl, pc = _sliced(plc, col, b, m)
            rsl, rpc = _sliced(plc, rep, rb, m)
            check(_nans_abi(plc, pc, rpc), orp.replace_nans(sl, rsl), t, (t, "nans sliced", b, rb))
            check(_nans_abi(plc, pc, _scalar(plc, -4.0, t)), orp.replace_nans(sl, orp.Scalar(-4.0, True, t)), t, (t, "nans sliced sc", b))


def _nans_abi(plc, col, rep):
    """replace_nans is C ABI / C++ only (pylibcudf has none): call b2_replace_nans / _scalar through the twin's library."""
    from cudf_b200 import _lib

    c = col if not isinstance(col, tuple) else _column(plc, col)
    v = c._view()
    out = C.c_void_p()
    if not isinstance(rep, plc.Scalar):
        rc = _column(plc, rep) if isinstance(rep, tuple) else rep  # kept alive across the call
        r = rc._view()
        _lib.check(_lib.lib.b2_replace_nans(C.byref(v), C.byref(r), None, C.byref(out)))
    else:
        _lib.check(_lib.lib.b2_replace_nans_scalar(C.byref(v), C.c_void_p(rep._handle), None, C.byref(out)))
    return plc.Column._from_handle(out.value)


def case_find_and_replace(plc, small):
    """find_and_replace_all over every type with k = 1, 16, 1000 and a table past the shared-memory budget; duplicates, absent
    values, null new values, +-0 and NaN in both the old values and the input."""
    rng = np.random.default_rng(7)
    n = 400 if small else 50_003
    for i, t in enumerate(ou.FIXED_WIDTH):
        for k in (1, 16, 1000, 7000):  # 7000 keys of 8 bytes and their positions pass the 48 KiB shared-memory budget
            if small and k == 7000 and t not in (ou.INT64, ou.FLOAT64):
                continue
            col = _rand(rng, n, t, 0.2 if i % 2 else 0.0)
            pool = _rand(rng, max(k, 8), t)[0]
            old = pool[rng.integers(0, len(pool), k)]  # duplicates
            if k > 1:
                old[0] = col[0][0]
            new = _rand(rng, k, t, 0.2 if k % 2 == 0 else 0.0)
            exp = orp.find_and_replace_all(col, (old, None, t), new)
            got = plc.replace.find_and_replace_all(_column(plc, col), _column(plc, (old, None, t)), _column(plc, new))
            check(got, exp, t, (t, k))
    for t in FLOATS:
        dt = ou.NP[t]
        x = np.array([0.0, -0.0, np.nan, 1.0, -1.0, np.inf, -np.inf, 2.0] * 40, dt)
        old = np.array([-0.0, np.nan, 1.0, 1.0, -np.inf], dt)
        new = np.array([5.0, 6.0, 7.0, 8.0, 9.0], dt)
        col = (x, np.arange(len(x)) % 7 != 3, t)
        check(plc.replace.find_and_replace_all(_column(plc, col), _column(plc, (old, None, t)), _column(plc, (new, None, t))),
              orp.find_and_replace_all(col, (old, None, t), (new, None, t)), t, (t, "specials"))


def case_clamp(plc, small):
    """clamp over every type: both bounds, one null bound, both null (a copy), with and without replacements; NaN and +-0."""
    rng = np.random.default_rng(11)
    n = 300 if small else 3 * 32 * 256 * 4 + 9
    for t in ou.FIXED_WIDTH:
        col = _rand(rng, n, t, 0.25)
        srt = np.sort(col[0][:50])
        lo, hi = srt[10], srt[40]
        lr, hr = srt[0], srt[49]
        for lv, hv in ((True, True), (True, False), (False, True), (False, False)):
            exp = orp.clamp(col, S(lo, lv, t), S(lr, True, t), S(hi, hv, t), S(hr, True, t))
            got = plc.replace.clamp(_column(plc, col), _scalar(plc, lo, t, lv), _scalar(plc, hi, t, hv), _scalar(plc, lr, t),
                                    _scalar(plc, hr, t))
            check(got, exp, t, (t, "clamp", lv, hv))
        exp = orp.clamp(col, S(lo, True, t), S(lo, True, t), S(hi, True, t), S(hi, True, t))
        check(plc.replace.clamp(_column(plc, col), _scalar(plc, lo, t), _scalar(plc, hi, t)), exp, t, (t, "clamp3"))
    for t in FLOATS:
        dt = ou.NP[t]
        x = np.array([np.nan, -0.0, 0.0, -1.0, 1.0, -np.inf, np.inf, 0.5], dt)
        col = (x, None, t)
        for lo, hi in ((0.0, 0.5), (-0.0, 0.0), (-1.0, np.nan)):
            exp = orp.clamp(col, S(lo, True, t), S(-7.0, True, t), S(hi, True, t), S(7.0, True, t))
            got = plc.replace.clamp(_column(plc, col), _scalar(plc, lo, t), _scalar(plc, hi, t), _scalar(plc, -7.0, t), _scalar(plc, 7.0, t))
            check(got, exp, t, (t, "float clamp", lo, hi))


def case_normalize(plc, small):
    """normalize_nans_and_zeros, copy and in place, bit for bit: NaNs of any payload and sign, +-0, with a mask and sliced."""
    rng = np.random.default_rng(13)
    n = 300 if small else 100_003
    for t in FLOATS:
        dt = ou.NP[t]
        it = np.uint32 if dt == np.float32 else np.uint64
        col = _rand(rng, n, t, 0.2)
        pick = rng.random(n) < 0.3
        payload = rng.integers(1, 1 << 20, int(pick.sum())).astype(it)
        exp_bits = (np.array(np.inf, dt).view(it) | payload) | (rng.integers(0, 2, int(pick.sum())).astype(it) << it(8 * dt().itemsize - 1))
        col[0][pick] = exp_bits.view(dt)
        col[0][rng.random(n) < 0.1] = -0.0
        check(plc.replace.normalize_nans_and_zeros(_column(plc, col)), orp.normalize_nans_and_zeros(col), t, (t, "copy"), bitwise=True)
        sl, pc = _sliced(plc, col, 5, n - 40)
        check(plc.replace.normalize_nans_and_zeros(pc), orp.normalize_nans_and_zeros(sl), t, (t, "slice"), bitwise=True)
        c = _column(plc, col)
        assert plc.replace.normalize_nans_and_zeros(c, inplace=True) is None
        check(c, orp.normalize_nans_and_zeros(col), t, (t, "inplace"), bitwise=True)
        c = _column(plc, col)
        plc.replace.normalize_nans_and_zeros(c.slice(3, 3 + 50), inplace=True)  # only the view's rows change
        want = col[0].copy()
        want[3:53] = orp.normalize_nans_and_zeros((col[0][3:53], None, t))[0]
        check(c, (want, col[1]), t, (t, "inplace slice"), bitwise=True)


def case_sliced_views(plc, small):
    """Views at offsets that are not multiples of 32 for every form; the replacement column at another offset."""
    rng = np.random.default_rng(17)
    n = 900 if small else 20_000
    for t in (ou.INT8, ou.INT16, ou.INT32, ou.FLOAT64, ou.TIMESTAMP_MS):
        col = _rand(rng, n, t, 0.35)
        rep = _rand(rng, n + 11, t, 0.2)  # sliced at another offset
        for b, m in [(0, n), (1, n - 40), (33, 300), (31, n - 64), (4, 129), (64, n - 100), (7, 0)]:
            sl, pc = _sliced(plc, col, b, m)
            rsl, rpc = _sliced(plc, rep, (b + 5) % 11, m)
            what = (t, b, m)
            check(plc.replace.replace_nulls(pc, rpc), orp.replace_nulls_column(sl, rsl), t, what + ("col",))
            for p in (orp.PRECEDING, orp.FOLLOWING):
                check(plc.replace.replace_nulls(pc, _policy(plc, p)), orp.replace_nulls_policy(sl, p), t, what + ("policy", p))
            lo, hi = np.sort(col[0][:9])[[2, 6]]
            check(plc.replace.clamp(pc, _scalar(plc, lo, t), _scalar(plc, hi, t)),
                  orp.clamp(sl, S(lo, True, t), S(lo, True, t), S(hi, True, t), S(hi, True, t)), t, what + ("clamp",))
            old = col[0][:5]
            new = rep[0][:5]
            check(plc.replace.find_and_replace_all(pc, _column(plc, (old, None, t)), rpc.slice(0, 5) if m >= 5 else _column(plc, (new, None, t))),
                  orp.find_and_replace_all(sl, (old, None, t), (rsl[0][:5], rsl[1][:5], t) if m >= 5 else (new, None, t)), t, what + ("find",))


def case_lengths(plc, small):
    """Lengths around words, vector steps, warps and look-back tiles, n = 1 and all-null columns."""
    rng = np.random.default_rng(19)
    lengths = [1, 2, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, TILE - 1, TILE, TILE + 1]
    if not small:
        lengths += [2 * TILE + 1, 8 * 1024 * 16 + 3]
    for n in lengths:
        for t in (ou.INT64, ou.UINT8, ou.FLOAT32):
            for nulls in (0.5, 1.0):
                col = _rand(rng, n, t, 0.0)
                col = (col[0], rng.random(n) >= nulls, t)
                rep = _rand(rng, n, t, 0.3)
                check(plc.replace.replace_nulls(_column(plc, col), _column(plc, rep)), orp.replace_nulls_column(col, rep), t, (n, t, "col"))
                check(plc.replace.replace_nulls(_column(plc, col), _scalar(plc, 3, t)), orp.replace_nulls_scalar(col, S(3, True, t)), t, (n, t, "sc"))
                for p in (orp.PRECEDING, orp.FOLLOWING):
                    check(plc.replace.replace_nulls(_column(plc, col), _policy(plc, p)), orp.replace_nulls_policy(col, p), t, (n, t, p))


def case_long_runs(plc, small):
    """Null runs across look-back tiles (at least three, so the look-back, FOLLOWING's reversed tile order and the carry across
    tiles run on the emulator too), both directions; a single valid row at either end; all null but one."""
    rng = np.random.default_rng(23)
    n = 3 * TILE + 123 if small else 40 * TILE + 123
    v = rng.integers(-10**9, 10**9, n).astype(np.int64)
    layouts = []
    valid = np.zeros(n, bool)
    valid[[0, n // 3, n // 3 + 1, n - 1]] = True
    layouts.append(valid)
    for at in (0, n - 1, n // 2):
        valid = np.zeros(n, bool)
        valid[at] = True
        layouts.append(valid)
    valid = rng.random(n) < 0.001
    layouts.append(valid)
    for valid in layouts:
        col = (v, valid, ou.INT64)
        for p in (orp.PRECEDING, orp.FOLLOWING):
            check(plc.replace.replace_nulls(_column(plc, col), _policy(plc, p)), orp.replace_nulls_policy(col, p), ou.INT64,
                  ("runs", int(valid.sum()), p))


def case_empty(plc, small):
    """Empty columns: an empty result of the input's type for every form."""
    for t in ou.FIXED_WIDTH:
        e = _column(plc, (np.zeros(0, ou.NP[t]), None, t))
        outs = [plc.replace.replace_nulls(e, e), plc.replace.replace_nulls(e, _scalar(plc, 1, t)),
                plc.replace.replace_nulls(e, _policy(plc, 0)), plc.replace.find_and_replace_all(e, e, e),
                plc.replace.clamp(e, _scalar(plc, 1, t), _scalar(plc, 2, t))]
        if t in FLOATS:
            outs.append(plc.replace.normalize_nans_and_zeros(e))
        for o in outs:
            assert o.size() == 0 and int(o.type().id()) == t, t


def case_errors(plc, small):
    """The reference's errors: data_type_error -> TypeError, logic_error -> RuntimeError; pylibcudf's argument errors."""
    i32 = _column(plc, (np.arange(10, dtype=np.int32), np.arange(10) % 2 == 0, ou.INT32))
    i64 = _column(plc, (np.arange(10, dtype=np.int64), None, ou.INT64))
    f64 = _column(plc, (np.arange(10, dtype=np.float64), None, ou.FLOAT64))
    short = _column(plc, (np.arange(4, dtype=np.int32), None, ou.INT32))
    s32, s64 = _scalar(plc, 1, ou.INT32), _scalar(plc, 1, ou.INT64)
    cases = [
        (lambda: plc.replace.replace_nulls(i32, i64), TypeError),
        (lambda: plc.replace.replace_nulls(i32, short), RuntimeError),
        (lambda: plc.replace.replace_nulls(i32, s64), TypeError),
        (lambda: plc.replace.replace_nulls(i32, 3), TypeError),
        (lambda: plc.replace.find_and_replace_all(i32, short, i32), RuntimeError),
        (lambda: plc.replace.find_and_replace_all(i32, i64, i64), TypeError),
        (lambda: plc.replace.find_and_replace_all(i64, i32, i32), TypeError),
        (lambda: plc.replace.find_and_replace_all(i64, _column(plc, (np.arange(3), np.array([1, 0, 1], bool), ou.INT64)), i64.slice(0, 3)),
         RuntimeError),
        (lambda: plc.replace.clamp(i32, s32, s64), TypeError),
        (lambda: plc.replace.clamp(i32, s32, s32, s64, s64), TypeError),
        (lambda: plc.replace.clamp(i32, s64, s64), TypeError),
        (lambda: plc.replace.clamp(i32, s32, s32, _scalar(plc, 1, ou.INT32, False), s32), RuntimeError),
        (lambda: plc.replace.clamp(i32, s32, s32, s32, None), ValueError),
        (lambda: plc.replace.normalize_nans_and_zeros(i32), RuntimeError),
        (lambda: plc.replace.normalize_nans_and_zeros(i32, inplace=True), RuntimeError),
        (lambda: _nans_abi(plc, i32, (np.arange(10, dtype=np.int32), None, ou.INT32)), RuntimeError),
        (lambda: _nans_abi(plc, f64, (np.arange(10, dtype=np.float32), None, ou.FLOAT32)), RuntimeError),
        (lambda: _nans_abi(plc, f64, (np.arange(4, dtype=np.float64), None, ou.FLOAT64)), RuntimeError),
        (lambda: _nans_abi(plc, f64, _scalar(plc, 1.0, ou.FLOAT32)), RuntimeError),
    ]
    for fn, exc in cases:
        with pytest.raises(exc):
            fn()
    # no type check where the reference returns a copy first
    check(plc.replace.replace_nulls(i64, s32), orp.copy((np.arange(10, dtype=np.int64), None, ou.INT64)), ou.INT64, "no-null copy")
    check(plc.replace.replace_nulls(i32, _scalar(plc, 1, ou.INT64, False)),
          orp.copy((np.arange(10, dtype=np.int32), np.arange(10) % 2 == 0, ou.INT32)), ou.INT32, "null scalar copy")


def case_integration(plc, small):
    """is_null -> replace_nulls, binary_operation -> clamp, replace_nulls (PRECEDING) -> drop_nulls."""
    rng = np.random.default_rng(29)
    n = 1000 if small else 1_000_003
    x = rng.normal(size=n)
    valid = rng.random(n) >= 0.3
    valid[0] = False
    xc = plc.Column.from_numpy(x, valid)
    isn = plc.unary.is_null(xc)
    filled = plc.replace.replace_nulls(isn, plc.Scalar.from_py(False, _dt(plc, ou.BOOL8)))
    fv, fm = filled.to_numpy()
    assert fm is None and np.array_equal(fv, ~valid)
    prod = plc.binaryop.binary_operation(xc, plc.Scalar.from_py(3.0, _dt(plc, ou.FLOAT64)), plc.binaryop.BinaryOperator.MUL,
                                         _dt(plc, ou.FLOAT64))
    cl = plc.replace.clamp(prod, _scalar(plc, -1.0, ou.FLOAT64), _scalar(plc, 1.0, ou.FLOAT64))
    check(cl, (np.clip(x * 3.0, -1.0, 1.0), valid), ou.FLOAT64, "mul -> clamp")
    ff = plc.replace.replace_nulls(xc, _policy(plc, orp.PRECEDING))
    assert ff.null_count() == 1
    kept = plc.stream_compaction.drop_nulls(plc.Table([ff]), [0], 1).columns()[0]
    exp, _ = orp.replace_nulls_policy((x, valid, ou.FLOAT64), orp.PRECEDING)
    kv, _ = kept.to_numpy()
    assert np.array_equal(kv, exp[1:])


def case_golden(plc, small):
    """The reference's known answers (tests/golden/replace_cases.py) through the library, errors included; normalize in place
    too, as the reference's test does."""
    from tests.golden.replace_cases import CASES
    from tests.test_replace_oracle import ERRORS, golden_args, same

    for c in CASES:
        for t in c["types"]:
            args = golden_args(c, t)
            keep = [_scalar(plc, a.value, a.type, a.valid) if isinstance(a, orp.Scalar) else _column(plc, a) if isinstance(a, tuple)
                    else _policy(plc, a) for a in args]
            fn = c["fn"]

            def run():
                if fn == "replace_nans":
                    return _nans_abi(plc, *keep)
                if fn == "clamp" and len(keep) == 5:  # the reference's (lo, lo_replace, hi, hi_replace) in pylibcudf's order
                    col, lo, lo_r, hi, hi_r = keep
                    return plc.replace.clamp(col, lo, hi, lo_r, hi_r)
                return getattr(plc.replace, fn)(*keep)

            if c["raises"]:
                with pytest.raises(ERRORS[c["raises"]]):
                    run()
                continue
            got = run()
            assert int(got.type().id()) == t, c["src"]
            same(*got.to_numpy(), c, t)
            if fn == "normalize_nans_and_zeros":
                assert plc.replace.normalize_nans_and_zeros(keep[0], inplace=True) is None
                same(*keep[0].to_numpy(), c, t)


PARITY = {
    "nulls by type": case_nulls_by_type, "nans by type": case_nans_by_type, "find_and_replace_all": case_find_and_replace,
    "clamp": case_clamp, "normalize": case_normalize, "sliced views": case_sliced_views, "lengths": case_lengths,
    "long runs": case_long_runs, "empty": case_empty, "errors": case_errors, "integration": case_integration,
    "golden": case_golden,
}


@pytest.mark.parametrize("name", list(PARITY))
def test_parity(plc, name):
    PARITY[name](plc, False)

"""Binary operations (cudf::binary_operation; pylibcudf's binaryop.binary_operation / is_supported_operation) through the C ABI
and the ctypes twin, against the reference's known answers (tests/golden/binaryop_cases.py) and the oracle
(tests/binaryop_oracle.py). Values are exact at rows that are valid and defined (POW, LOG_BASE and ATAN2: within 4 ulp); the
validity, null count and presence of a mask are exact.

The parity cases are functions of (plc, small): tests/test_emu_binaryop.py runs them at reduced sizes on the kernel emulator,
this file at full size on the GPU."""
import numpy as np
import pytest

from tests import binaryop_oracle as ob
from tests.golden.binaryop_cases import CASES
from tests.test_binaryop_oracle import out_type
from tests.test_binaryop_oracle import operand as golden_operand

pytestmark = pytest.mark.gpu

NUMERIC = ob.NUMERIC
BLOCK = 256  # threads per CTA of binop_kernel


def _dt(plc, t):
    return plc.DataType(plc.TypeId(t))


def _rand(rng, n, t, nulls=0.0, shift=False):
    """Values of type id t with the edge values of the type mixed in; valid None or a bool array with `nulls` of them null."""
    dt = np.dtype(ob.NP[t])
    if dt == np.bool_:
        v = rng.random(n) < 0.5
    elif dt.kind == "f":
        v = (rng.normal(size=n) * 100).astype(dt)
        special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 0.5, -2.5, 1.0, 3.0], dt)
        pick = rng.random(n) < 0.2
        v[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    elif shift:
        v = rng.integers(0, 36, n).astype(dt)
    else:
        info = np.iinfo(dt)
        lo = -100 if info.min < 0 else 0
        v = rng.integers(lo, 100, n).astype(dt)
        special = np.array([info.min, info.max, 0, 1, info.max // 2 + 1], dtype=dt)
        if info.min < 0:
            special = np.concatenate([special, np.array([-1], dt)])
        pick = rng.random(n) < 0.1
        v[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    valid = (rng.random(n) >= nulls) if nulls else None
    return v, valid, t


def _plc_operand(plc, o):
    vals, valid, t = o
    if np.asarray(vals).ndim == 0:
        return plc.Scalar.from_py(vals.item() if valid else None, _dt(plc, t))
    return plc.Column.from_numpy(vals, valid, dtype=_dt(plc, t))  # chrono: the storage integers


def _ulps(a, b):
    """Distance in units in the last place between two float arrays of one dtype (equal NaNs and infinities: 0)."""
    it = np.int32 if a.dtype == np.float32 else np.int64
    ia, ib = a.view(it).astype(np.int64), b.view(it).astype(np.int64)
    ia = np.where(ia < 0, np.iinfo(it).min - ia, ia)
    ib = np.where(ib < 0, np.iinfo(it).min - ib, ib)
    d = np.abs(ia - ib)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    return np.where(same, 0, d)


def check(plc, op, lhs, rhs, out, what, lhs_col=None, rhs_col=None):
    """binary_operation(lhs, rhs, op, out) equals the oracle; lhs_col / rhs_col: plc operands to pass instead (sliced views)."""
    exp, exp_valid, defined, nullable = ob.binop(op, lhs, rhs, out)
    got = plc.binaryop.binary_operation(lhs_col or _plc_operand(plc, lhs), rhs_col or _plc_operand(plc, rhs), plc.binaryop.BinaryOperator(op),
                                        _dt(plc, out))
    assert int(got.type().id()) == out, what
    gv, gm = got.to_numpy()
    n = len(exp)
    assert got.size() == n, what
    assert (gm is not None) == nullable, (what, "mask", gm is not None, nullable)
    valid = np.ones(n, bool) if gm is None else gm
    assert np.array_equal(valid, exp_valid), (what, "validity", np.nonzero(valid != exp_valid)[0][:10])
    assert got.null_count() == int((~exp_valid).sum()), (what, "null_count")
    cmp = exp_valid & defined
    g, e = gv[cmp], exp[cmp]
    if op in ob.INEXACT_OPS and e.dtype.kind == "f":
        bad = _ulps(g, e) > 4
    elif op in ob.INEXACT_OPS and e.dtype.kind in "iu":
        # the double result within 4 ulp, then truncated: the integers may differ by that much, plus one
        ed = e.astype(np.float64)
        bad = np.abs(g.astype(np.float64) - ed) > 4 * np.spacing(np.abs(ed)) + 1
    elif e.dtype.kind == "f":
        bad = ~((g == e) | (np.isnan(g) & np.isnan(e)))
    else:
        bad = g != e
    assert not bad.any(), (what, np.nonzero(cmp)[0][np.nonzero(bad)[0][:5]], g[bad][:5], e[bad][:5])


def _raises(plc, op, lhs, rhs, out, exc=TypeError):
    with pytest.raises(exc):
        plc.binaryop.binary_operation(_plc_operand(plc, lhs), _plc_operand(plc, rhs), plc.binaryop.BinaryOperator(op), _dt(plc, out))


# (lhs, rhs, out) triples beyond the all-same ones: every compute type, mixed signed / unsigned / float, narrowing outputs
I8, I16, I32, I64, U8, U16, U32, U64, F32, F64, B8 = NUMERIC
MIXED = [(I8, I16, I32), (I32, U32, I64), (I64, U64, U64), (U8, I8, I16), (I64, F32, F64), (F32, F64, F32), (B8, I8, I32),
         (U16, U16, U8), (I32, I32, I64), (U64, I8, F64), (I64, I64, I8), (F64, I32, I32), (U32, I64, U32), (I16, U64, I64),
         (B8, B8, I32), (F32, I32, U8)]


def triples(op):
    same = [(t, t, B8 if op in ob.BOOL_OPS else t) for t in NUMERIC]
    mixed = [(a, b, B8 if op in ob.BOOL_OPS else o) for a, b, o in MIXED]
    return same + mixed


# ---- parity cases ------------------------------------------------------------------------------------------------------
def case_type_matrix(plc, small):
    """Every operator over the sampled type matrix, column by column, nulls on one side or the other; unsupported -> TypeError."""
    rng = np.random.default_rng(7)
    n = 200 if small else 3 * 32 * BLOCK + 45
    for op in ob.ALL_OPS:
        for i, (lt, rt, out) in enumerate(triples(op)):
            shift = op in (ob.SHIFT_LEFT, ob.SHIFT_RIGHT, ob.SHIFT_RIGHT_UNSIGNED)
            lhs = _rand(rng, n, lt, 0.15 if i % 2 == 0 else 0.0)
            rhs = _rand(rng, n, rt, 0.15 if i % 2 == 1 else 0.0, shift=shift)
            if ob.is_supported(out, lt, rt, op):
                check(plc, op, lhs, rhs, out, (op, lt, rt, out))
            else:
                _raises(plc, op, lhs, rhs, out)


def case_operand_forms(plc, small):
    """Column op scalar and scalar op column, valid and null scalars, with and without column nulls."""
    rng = np.random.default_rng(11)
    n = 300 if small else 2 * 32 * BLOCK * 4 + 17
    ops = [ob.ADD, ob.SUB, ob.DIV, ob.TRUE_DIV, ob.FLOOR_DIV, ob.PYMOD, ob.POW, ob.SHIFT_LEFT, ob.BITWISE_XOR, ob.LOGICAL_OR,
           ob.GREATER, ob.LESS_EQUAL, ob.NULL_EQUALS, ob.NULL_NOT_EQUALS, ob.NULL_MAX, ob.NULL_MIN, ob.NULL_LOGICAL_AND,
           ob.NULL_LOGICAL_OR]
    for op in ops:
        for lt, rt, out in [(I64, I64, I64), (F64, F64, F64), (I32, F32, F64), (U8, I32, I64), (B8, B8, B8), (I32, I32, I32)]:
            out = B8 if op in ob.BOOL_OPS else out
            if not ob.is_supported(out, lt, rt, op):
                continue
            for nulls in (0.0, 0.3):
                col_l, col_r = _rand(rng, n, lt, nulls), _rand(rng, n, rt, nulls, shift=op == ob.SHIFT_LEFT)
                for valid in (True, False):
                    sr = (np.asarray(_rand(rng, 1, rt, shift=op == ob.SHIFT_LEFT)[0][0]), valid, rt)
                    sl = (np.asarray(_rand(rng, 1, lt)[0][0]), valid, lt)
                    check(plc, op, col_l, sr, out, (op, lt, rt, "cs", nulls, valid))
                    check(plc, op, sl, col_r, out, (op, lt, rt, "sc", nulls, valid))


def case_sliced_views(plc, small):
    """Views whose offsets are not multiples of 32 (nor of the vector width), nulls in either operand, both paths."""
    rng = np.random.default_rng(13)
    n = 700 if small else 20000
    for lt, rt, out, op in [(I64, I64, I64, ob.ADD), (I32, I32, I32, ob.MUL), (F64, F64, B8, ob.GREATER), (I64, I32, I64, ob.SUB),
                            (F32, F32, F32, ob.NULL_MIN), (B8, B8, B8, ob.NULL_LOGICAL_OR), (I32, I32, B8, ob.LESS)]:
        lhs, rhs = _rand(rng, n, lt, 0.2), _rand(rng, n, rt, 0.1)
        lc, rc = _plc_operand(plc, lhs), _plc_operand(plc, rhs)
        for (lb, rb, m) in [(0, 0, n), (1, 1, n - 40), (33, 2, 300), (31, 45, n - 64), (4, 0, 129), (64, 32, n - 100)]:
            sl = (lhs[0][lb:lb + m], lhs[1][lb:lb + m], lt)
            sr = (rhs[0][rb:rb + m], rhs[1][rb:rb + m], rt)
            check(plc, op, sl, sr, out, (op, lb, rb, m), lhs_col=lc.slice(lb, lb + m), rhs_col=rc.slice(rb, rb + m))
            check(plc, op, sl, (np.asarray(rhs[0][0]), True, rt), out, (op, lb, "scalar"), lhs_col=lc.slice(lb, lb + m))


def case_lengths(plc, small):
    """Lengths around 32-row words, vector tiles (64 / 128 rows per warp) and 256-thread blocks, and empty columns."""
    rng = np.random.default_rng(17)
    lengths = [0, 1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025]
    if not small:
        lengths += [2047, 2048, 2049, 8 * 1024 - 1, 8 * 1024 + 1, 32 * BLOCK * 16 + 3]
    for n in lengths:
        for lt, rt, out, op, nulls in [(I64, I64, I64, ob.ADD, 0.0), (I32, I32, I32, ob.ADD, 0.25), (F64, F64, B8, ob.GREATER, 0.1),
                                       (B8, B8, B8, ob.LOGICAL_AND, 0.0), (I16, I16, B8, ob.NULL_EQUALS, 0.3)]:
            lhs, rhs = _rand(rng, n, lt, nulls), _rand(rng, n, rt, nulls)
            check(plc, op, lhs, rhs, out, (n, op))
            check(plc, op, lhs, (np.asarray(_rand(rng, 1, rt)[0][0]), True, rt), out, (n, op, "cs"))


def case_chrono(plc, small):
    """Timestamps and durations against the same type: comparisons, NULL_EQUALS / NULL_NOT_EQUALS, NULL_MAX / NULL_MIN."""
    rng = np.random.default_rng(19)
    n = 150 if small else 5000
    for t in range(12, 22):
        base = ob.NP[ob.storage(t)]
        lhs = (rng.integers(-50, 50, n).astype(base), rng.random(n) >= 0.2, t)
        rhs = (rng.integers(-50, 50, n).astype(base), rng.random(n) >= 0.2, t)
        for op in sorted(ob.COMPARISONS) + [ob.NULL_EQUALS, ob.NULL_NOT_EQUALS]:
            check(plc, op, lhs, rhs, B8, (t, op))
        for op in (ob.NULL_MAX, ob.NULL_MIN):
            check(plc, op, lhs, rhs, t, (t, op))
        check(plc, ob.LESS, lhs, (np.asarray(base(3)), True, t), B8, (t, "cs"))
        _raises(plc, ob.ADD, lhs, rhs, t)
        _raises(plc, ob.EQUAL, lhs, (rhs[0].astype(np.int64), rhs[1], ob.INT64), B8)
    _raises(plc, ob.EQUAL, (np.zeros(4, np.int64), None, 14), (np.zeros(4, np.int64), None, 13), B8)  # ms against s


def case_errors(plc, small):
    """Unsupported operators and types -> TypeError; differing sizes -> ValueError; a type id outside type_id -> RuntimeError."""
    a = (np.arange(10, dtype=np.int64), None, I64)
    f = (np.arange(10, dtype=np.float64), None, F64)
    _raises(plc, ob.GENERIC_BINARY, a, a, I64)
    _raises(plc, ob.BITWISE_AND, f, f, F64)
    _raises(plc, ob.SHIFT_RIGHT_UNSIGNED, (np.ones(10, bool), None, B8), (np.ones(10, bool), None, B8), B8)
    _raises(plc, ob.GREATER, a, a, I64)
    _raises(plc, ob.ADD, a, a, int(plc.TypeId.STRING))
    _raises(plc, ob.ADD, a, a, int(plc.TypeId.DECIMAL64))
    _raises(plc, ob.INVALID_BINARY, a, a, I64)
    _raises(plc, ob.ADD, a, (np.arange(9, dtype=np.int64), None, I64), I64, exc=ValueError)
    _raises(plc, ob.ADD, (np.asarray(np.int64(1)), True, I64), a, int(plc.TypeId.NUM_TYPE_IDS), exc=RuntimeError)
    with pytest.raises(ValueError):
        plc.binaryop.binary_operation(plc.Scalar.from_py(1, _dt(plc, I64)), plc.Scalar.from_py(1, _dt(plc, I64)),
                                      plc.binaryop.BinaryOperator.ADD, _dt(plc, I64))


def case_is_supported(plc, small):
    """is_supported_operation equals the oracle over every (op, out, lhs, rhs) of the numeric types and over the chrono ones."""
    B = plc.binaryop
    for op in range(35):
        for out in NUMERIC + [12, 23]:
            for lt in NUMERIC + ([12, 13, 17] if out in (B8, 12) else []):
                for rt in NUMERIC + [12, 13, 17]:
                    got = B.is_supported_operation(_dt(plc, out), _dt(plc, lt), _dt(plc, rt), B.BinaryOperator(op))
                    assert got == ob.is_supported(out, lt, rt, op), (op, out, lt, rt)


def case_filter(plc, small):
    """The end-to-end filter a query engine runs: binary_operation(col, scalar, GREATER, BOOL8), then apply_boolean_mask."""
    rng = np.random.default_rng(23)
    n = 1000 if small else 1_000_003
    price = rng.normal(size=n) * 10
    valid = rng.random(n) >= 0.1
    qty = rng.integers(0, 100, n).astype(np.int32)
    pc = plc.Column.from_numpy(price, valid)
    mask = plc.binaryop.binary_operation(pc, plc.Scalar.from_py(5.0, _dt(plc, F64)), plc.binaryop.BinaryOperator.GREATER,
                                         _dt(plc, B8))
    out = plc.stream_compaction.apply_boolean_mask(plc.Table([pc, plc.Column.from_numpy(qty)]), mask)
    keep = valid & (price > 5.0)
    got_p, _ = out.columns()[0].to_numpy()
    got_q, _ = out.columns()[1].to_numpy()
    assert np.array_equal(got_p, price[keep]) and np.array_equal(got_q, qty[keep])


PARITY = {
    "type matrix": case_type_matrix, "operand forms": case_operand_forms, "sliced views": case_sliced_views,
    "lengths": case_lengths, "chrono": case_chrono, "errors": case_errors, "is_supported": case_is_supported, "filter": case_filter,
}


@pytest.mark.parametrize("name", list(PARITY))
def test_parity(plc, name):
    PARITY[name](plc, False)


def test_golden(plc, case=None):
    for c in ([case] if case else CASES):
        lhs, rhs = golden_operand(c["lhs"]), golden_operand(c["rhs"])
        if "raises" in c:
            with pytest.raises({"ValueError": ValueError, "RuntimeError": RuntimeError}[c["raises"]]):
                plc.binaryop.binary_operation(_plc_operand(plc, lhs), _plc_operand(plc, rhs), plc.binaryop.BinaryOperator(c["op"]),
                                              plc.DataType(plc.TypeId(out_type(c))))
            continue
        got = plc.binaryop.binary_operation(_plc_operand(plc, lhs), _plc_operand(plc, rhs), plc.binaryop.BinaryOperator(c["op"]),
                                            plc.DataType(plc.TypeId(out_type(c))))
        vals, valid = got.to_numpy()
        valid = np.ones(len(vals), bool) if valid is None else valid
        assert [v.item() if ok else None for v, ok in zip(vals, valid)] == c["expect"], c["src"]

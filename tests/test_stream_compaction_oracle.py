"""CPU: the stream compaction oracle against the reference's known answers (tests/golden/stream_compaction_cases.py), and the
stream compaction kernels on the SIMT emulator (tests/emu) against the oracle."""
import numpy as np
import pytest

from oracle import stream_compaction as osc
from tests.golden.stream_compaction_cases import CASES
from tests.helpers import assert_columns_equal, make_col
from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (fixture)


def _cols(spec):
    return [make_col(vals, dt) for vals, dt in spec]


def canonical(cols):
    """Rows in a canonical order (by every column; null first, NaN last): `distinct` cases compare after this sort."""
    n = len(cols[0][0]) if cols else 0

    def key(i):
        out = []
        for v, m in cols:
            if m is not None and not m[i]:
                out.append((0, 0.0))
            else:
                x = float(v[i])
                out.append((2, 0.0) if np.isnan(x) else (1, x))
        return out
    return osc.gather(cols, sorted(range(n), key=key))


def run_case(case, ops, make_table, make_mask):
    """Runs one golden case through `ops` (the oracle or a binding's stream_compaction); returns (result, expected)."""
    t = make_table(_cols(case["table"]))
    op = case["op"]
    if op in ("apply_boolean_mask", "apply_deletion_mask"):
        got = getattr(ops, op)(t, make_mask(make_col(*case["mask"])))
    elif op in ("drop_nulls", "drop_nans"):
        got = getattr(ops, op)(t, case["keys"], case["threshold"])
    elif op == "unique":
        got = ops.unique(t, case["keys"], case["keep"], case["nulls_equal"])
    else:
        got = getattr(ops, op)(t, case["keys"], case["keep"], case["nulls_equal"], case["nans_equal"])
    exp = _cols(case["expected"])
    return got, exp


class _OracleOps:
    apply_boolean_mask = staticmethod(lambda t, m: osc.apply_boolean_mask(t, m))
    apply_deletion_mask = staticmethod(lambda t, m: osc.apply_boolean_mask(t, m, True))
    drop_nulls = staticmethod(osc.drop_nulls)
    drop_nans = staticmethod(osc.drop_nans)
    unique = staticmethod(osc.unique)
    stable_distinct = staticmethod(osc.stable_distinct)
    distinct = staticmethod(osc.stable_distinct)


def check_case(case, got, exp):
    if case["op"] == "distinct":
        got, exp = canonical(got), canonical(exp)
    assert len(got) == len(exp), case["src"]
    for j, (g, e) in enumerate(zip(got, exp)):
        assert_columns_equal(g, e, what=f"{case['src']} col {j}")


@pytest.mark.parametrize("case", CASES, ids=[c["src"] for c in CASES])
def test_oracle_golden(case):
    got, exp = run_case(case, _OracleOps, lambda cols: cols, lambda m: m)
    check_case(case, got, exp)


def test_oracle_distinct_semantics():
    k = make_col([1.0, -0.0, 0.0, float("nan"), float("nan"), None, None, 1.0], "float64")
    assert osc.distinct_indices([k], osc.KEEP_FIRST).tolist() == [0, 1, 3, 5]
    assert osc.distinct_indices([k], osc.KEEP_LAST).tolist() == [2, 4, 6, 7]
    assert osc.distinct_indices([k], osc.KEEP_NONE).tolist() == []
    assert osc.distinct_indices([k], osc.KEEP_NONE, nulls_equal=1).tolist() == [5, 6]
    assert osc.distinct_indices([k], osc.KEEP_NONE, nulls_equal=1, nans_equal=1).tolist() == [3, 4, 5, 6]


EMU_CODE = r"""
from oracle import stream_compaction as osc
sc = plc.stream_compaction
rng = np.random.default_rng(21)
def tab(cols):
    return plc.Table([plc.Column.from_numpy(v, m) for v, m in cols])
def check(t, exp, what):
    for j, (g, e) in enumerate(zip([c.to_numpy() for c in t.columns()], exp)):
        assert_columns_equal(g, e, what=f"{what} {j}")
for n in (1, 8191, 8193, 3 * 8192 + 5):
    v = rng.integers(0, 50, n).astype(np.int64); v.sort()
    f = (rng.integers(0, 5, n) * 0.5); f[rng.random(n) < 0.1] = np.nan; f[rng.random(n) < 0.1] = -0.0
    cols = [(v, rng.random(n) < 0.9), (f, rng.random(n) < 0.8), (np.arange(n, dtype=np.int32), None)]
    t = tab(cols)
    mv, mm = rng.random(n) < 0.5, rng.random(n) < 0.9
    check(sc.apply_boolean_mask(t, plc.Column.from_numpy(mv, mm)), osc.apply_boolean_mask(cols, (mv, mm)), (n, 'mask'))
    check(sc.drop_nulls(t, [0, 1], 1), osc.drop_nulls(cols, [0, 1], 1), (n, 'nulls'))
    check(sc.drop_nans(t, [1]), osc.drop_nans(cols, [1]), (n, 'nans'))
    for keep in (1, 2, 3):
        for ne in (0, 1):
            check(sc.unique(t, [0], sc.DuplicateKeepOption(keep), plc.NullEquality(ne)), osc.unique(cols, [0], keep, ne), (n, 'unique', keep, ne))
            for keys in ([0], [0, 1]):
                for nan in (0, 1):
                    got = sc.stable_distinct(t, keys, sc.DuplicateKeepOption(keep), plc.NullEquality(ne), plc.NanEquality(nan))
                    check(got, osc.stable_distinct(cols, keys, keep, ne, nan), (n, 'distinct', keys, keep, ne, nan))
print('COMPACTION_OK')
"""


def test_emu_stream_compaction(emu_lib):  # noqa: F811
    """compact_kernel (several tiles: the look-back), unique_flags_kernel and the distinct insert / mark kernels with packed
    (8-byte) and wide (16-byte) keys, on the emulator."""
    run(EMU_CODE, "COMPACTION_OK")

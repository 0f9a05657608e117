"""CPU: the replacement oracle (tests/replace_oracle.py) against the reference's known answers (tests/golden/replace_cases.py),
errors included; tests/test_replace_gpu.py holds the library to the same answers and to the oracle on the GPU."""
import numpy as np
import pytest

from tests import replace_oracle as orp
from tests import unary_oracle as ou
from tests.golden.replace_cases import CASES

ERRORS = {"TypeError": TypeError, "RuntimeError": RuntimeError}


def _array(values, dt):
    """values as dtype dt; integers through int64, so negative values wrap into the unsigned types as the typed tests' do"""
    if not values:
        return np.zeros(0, dt)
    return np.array(values, np.float64 if np.dtype(dt).kind == "f" else np.int64).astype(dt)


def golden_args(c, t):
    """The case's arguments for type t: oracle columns (values, valid, type), Scalars, or a replace policy."""
    out = []
    for a in c["args"]:
        if isinstance(a, int):
            out.append(a)
        elif "col" in a:
            at = a["type"] or t
            vals = _array(a["col"], ou.NP[at])
            out.append((vals, None if a["valid"] is None else np.array(a["valid"], bool), at))
        else:
            out.append(orp.Scalar(a["scalar"], a["valid"], a["type"] or t))
    return out


def oracle_call(fn, args):
    if fn == "replace_nulls":
        r = args[1]
        if isinstance(r, int):
            return orp.replace_nulls_policy(args[0], r)
        return orp.replace_nulls_scalar(args[0], r) if isinstance(r, orp.Scalar) else orp.replace_nulls_column(args[0], r)
    if fn == "replace_nans":
        return orp.replace_nans(*args)
    if fn == "find_and_replace_all":
        return orp.find_and_replace_all(*args)
    if fn == "clamp":
        if len(args) == 3:
            col, lo, hi = args
            return orp.clamp(col, lo, lo, hi, hi)
        return orp.clamp(*args)
    return orp.normalize_nans_and_zeros(*args)


def expected(c, t):
    dt = ou.NP[t]
    vals = _array(c["expect"], dt)
    valid = np.ones(len(vals), bool) if c["expect_valid"] is None else np.array(c["expect_valid"], bool)
    return vals, valid


def same(vals, valid, c, t):
    """(vals, valid) of a result equal the case's answer at valid rows (bit for bit where the case says so)."""
    ev, em = expected(c, t)
    m = np.ones(len(vals), bool) if valid is None else valid
    assert np.array_equal(m, em), (c["src"], t, "validity")
    if c["bitwise"]:
        assert np.array_equal(vals[m].view(np.uint8), ev[m].view(np.uint8)), (c["src"], t)
    else:
        assert np.array_equal(vals[m], ev[m], equal_nan=vals.dtype.kind == "f"), (c["src"], t, vals, ev)


@pytest.mark.parametrize("c", CASES, ids=[c["src"] for c in CASES])
def test_oracle_matches_golden(c):
    for t in c["types"]:
        args = golden_args(c, t)
        if c["raises"]:
            with pytest.raises(ERRORS[c["raises"]]):
                oracle_call(c["fn"], args)
            continue
        same(*oracle_call(c["fn"], args), c, t)

"""Sort-based groupby path (cpp/src/groupby/sort/aggregate.cpp): MEDIAN / NUNIQUE / NTH_ELEMENT (no hash implementation in the
reference either), pre-sorted keys, and the hash path's aggregations recomputed through the sort path (B2_GROUPBY_SORT=1).
Golden vectors: cpp/tests/groupby/{median_tests.cpp:25-42, nunique_tests.cpp:25-45, nth_element_tests.cpp:23-122}."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.helpers import assert_columns_equal
from tests.impls import OracleImpl, PlcImpl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = np.array([1, 2, 3, 1, 2, 2, 1, 3, 3, 2], np.int32)
VALS = np.arange(10)


def _one(impl, keys, vals, kind, valid=None):
    k, r = impl.groupby([(keys, None)], [((vals, valid), [kind])])
    return k[0], r[0][0]


@pytest.mark.parametrize("which", ["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def test_golden_median_nunique_nth(request, which):
    impl = OracleImpl() if which == "oracle" else PlcImpl(request.getfixturevalue("plc"))
    for vdt in (np.int8, np.int32, np.int64, np.float32, np.float64, np.uint16):
        v = VALS.astype(vdt)
        k, (out, m) = _one(impl, KEYS, v, "median")
        assert k[0].tolist() == [1, 2, 3] and out.dtype == np.float64 and out.tolist() == [3.0, 4.5, 7.0] and (m is None or m.all())
        k, (out, m) = _one(impl, KEYS, v, "nunique")
        assert out.dtype == np.int32 and out.tolist() == [3, 4, 3]
        for n, exp in ((0, [0, 1, 2]), (1, [3, 4, 7]), (2, [6, 5, 8]), (-1, [6, 9, 8]), (-2, [3, 5, 7]), (-3, [0, 4, 2])):
            k, (out, m) = _one(impl, KEYS, v, f"nth{n}")
            assert out.dtype == np.dtype(vdt) and out.tolist() == exp and (m is None or m.all())
        v2 = np.array([0, 1, 2, 3, 4, 5, 3, 2, 2, 9]).astype(vdt)
        k, (out, m) = _one(impl, KEYS, v2, "nth3")            # basic_out_of_bounds: {null, 9, null}
        assert m.tolist() == [False, True, False] and out[1] == 9
        k, (out, m) = _one(impl, KEYS, v2, "nth-4")           # negative_out_of_bounds: {null, 1, null}
        assert m.tolist() == [False, True, False] and out[1] == 1
    # nunique basic_duplicates (nunique_tests.cpp:62-80): vals {0, 1, 2, 3, 4, 5, 3, 2, 2, 9} -> {2, 4, 1}
    k, (out, m) = _one(impl, KEYS, np.array([0, 1, 2, 3, 4, 5, 3, 2, 2, 9], np.int32), "nunique")
    assert out.tolist() == [2, 4, 1]
    # empty input
    k, (out, m) = _one(impl, KEYS[:0], VALS[:0].astype(np.int32), "median")
    assert len(k[0]) == 0 and len(out) == 0 and out.dtype == np.float64


@pytest.mark.gpu
def test_random_vs_oracle(plc):
    rng = np.random.default_rng(17)
    cu, o = PlcImpl(plc), OracleImpl()
    for n, G in ((1, 1), (500, 7), (20_000, 300), (30_000, 9000)):
        for vdt in (np.int32, np.int64, np.float64, np.float32, np.uint8):
            k = rng.integers(0, G, n).astype(np.int64)
            if np.dtype(vdt).kind == "f":
                v = (rng.standard_normal(n) * 5).round(0).astype(vdt)
                v[rng.random(n) < 0.02] = np.nan
                v[rng.random(n) < 0.02] = -0.0
            else:
                v = rng.integers(0, 40, n).astype(vdt)
            valid = rng.random(n) < 0.85
            kinds = ["nunique", "nth0", "nth-1", "nth2", "count", "count_all", "median"]
            gk, gr = cu.groupby([(k, None)], [((v, valid), kinds)])
            ek, er = o.groupby([(k, None)], [((v, valid), kinds)])
            assert_columns_equal(gk[0], ek[0], what="keys")   # the sort path returns the groups in ascending key order, like the oracle
            for j, kind in enumerate(kinds):
                # MEDIAN too is exact: the oracle interpolates with the reference's formula, NaN ranked last
                assert_columns_equal(gr[0][j], er[0][j], what=f"{kind} {vdt}")
    # null keys: excluded / one group
    k, km = rng.integers(0, 5, 2000).astype(np.int32), rng.random(2000) < 0.9
    v = rng.integers(0, 9, 2000).astype(np.int32)
    for inc in (False, True):
        gk, gr = cu.groupby([(k, km)], [((v, None), ["nunique", "median"])], include_nulls=inc)
        ek, er = o.groupby([(k, km)], [((v, None), ["nunique", "median"])], include_nulls=inc)
        assert_columns_equal(gk[0], ek[0], what="keys")
        assert_columns_equal(gr[0][0], er[0][0]); assert_columns_equal(gr[0][1], er[0][1])


@pytest.mark.gpu
def test_hash_aggregations_through_the_sort_path():
    """B2_GROUPBY_SORT=1: SUM / MIN / MAX / MEAN / COUNT / PRODUCT / SUM_OF_SQUARES / M2 / VARIANCE / STD on the sort-based path equal
    the oracle (the same checks as the hash path's tests, M2 / VARIANCE / STD in the sort path's two-pass form); also keys declared
    pre-sorted (sorted::YES)."""
    code = r"""
import os, sys
sys.path.insert(0, '.')
import numpy as np
import torch
if os.environ.get('B2_EMU_RUN') == '1' and not torch.cuda.is_available():
    from tests.emu.harness import install
    install()
import cudf_b200.pylibcudf as plc
from tests.helpers import assert_columns_equal
from tests.impls import OracleImpl, PlcImpl
cu, o = PlcImpl(plc), OracleImpl()
rng = np.random.default_rng(23)
for n, G in ((300, 5), (25_000, 400)):
    for vdt in (np.int32, np.int64, np.float64, np.uint16):
        k = rng.integers(0, G, n).astype(np.int32)
        v = (rng.standard_normal(n) * 3).astype(vdt) if np.dtype(vdt).kind == 'f' else rng.integers(0, 7, n).astype(vdt)
        valid = rng.random(n) < 0.9
        kinds = ["sum", "min", "max", "mean", "count", "count_all", "sum_of_squares", "m2", "var", "std", "var0"]
        for vm in (None, valid):
            gk, gr = cu.groupby([(k, None)], [((v, vm), kinds)])
            ek, er = o.groupby([(k, None)], [((v, vm), kinds)], sort_path=True)
            assert_columns_equal(gk[0], ek[0], what="keys")
            for j, kind in enumerate(kinds):
                assert_columns_equal(gr[0][j], er[0][j], rtol=1e-9, what=f"{kind} {vdt}")
print('SORT_PATH_OK')
"""
    env = dict(os.environ, B2_GROUPBY_SORT="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert "SORT_PATH_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-2500:]

"""CPU functional checks of the CUDA kernels on the SIMT emulator in tests/emu (test infrastructure, see
tests/emu/include/cuda_runtime.h): the library's .cu files are compiled as C++ and every kernel runs with fibers for
threads. This covers index arithmetic, barrier structure and protocol logic — in particular of the opt-in paths that
were written without hardware access — against the same oracle as the GPU parity tests. It says nothing about memory
ordering or speed; the `-m gpu` tests remain the parity gate.

Each case runs in a subprocess because tests/emu/harness.install() rebinds the ctypes entry points of the package.
"""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="the emulator build needs g++")

PRELUDE = r"""
import os, sys, ctypes as C
sys.path.insert(0, '.')
from tests.emu.harness import install
install()
import numpy as np
import cudf_b200.pylibcudf as plc
from cudf_b200 import _lib as L
from oracle import sort as osort, join as ojoin
from tests.helpers import assert_columns_equal
from tests.impls import OracleImpl, PlcImpl, sort_groups
cu, o = PlcImpl(plc), OracleImpl()
"""


@pytest.fixture(scope="module")
def emu_lib():
    sys.path.insert(0, ROOT)
    from tests.emu.build_emu import build

    return build()


def run(code: str, marker: str, env=None, timeout=900):
    e = dict(os.environ)
    for k in ("B2_JOIN_RADIX_CAPACITY", "B2_SORT_PLAN_READBACK_MIN", "B2_GROUPBY_PARTITION_ROWS", "B2_GROUPBY_SMEM_SLOTS", "B2_SORT_HYBRID", "B2_SORT_HYBRID_MIN", "B2_SORT_FIX_FAST", "B2_SORT_CARRY", "B2_JOIN_RADIX_ROWS", "B2_GROUPBY_EST", "B2_GROUPBY_EST_MIN", "B2_GROUPBY_EST_CAP", "B2_SORT_PORTION"):
        e.pop(k, None)
    e.update(env or {})
    r = subprocess.run([sys.executable, "-c", PRELUDE + code], capture_output=True, text=True, env=e, cwd=ROOT, timeout=timeout)
    assert marker in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


SORT_PAYLOAD = r"""
rng = np.random.default_rng(5)
for n in (1, 33, 6144, 6145, 20_003):
    for kdt in (np.int64, np.int32, np.uint16, np.float64):
        for vdt in (np.int64, np.float32):
            keys = (rng.standard_normal(n) * 50).astype(kdt)
            vals = rng.integers(0, 1 << 30, n).astype(vdt)
            for order in ((0, 1) if np.dtype(kdt).kind != 'f' else (0,)):
                got = plc.sorting.sort_by_key(plc.Table([plc.Column.from_numpy(vals)]), plc.Table([plc.Column.from_numpy(keys)]), [order], [])
                exp = osort.sort_by_key([(vals, None)], [(keys, None)], [order])[0][0]
                assert np.array_equal(got.columns()[0].to_numpy()[0], exp), (n, kdt, vdt, order)
print('SORT_PAYLOAD_OK')
"""


def test_emu_validated_paths(emu_lib):
    """The shipped kernels on the emulator: sort (multi-tile look-back, nulls, floats, multi-column, portions), join,
    groupby, scan / reduce / segmented reduce. Mostly a fidelity check of the emulator itself."""
    run(SORT_PAYLOAD + r"""
rng = np.random.default_rng(6)
n = 15_000
k = rng.integers(-50, 50, n).astype(np.int32); kv = rng.random(n) < 0.9
f = rng.standard_normal(n); f[::97] = np.nan; f[::89] = -0.0
for cols, order, prec in [([(k, kv)], [1], [0]), ([(f, None)], [0], [1]), ([(k, kv), (f, None)], [0, 1], [1, 0])]:
    got = plc.sorting.sorted_order(plc.Table([plc.Column.from_numpy(v, m) for v, m in cols]), order, prec).to_numpy()[0]
    assert np.array_equal(got, osort.sorted_order(cols, order, prec)), (order, prec)
l = [(rng.integers(0, 300, 5000).astype(np.int64), rng.random(5000) < 0.9)]
r = [(rng.integers(0, 300, 3000).astype(np.int64), None)]
for kind in ("inner_join", "left_join", "full_join"):
    for ne in (0, 1):
        got, exp = getattr(cu, kind)(l, r, ne), getattr(o, kind)(l, r, ne)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (kind, ne)
keys = [(rng.integers(0, 700, n).astype(np.int64), rng.random(n) < 0.95)]
vals = (rng.integers(-1000, 1000, n).astype(np.int32), rng.random(n) < 0.8)
kinds = ["sum", "min", "max", "count", "count_all"]
gk, gr = sort_groups(*cu.groupby(keys, [(vals, kinds)])); ek, er = sort_groups(*o.groupby(keys, [(vals, kinds)]))
assert_columns_equal(gk[0], ek[0], what="keys")
for j, kind in enumerate(kinds):
    assert_columns_equal(gr[0][j], er[0][j], what=kind)
x = (rng.integers(-100, 100, 70_000).astype(np.int64), rng.random(70_000) < 0.9)
assert_columns_equal(cu.scan(x, "sum"), o.scan(x, "sum"), what="scan")
assert cu.reduce(x, "sum", np.int64) == o.reduce(x, "sum", np.int64)
offs = np.sort(rng.integers(0, 70_000, 300)).astype(np.int32); offs[0] = 0
assert_columns_equal(cu.segmented_reduce(x, offs, "sum", np.int64), o.segmented_reduce(x, offs, "sum", np.int64), what="segmented")
print('VALIDATED_OK')
""", "VALIDATED_OK", env={"B2_SORT_PORTION": "12288"})


def test_emu_sort_carry_payload(emu_lib):
    run(SORT_PAYLOAD, "SORT_PAYLOAD_OK", env={"B2_SORT_CARRY": "1"})


def test_emu_sort_hybrid(emu_lib):
    """Partial LSD passes + segment fix-up (the default plan for large 64-bit key columns), including the overflow rerun."""
    from tests.snippets.hybrid_sort import CODE

    for env in ({"B2_SORT_FIX_FAST": "0"}, {"B2_SORT_CARRY": "0", "B2_SORT_FIX_FAST": "1"}, {"B2_SORT_PLAN_READBACK_MIN": "0"}):
        code = "SIZES = (3, 100, 2047, 2049, 6145, 20011)\n" + CODE
        if "B2_SORT_PLAN_READBACK_MIN" in env:  # skipped passes are not launched at all: the launch-count check does not apply
            code = code.replace("assert b > a + 8, (a, b)", "assert b > a, (a, b)")
        run(code, "HYBRID_OK", env=dict(env, B2_SORT_HYBRID_MIN="0"))


def test_emu_groupby_partitioned(emu_lib):
    """Partition + shared-memory aggregation path of the hash groupby, with and without shared-table overflow."""
    from tests.snippets.partitioned_groupby import CODE

    cases = "CASES = [(1, 1), (100, 7), (5000, 300), (40_000, 20_000), (60_000, 3)]\n"
    # B2_GROUPBY_EST: histogram-free partition pass (estimated bases); a forced tiny capacity exercises its overflow fallback
    for env in ({"B2_GROUPBY_EST": "0"}, {"B2_GROUPBY_EST": "0", "B2_GROUPBY_SMEM_SLOTS": "64"}, {"B2_GROUPBY_EST": "1", "B2_GROUPBY_EST_MIN": "1"},
                {"B2_GROUPBY_EST": "1", "B2_GROUPBY_EST_MIN": "1", "B2_GROUPBY_EST_CAP": "40"}):
        run(cases + CODE, "PGB_OK", env=dict(env, B2_GROUPBY_PARTITION_ROWS="1"))


def test_emu_sort_by_key_aliased_column(emu_lib):
    """sort_by_key(T, T): the values and the keys are the same column."""
    run(r"""
rng = np.random.default_rng(11)
for n in (1, 33, 6145, 20_003):
    for dt in (np.int64, np.int32, np.uint16, np.int8, np.uint64):
        keys = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
        for order in (0, 1):
            c = plc.Column.from_numpy(keys)
            got = plc.sorting.sort_by_key(plc.Table([c]), plc.Table([c]), [order], []).columns()[0].to_numpy()[0]
            exp = np.sort(keys, kind='stable')
            assert np.array_equal(got, exp[::-1] if order else exp), (n, dt, order)
print('ALIAS_OK')
""", "ALIAS_OK")


def test_emu_radix_inner_join(emu_lib):
    """Partitioned shared-memory join incl. the MIX partition kernels, multi-chunk partitions and packed / float keys."""
    code = r"""
rng = np.random.default_rng(78)
def check(l, r, tag, kinds=("inner_join",)):
    for kind in kinds:
        got, exp = getattr(cu, kind)(l, r), getattr(ojoin, kind)(l, r)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (tag, kind)
check([(rng.integers(0, 5000, 20_000), None)], [(rng.integers(0, 5000, 8_000), None)], 'int64')
check([(rng.integers(0, 90_000, 7_000), None)], [(rng.integers(0, 90_000, 9_000), None)], 'sparse', ("left_join", "full_join"))
b = rng.integers(0, 1000, 60_000); b[:40_000] = 424242
p = rng.integers(0, 1000, 80_000); p[:30] = 424242
check([(p, None)], [(b, None)], 'three chunks')
# packed two-column float key with -0 / NaN (row equality of the reference)
l = [(rng.integers(0, 50, 2000).astype(np.int32), None), (np.where(rng.random(2000) < 0.3, np.nan, -0.0).astype(np.float32), None)]
r = [(rng.integers(0, 50, 900).astype(np.int32), None), (np.where(rng.random(900) < 0.3, np.nan, 0.0).astype(np.float32), None)]
check(l, r, 'two columns, float specials')
# probe-side hot key: 150000 probe rows of one key -> its partition is split into three work items
p = rng.integers(0, 100_000, 200_000); p[:150_000] = 777
b = rng.integers(0, 100_000, 30_000); b[:5] = 777
check([(p, None)], [(b, None)], 'probe pieces')
# a left join whose hot probe key spans several pieces AND several build chunks
p = rng.integers(0, 100_000, 90_000); p[:70_000] = 555
b = rng.integers(0, 100_000, 40_000); b[:20_000] = 555
check([(p[:DUPN], None)], [(b, None)], 'dup x chunks', ("inner_join", "left_join"))
print('RADIX_JOIN_OK')
"""
    run("DUPN = 600\n" + code, "RADIX_JOIN_OK", env={"B2_JOIN_RADIX_ROWS": "1"})
    # output-size guess too small: the walk is repeated with the exact size (first case only: the emulator is slow)
    short = code[:code.index("check([(rng.integers(0, 90_000, 7_000)")] + "print('RADIX_JOIN_OK')\n"
    run(short, "RADIX_JOIN_OK", env={"B2_JOIN_RADIX_ROWS": "1", "B2_JOIN_RADIX_CAPACITY": "100"})


def test_emu_wide_keys(emu_lib):
    run(r"""
rng = np.random.default_rng(91)
for nl, nr in [(1, 1), (20_000, 7_000), (3_000, 50_000)]:
    l = [(rng.integers(0, 40, nl).astype(np.int64), None), (rng.integers(0, 30, nl).astype(np.int64), rng.random(nl) < 0.9)]
    r = [(rng.integers(0, 40, nr).astype(np.int64), None), (rng.integers(0, 30, nr).astype(np.int64), rng.random(nr) < 0.9)]
    for kind in ("inner_join", "left_join", "full_join"):
        for ne in (0, 1):
            got, exp = getattr(cu, kind)(l, r, ne), getattr(o, kind)(l, r, ne)
            assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), (nl, nr, kind, ne)
    assert cu.inner_join_size(l, r) == o.inner_join_size(l, r)
f = np.array([0.0, -0.0, np.nan, 1.5, np.nan, 2.0])
l = [(np.arange(6, dtype=np.int32) % 2, None), (f, None), (np.arange(6, dtype=np.int64) % 2, None)]
r = [(np.array([0, 1, 0, 1], np.int32), None), (np.array([-0.0, np.nan, np.nan, 1.5]), None), (np.array([0, 1, 0, 1], np.int64), None)]
got, exp = cu.inner_join(l, r), o.inner_join(l, r)
assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
n = 60_000
keys = [(rng.integers(0, 50, n).astype(np.int64), None), (rng.integers(-20, 20, n).astype(np.int64), rng.random(n) < 0.95)]
vals = (rng.integers(-1000, 1000, n).astype(np.int32), rng.random(n) < 0.8)
kinds = ["sum", "min", "max", "count", "count_all"]
for inc in (False, True):
    gk, gr = sort_groups(*cu.groupby(keys, [(vals, kinds)], include_nulls=inc))
    ek, er = sort_groups(*o.groupby(keys, [(vals, kinds)], include_nulls=inc))
    for a, b in zip(gk, ek):
        assert_columns_equal(a, b, what="keys")
    for j, kind in enumerate(kinds):
        assert_columns_equal(gr[0][j], er[0][j], what=kind)
nn = [(keys[0][0], None), (keys[1][0], None)]
gk, gr = cu.groupby_scan(nn, [(vals, ["sum", "count"])]); ek, er = o.groupby_scan(nn, [(vals, ["sum", "count"])])
for a, b in zip(gk, ek):
    assert_columns_equal(a, b, what="scan keys")
for j in range(2):
    assert_columns_equal(gr[0][j], er[0][j], what=f"scan {j}")
print('WIDE_OK')
""", "WIDE_OK")


def test_emu_staged_peer_scatter(emu_lib):
    """b2_partition_scatter_staged against b2_partition_scatter and a numpy stable partition ("peer" buffers are host arrays)."""
    run(r"""
rng = np.random.default_rng(12)
for n, P, dt in [(1, 1, np.int64), (17, 2, np.int64), (4096, 8, np.int64), (4097, 8, np.int32), (3 * 4096 + 5, 5, np.int64),
                 (20000, 128, np.int16), (9000, 3, np.uint8), (30000, 8, np.float64)]:
    keys = rng.integers(0, 1 << 20, n).astype(np.int64)
    vals = rng.integers(0, 100, n).astype(dt)
    splitters = np.sort(rng.integers(0, 1 << 20, max(P - 1, 0))).astype(np.int64)
    sp_buf = np.concatenate([splitters, np.zeros(8, np.int64)])
    kcol, vcol = plc.Column.from_numpy(keys), plc.Column.from_numpy(vals)
    ids = np.searchsorted(splitters, keys, side='right') if P > 1 else np.zeros(n, np.int64)
    for name in ("b2_partition_scatter", "b2_partition_scatter_staged"):
        plan, counts, kv = C.c_void_p(), (C.c_int64 * P)(), kcol._view()
        L.check(L.lib.b2_partition_plan_create(C.byref(kv), 0, C.c_void_p(sp_buf.ctypes.data) if P > 1 else None, P, None, C.byref(plan), counts))
        outs = [np.full(int(counts[b]) + 8, 113, dtype=dt) for b in range(P)]
        dest, cv = (C.c_void_p * P)(*[x.ctypes.data for x in outs]), vcol._view()
        L.check(getattr(L.lib, name)(plan, C.byref(cv), dest, None))
        L.lib.b2_partition_plan_free(plan)
        for b in range(P):
            assert int(counts[b]) == int((ids == b).sum())
            assert np.array_equal(outs[b][:int(counts[b])], vals[ids == b]), (name, n, P, b)
            assert (outs[b][int(counts[b]):] == 113).all(), (name, n, P, b, 'wrote past the bucket')
print('STAGED_OK')
""", "STAGED_OK")


def test_emu_cpp_api(emu_lib, tmp_path):
    """tests/cpp/api_smoke.cpp (the cudf:: header surface over the C ABI) linked against the emulator library."""
    exe = tmp_path / "api_smoke_emu"
    cmd = ["g++", "-std=c++17", f"-I{ROOT}/include", f"-I{ROOT}/tests/emu/include", f"{ROOT}/tests/cpp/api_smoke.cpp", "-o", str(exe),
           f"-L{os.path.dirname(str(emu_lib))}", "-lcudf_b200_emu", f"-Wl,-rpath,{os.path.dirname(str(emu_lib))}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert "CPP_API_OK" in r.stdout, r.stdout + r.stderr


def test_emu_late_suites(emu_lib):
    """The gpu-marked cases of tests/test_zzzz_match_context.py (match context, partitioned probes, finalize) and
    tests/test_zzzz_var_std.py (SUM_OF_SQUARES / M2 / VARIANCE / STD) and tests/test_zzzz_segmented_sort.py on the emulator."""
    e = dict(os.environ, B2_EMU_RUN="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_zzzz_match_context.py", "tests/test_zzzz_var_std.py",
                        "tests/test_zzzz_segmented_sort.py", "tests/test_zzzz_rank.py", "tests/test_zzzz_partitioning.py", "-q", "-m", "gpu",
                        "--deselect", "tests/test_zzzz_partitioning.py::test_dlpack_roundtrip",  # needs torch.cuda tensors
                        "-p", "no:cacheprovider"],
                       capture_output=True, text=True, env=e, cwd=ROOT, timeout=900)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]

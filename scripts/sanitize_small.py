"""Small invocations of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck):
   compute-sanitizer --tool racecheck python scripts/sanitize_small.py
Role of the reference's ci/run_compute_sanitizer_test.sh:12-13 for this library. Sizes span several tiles but stay small:
the sanitizer slows kernels down by orders of magnitude."""
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
os.environ.setdefault("B2_SORT_HYBRID_MIN", "0")
os.environ.setdefault("B2_GROUPBY_PARTITION_ROWS", "1")
os.environ.setdefault("B2_JOIN_RADIX_ROWS", "1")
import numpy as np

import cudf_b200.pylibcudf as plc
from oracle import join as ojoin
from oracle import sort as osort

rng = np.random.default_rng(1)
n = int(os.environ.get("B2_SAN_ROWS", "40000"))
k = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
v = rng.integers(0, 1 << 40, n).astype(np.int64)
kc, vc = plc.Column.from_numpy(k), plc.Column.from_numpy(v)
got = plc.sorting.sort_by_key(plc.Table([vc]), plc.Table([kc]), [0], []).columns()[0].to_numpy()[0]
assert np.array_equal(got, osort.sort_by_key([(v, None)], [(k, None)], [0])[0][0])
so = plc.sorting.sorted_order(plc.Table([kc]), [1], []).to_numpy()[0]
assert np.array_equal(so, osort.sorted_order([(k, None)], [1]))
m = rng.random(n) < 0.8
so = plc.sorting.sorted_order(plc.Table([plc.Column.from_numpy(k.astype(np.int32), m)]), [0], [1]).to_numpy()[0]
assert np.array_equal(so, osort.sorted_order([(k.astype(np.int32), m)], [0], [1]))
# join (partitioned path forced, then the hash table path)
lk, rk = rng.integers(0, 5000, n), rng.integers(0, 5000, n // 2)
for env in ("1", "0"):
    os.environ["B2_JOIN_RADIX_ROWS"] = env
    l, r = plc.join.inner_join(plc.Table([plc.Column.from_numpy(lk)]), plc.Table([plc.Column.from_numpy(rk)]), plc.NullEquality.EQUAL)
    g = ojoin.canonical(l.to_numpy()[0], r.to_numpy()[0])
    e = ojoin.inner_join([(lk, None)], [(rk, None)])
    assert np.array_equal(g[0], e[0]) and np.array_equal(g[1], e[1])
# groupby (partitioned path forced, then the global-table path)
gk = rng.integers(0, 700, n).astype(np.int64)
gv = rng.random(n)
for env in ("1", "0"):
    os.environ["B2_GROUPBY_PARTITION_ROWS"] = env
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_numpy(gk)]))
    keys_out, res = gb.aggregate([plc.groupby.GroupByRequest(plc.Column.from_numpy(gv), [plc.aggregation.sum(), plc.aggregation.count()])])
    o = np.argsort(keys_out.columns()[0].to_numpy()[0])
    assert np.array_equal(res[0].columns()[1].to_numpy()[0][o], np.bincount(gk, minlength=700)[np.unique(gk)])
# scan / reduce / segmented reduce / partition / pack
x = plc.Column.from_numpy(rng.integers(-100, 100, n).astype(np.int64), rng.random(n) < 0.9)
plc.reduce.scan(x, plc.aggregation.sum(), plc.reduce.ScanType.INCLUSIVE)
plc.reduce.reduce(x, plc.aggregation.sum(), plc.DataType(plc.TypeId.INT64))
t = plc.Table([kc, vc])
plc.partitioning.hash_partition(t, [0], 13)
plc.contiguous_split.unpack(plc.contiguous_split.pack(t))
# unary operations and casts: vector and generic paths, a sliced view, is_null / is_nan
xf = plc.Column.from_numpy(rng.normal(size=n), rng.random(n) < 0.9)
plc.unary.unary_operation(xf, plc.unary.UnaryOperator.SQRT)
plc.unary.unary_operation(xf.slice(3, n - 5), plc.unary.UnaryOperator.SIN)
plc.unary.unary_operation(x, plc.unary.UnaryOperator.NEGATE)
plc.unary.cast(x, plc.DataType(plc.TypeId.FLOAT64))
plc.unary.cast(xf, plc.DataType(plc.TypeId.INT32))
plc.unary.cast(plc.Column.from_numpy(k, dtype=plc.DataType(plc.TypeId.TIMESTAMP_NANOSECONDS)), plc.DataType(plc.TypeId.TIMESTAMP_DAYS))
plc.unary.is_null(x.slice(1, n - 1))
plc.unary.is_nan(xf)
print("SANITIZE_SMALL_OK")

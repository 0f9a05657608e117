"""Small driver for ncu captures of one operation (after one warm-up call):
  python scripts/profile_ops.py --op sort_by_key|sort|inner_join|groupby|scan [--rows N]
Other paths are selected with their environment switches (README), e.g. B2_SORT_CARRY=0, B2_JOIN_RADIX_ROWS=1."""
import argparse
import ctypes as C
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch

import cudf_b200.pylibcudf as plc
from cudf_b200 import _lib

ap = argparse.ArgumentParser()
ap.add_argument("--op", default="sort_by_key", choices=["sort_by_key", "sort_by_key_payload", "sort", "inner_join", "groupby", "scan"])
ap.add_argument("--rows", type=int, default=1 << 27)
ap.add_argument("--reps", type=int, default=1)
a = ap.parse_args()
n = a.rows


def fill(dtype, stream_id, kind=0, modulus=0):
    t = torch.empty(n, dtype=dtype, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(t.data_ptr()), n, 0x5EED0001, stream_id << 40, kind, modulus, _lib.stream_arg(None)))
    return t


keys = fill(torch.int64, 0)
kt = plc.Table([plc.Column.from_torch(keys)])
if a.op == "sort_by_key":
    fn = lambda: plc.sorting.sort_by_key(kt, kt, [0], [])
elif a.op == "sort_by_key_payload":
    pay = fill(torch.float64, 8, kind=1)
    pt = plc.Table([plc.Column.from_torch(pay)])
    fn = lambda: plc.sorting.sort_by_key(pt, kt, [0], [])
elif a.op == "sort":
    fn = lambda: plc.sorting.sort(kt, [0], [])
elif a.op == "inner_join":
    rk = fill(torch.int64, 1)
    lk = fill(torch.int64, 6)
    lk[::10] = rk[::10]
    L, R = plc.Table([plc.Column.from_torch(lk)]), plc.Table([plc.Column.from_torch(rk)])
    fn = lambda: plc.join.inner_join(L, R, plc.NullEquality.EQUAL)
elif a.op == "groupby":
    gk = fill(torch.int64, 9, kind=2, modulus=1_000_000)
    gv = fill(torch.float64, 8, kind=1)
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_torch(gk)]))
    reqs = [plc.groupby.GroupByRequest(plc.Column.from_torch(gv), [plc.aggregation.sum(), plc.aggregation.count()])]
    fn = lambda: gb.aggregate(reqs)
else:
    col = plc.Column.from_torch(keys)
    fn = lambda: plc.reduce.scan(col, plc.aggregation.sum(), plc.reduce.ScanType.INCLUSIVE)
for _ in range(1 + a.reps):
    out = fn()
    torch.cuda.synchronize()
print("done", a.op, n)

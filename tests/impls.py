"""Two implementations behind one tiny interface so that the same golden/parity cases run against the
oracle (CPU) and against the CUDA path through the pylibcudf-named shim (GPU)."""
from __future__ import annotations

import numpy as np

import oracle
from oracle import groupby as ogb
from oracle import join as ojoin
from oracle import reduce as ored

KINDS = {"sum": 0, "product": 2, "min": 3, "max": 4, "count": 5, "count_all": 6, "mean": 10, "sum_of_squares": 9, "m2": 11,
         "var": 12, "std": 13, "argmax": 16, "argmin": 17, "var0": (12, 0), "var2": (12, 2), "std0": (13, 0), "std2": (13, 2),
         "median": 14, "nunique": 18, "nth0": (19, 0), "nth1": (19, 1), "nth2": (19, 2), "nth3": (19, 3), "nth-1": (19, -1), "nth-2": (19, -2),
         "nth-3": (19, -3), "nth-4": (19, -4)}


class OracleImpl:
    name = "oracle"

    def inner_join(self, l, r, ne=0):
        return ojoin.inner_join(l, r, ne)

    def left_join(self, l, r, ne=0):
        return ojoin.left_join(l, r, ne)

    def full_join(self, l, r, ne=0):
        return ojoin.full_join(l, r, ne)

    def inner_join_size(self, l, r, ne=0):
        return ojoin.inner_join_size(l, r, ne)

    def match_counts(self, l, r, ne=0, kind="inner"):
        return ojoin.match_counts(l, r, ne, kind)

    def partitioned_join(self, l, r, ne=0, kind="inner", bounds=(0,)):
        """The whole join, however it is partitioned (the partitioned API must reproduce it)."""
        return getattr(ojoin, f"{kind}_join")(l, r, ne)

    def groupby(self, keys, requests, include_nulls=False, sort_path=None):
        k, res = ogb.aggregate(keys, [(c, [KINDS[x] for x in kinds]) for c, kinds in requests], 1 if include_nulls else 0, sort_path)
        return k, res

    def groupby_scan(self, keys, requests, include_nulls=False):
        return ogb.scan(keys, [(c, [KINDS[x] for x in kinds]) for c, kinds in requests], 1 if include_nulls else 0)

    def reduce(self, col, kind, out_dtype, init=None):
        return ored.reduce(col[0], col[1], KINDS[kind], out_dtype, init)

    def scan(self, col, kind, inclusive=True, include=False):
        return ored.scan(col[0], col[1], KINDS[kind], inclusive, 1 if include else 0)

    def segmented_reduce(self, col, offsets, kind, out_dtype, include=False, init=None):
        return ored.segmented_reduce(col[0], col[1], offsets, KINDS[kind], out_dtype, 1 if include else 0, init)


class PlcImpl:
    name = "cuda"

    def __init__(self, plc):
        self.plc = plc

    def _tbl(self, cols):
        return self.plc.Table([self.plc.Column.from_numpy(v, m) for v, m in cols])

    def _pairs(self, res):
        l, r = res
        return ojoin.canonical(l.to_numpy()[0], r.to_numpy()[0])

    def inner_join(self, l, r, ne=0):
        return self._pairs(self.plc.join.inner_join(self._tbl(l), self._tbl(r), ne))

    def left_join(self, l, r, ne=0):
        return self._pairs(self.plc.join.left_join(self._tbl(l), self._tbl(r), ne))

    def full_join(self, l, r, ne=0):
        return self._pairs(self.plc.join.full_join(self._tbl(l), self._tbl(r), ne))

    def inner_join_size(self, l, r, ne=0):
        hj = self.plc.join.HashJoin(self._tbl(r), ne)
        return hj.inner_join_size(self._tbl(l))

    def match_counts(self, l, r, ne=0, kind="inner"):
        hj = self.plc.join.HashJoin(self._tbl(r), ne)
        ctx = getattr(hj, f"{kind}_join_match_context")(self._tbl(l))
        return ctx._match_counts.to_numpy()[0]

    def partitioned_join(self, l, r, ne=0, kind="inner", bounds=(0,)):
        """match context -> one partitioned probe per [bounds[i], bounds[i+1]) -> concatenation (full: finalize)."""
        plc = self.plc
        hj = plc.join.HashJoin(self._tbl(r), ne)
        lt = self._tbl(l)
        ctx = getattr(hj, f"{kind}_join_match_context")(lt)
        n = lt.num_rows()
        cuts = sorted(set([0, n] + [b for b in bounds if 0 <= b <= n]))
        parts = [getattr(hj, f"partitioned_{kind}_join")(plc.join.JoinPartitionContext(ctx, a, b)) for a, b in zip(cuts[:-1], cuts[1:])]
        if kind == "full":
            lo, ro = plc.join.HashJoin.finalize_partitioned_full_join([p[0] for p in parts], [p[1] for p in parts], n, len(r[0][0]))
            return ojoin.canonical(lo.to_numpy()[0], ro.to_numpy()[0])
        ls = [p[0].to_numpy()[0] for p in parts] or [np.empty(0, np.int32)]
        rs = [p[1].to_numpy()[0] for p in parts] or [np.empty(0, np.int32)]
        return ojoin.canonical(np.concatenate(ls), np.concatenate(rs))

    def _agg(self, name):
        a = self.plc.aggregation
        if name in ("var0", "var2", "std0", "std2"):
            return (a.variance if name[0] == "v" else a.std)(int(name[-1]))
        if name.startswith("nth"):
            return a.nth_element(int(name[3:]))
        if name in ("median", "nunique"):
            return getattr(a, name)()
        return {"sum": a.sum, "min": a.min, "max": a.max, "mean": a.mean, "product": a.product, "sum_of_squares": a.sum_of_squares,
                "m2": a.m2, "var": a.variance, "std": a.std, "argmax": a.argmax, "argmin": a.argmin,
                "count": lambda: a.count(self.plc.NullPolicy.EXCLUDE), "count_all": lambda: a.count(self.plc.NullPolicy.INCLUDE)}[name]()

    def _gb(self, keys, requests, include_nulls, scan):
        plc = self.plc
        gb = plc.groupby.GroupBy(self._tbl(keys), plc.NullPolicy.INCLUDE if include_nulls else plc.NullPolicy.EXCLUDE)
        reqs = [plc.groupby.GroupByRequest(plc.Column.from_numpy(c[0], c[1]), [self._agg(k) for k in kinds]) for c, kinds in requests]
        k, res = (gb.scan if scan else gb.aggregate)(reqs)
        kcols = [c.to_numpy() for c in k.columns()]
        rcols = [[c.to_numpy() for c in t.columns()] for t in res]
        return kcols, rcols

    def groupby(self, keys, requests, include_nulls=False):
        return self._gb(keys, requests, include_nulls, False)

    def groupby_scan(self, keys, requests, include_nulls=False):
        return self._gb(keys, requests, include_nulls, True)

    def reduce(self, col, kind, out_dtype, init=None):
        plc = self.plc
        c = plc.Column.from_numpy(col[0], col[1])
        s = None
        if init is not None:
            s = plc.Scalar.from_py(init[0], c.type(), valid=init[1])
        out = plc.reduce.reduce(c, self._agg(kind), plc.DataType.from_numpy(out_dtype), s)
        v, ok = out._get()
        return (v if ok else None), ok

    def scan(self, col, kind, inclusive=True, include=False):
        plc = self.plc
        c = plc.Column.from_numpy(col[0], col[1])
        out = plc.reduce.scan(c, self._agg(kind), plc.reduce.ScanType.INCLUSIVE if inclusive else plc.reduce.ScanType.EXCLUSIVE,
                              plc.NullPolicy.INCLUDE if include else plc.NullPolicy.EXCLUDE)
        return out.to_numpy()

    def segmented_reduce(self, col, offsets, kind, out_dtype, include=False, init=None):
        plc = self.plc
        c = plc.Column.from_numpy(col[0], col[1])
        o = plc.Column.from_numpy(np.asarray(offsets, dtype=np.int32))
        s = None
        if init is not None:
            s = plc.Scalar.from_py(init[0], c.type(), valid=init[1])
        out = plc.reduce.segmented_reduce(c, o, self._agg(kind), plc.DataType.from_numpy(out_dtype),
                                          plc.NullPolicy.INCLUDE if include else plc.NullPolicy.EXCLUDE, s)
        return out.to_numpy()


def sort_groups(keys, results):
    """Canonical order for groupby output: sort groups by key (nulls first)."""
    from oracle import sort as osort

    order = osort.sorted_order(keys, [0] * len(keys), [1] * len(keys)) if keys and len(keys[0][0]) else np.empty(0, np.int32)
    take = lambda c: (np.asarray(c[0])[order], None if c[1] is None else np.asarray(c[1])[order])
    return [take(k) for k in keys], [[take(c) for c in per] for per in results]

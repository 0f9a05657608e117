"""Hash-groupby semantics: cpp/src/groupby/groupby.cu:40-71,220-259, hash/{groupby.cu,compute_groupby.cu,
extract_single_pass_aggs.cpp,hash_compound_agg_finalizer.cu,output_utils.cu}, device_aggregators.cuh:428-446,
result types cpp/include/cudf/detail/aggregation/aggregation.hpp:879-970; grouped scan:
cpp/src/groupby/sort/{scan.cpp,group_scan_util.cuh:77-128}. Output here is canonical: groups in sorted key
order (nulls first); the reference's order is arbitrary (groupby.hpp:148-150)."""
from __future__ import annotations

import numpy as np

from . import sort as osort

SUM, PRODUCT, MIN, MAX, COUNT_VALID, COUNT_ALL, MEAN = 0, 2, 3, 4, 5, 6, 10
ARGMAX, ARGMIN = 16, 17  # row index of the extreme value; the first row among ties (the reference leaves ties open)
SUM_OF_SQUARES, M2, VARIANCE, STD = 9, 11, 12, 13  # a kind may also be the pair (VARIANCE | STD, ddof); ddof defaults to 1
MEDIAN, NUNIQUE, NTH_ELEMENT = 14, 18, 19  # sort-based path only (cpp/src/groupby/sort/aggregate.cpp; group_quantiles.cu, group_nunique.cu,
# group_nth_element.cu); NTH_ELEMENT is the pair (NTH_ELEMENT, n), null_policy INCLUDE; NUNIQUE skips nulls; MEDIAN = 0.5 quantile, linear
EXCLUDE, INCLUDE = 0, 1


def _group_ids(key_cols, include_nulls):
    """-> (order of rows sorted by key (stable), group id per sorted row, keep mask per row)."""
    n = len(key_cols[0][0]) if key_cols else 0
    keep = np.ones(n, dtype=bool)
    if not include_nulls:
        for _, m in key_cols:
            if m is not None:
                keep &= np.asarray(m, dtype=bool)
    ranks = [osort._column_rank(v, m, osort.ASCENDING, osort.BEFORE) for v, m in key_cols]
    rows = np.nonzero(keep)[0]
    if len(rows) == 0:
        return rows, np.empty(0, dtype=np.int64), keep
    sub = [r[rows] for r in ranks]
    o = np.lexsort(tuple(reversed(sub))) if len(sub) > 1 else np.argsort(sub[0], kind="stable")
    rows = rows[o]
    stacked = np.stack([r[rows] for r in ranks], axis=1)
    new = np.ones(len(rows), dtype=bool)
    new[1:] = (stacked[1:] != stacked[:-1]).any(axis=1)
    gid = np.cumsum(new) - 1
    return rows, gid, keep


def result_dtype(kind, in_dtype):
    in_dtype = np.dtype(in_dtype)
    if isinstance(kind, tuple):
        kind = kind[0]
    if kind in (M2, VARIANCE, STD):
        return np.dtype(np.float64)  # aggregation.hpp:997-1013
    if kind == SUM or kind == PRODUCT or kind == SUM_OF_SQUARES:
        if in_dtype.kind in "iu" or in_dtype == np.bool_:
            return np.dtype(np.int64)  # aggregation.hpp:935-939: every integral source sums into int64
        return in_dtype
    if kind in (COUNT_VALID, COUNT_ALL, ARGMAX, ARGMIN, NUNIQUE):
        return np.dtype(np.int32)
    if kind == MEDIAN:
        return np.dtype(np.float64)
    if kind == MEAN:
        return np.dtype(np.float64)
    return in_dtype


def takes_sort_path(requests) -> bool:
    """cpp/src/groupby/groupby.cu:65-69: a request holding an aggregation without a hash implementation sends the whole call
    down the sort-based path (as do keys declared sorted, which the oracle is not told about)."""
    return any((k[0] if isinstance(k, tuple) else k) in (MEDIAN, NUNIQUE, NTH_ELEMENT) for _, kinds in requests for k in kinds)


def aggregate(key_cols, requests, null_handling=EXCLUDE, sort_path=None):
    """requests: list of ((values, valid), [kinds]).
    sort_path: M2 / VARIANCE / STD as the sort-based path computes them (two passes) rather than the hash path's one-pass
    formula; None decides as the reference's dispatch does (takes_sort_path).
    -> (key columns [(values, valid)], results[request][kind] = (values, valid | None))."""
    if sort_path is None:
        sort_path = takes_sort_path(requests)
    n = len(key_cols[0][0]) if key_cols else 0
    for (vals, _), _k in requests:
        if len(vals) != n:
            raise RuntimeError("Size mismatch between request values and groupby keys.")
    rows, gid, _ = _group_ids(key_cols, null_handling == INCLUDE)
    ng = int(gid[-1]) + 1 if len(gid) else 0
    first = np.nonzero(np.concatenate([[True], gid[1:] != gid[:-1]]))[0] if ng else np.empty(0, dtype=np.int64)
    out_keys = []
    for v, m in key_cols:
        kv = np.asarray(v)[rows[first]] if ng else np.empty(0, dtype=np.asarray(v).dtype)
        km = (np.asarray(m)[rows[first]] if m is not None else None) if ng else (None if m is None else np.empty(0, bool))
        out_keys.append((kv, km))
    results = []
    for (vals, valid), kinds in requests:
        vals = np.asarray(vals)
        v = vals[rows]
        m = np.ones(len(rows), bool) if valid is None else np.asarray(valid, dtype=bool)[rows]
        has_nulls = valid is not None and not np.asarray(valid).all()
        per = []
        vc = np.bincount(gid[m], minlength=ng).astype(np.int64) if ng else np.empty(0, np.int64)
        for kind in kinds:
            ddof = 1
            if isinstance(kind, tuple):
                kind, ddof = kind
            rdt = result_dtype(kind, vals.dtype)
            if kind in (SUM_OF_SQUARES, M2, VARIANCE, STD):
                # device_aggregators.cuh:309-321 (value * value in the SUM target type) and
                # cpp/src/groupby/common/m2_var_std.cu:35-62,150-196
                xv, xg = v[m], gid[m]
                sdt = np.dtype(np.float64) if vals.dtype.kind == "f" else np.dtype(np.int64)
                with np.errstate(over="ignore", invalid="ignore"):
                    sq = np.zeros(ng, dtype=sdt)
                    np.add.at(sq, xg, xv.astype(sdt) * xv.astype(sdt))
                    sm = np.zeros(ng, dtype=sdt)
                    np.add.at(sm, xg, xv.astype(sdt))
                    if kind == SUM_OF_SQUARES:
                        per.append((sq.astype(rdt), (vc > 0) if has_nulls else None))
                        continue
                    cnt = np.maximum(vc, 1).astype(np.float64)
                    df = vc - ddof
                    ok = (vc != 0) & (df > 0)
                    if sort_path:
                        # two passes in float64 (cpp/src/groupby/sort/group_m2.cu:34-58, group_std.cu:19-52): the group MEAN, then
                        # (x - mean)^2 per value, divided by (n - ddof) for VARIANCE / STD, summed; STD = sqrt(VARIANCE)
                        # the MEAN is the sort path's: SUM / COUNT_VALID (aggregate.cpp:275-298), with an integral SUM in (wrapping)
                        # int64, so a UINT64 value at or above 2^63 or a sum past 2^63 shifts the mean as in the reference
                        xd = xv.astype(np.float64)
                        s1 = sm.astype(np.float64)
                        d = xd - (s1 / cnt)[xg]
                        t = d * d
                        if kind != M2:
                            t = np.where(ok[xg], t / np.where(ok, df, 1)[xg], 0.0)
                        acc = np.zeros(ng)
                        np.add.at(acc, xg, t)
                        if kind == M2:
                            per.append((acc, None))
                            continue
                        var = np.where(ok, acc, 0.0)
                    else:
                        m2v = np.where(vc == 0, 0.0, sq.astype(np.float64) - sm.astype(np.float64) * sm.astype(np.float64) / cnt)
                        if kind == M2:
                            per.append((m2v, None))
                            continue
                        var = np.where(ok, m2v / np.where(ok, df, 1), 0.0)
                    out = var if kind == VARIANCE else np.sqrt(np.where(ok, var, 0.0))
                per.append((out, None if ok.all() else ok))
                continue
            if kind in (MEDIAN, NUNIQUE, NTH_ELEMENT):
                out = np.zeros(ng, dtype=rdt)
                ok = np.ones(ng, bool)
                for g in range(ng):
                    sel = gid == g
                    gv, gm = v[sel], m[sel]
                    if kind == NTH_ELEMENT:      # rows in input order inside the group (rows is a stable order)
                        idx = ddof if ddof >= 0 else len(gv) + ddof
                        if 0 <= idx < len(gv) and gm[idx]:
                            out[g] = gv[idx]
                        else:
                            ok[g] = False
                    elif kind == NUNIQUE:
                        x = gv[gm]
                        if x.dtype.kind == "f":
                            x = np.where(x == 0, 0.0, x)          # -0 == +0; np.unique treats NaNs as one value
                        out[g] = len(np.unique(x))
                    else:
                        # ranked in the value type (stable, -0 == +0, NaN last), then interpolate::linear
                        # (cpp/src/quantiles/quantiles_util.hpp:23-36,73-89): (1 - f) * a + f * b, each product rounded on its own
                        x = np.sort(gv[gm], kind="stable").astype(np.float64)
                        if len(x) == 0:
                            ok[g] = False
                        else:
                            pos = (len(x) - 1) * 0.5
                            lo, hi = int(np.floor(pos)), int(np.ceil(pos))
                            f = np.float64(pos - lo)
                            with np.errstate(invalid="ignore", over="ignore"):
                                out[g] = (np.float64(1.0) - f) * x[lo] + f * x[hi]
                per.append((out, None if (kind == NUNIQUE or ok.all()) else ok))
                continue
            if kind in (ARGMAX, ARGMIN):
                # global_memory_aggregator.cuh:155-200, in the order of MIN / MAX: NaN ranks above +inf and NaNs tie
                out = np.full(ng, -1, np.int32)
                xv, xg, xr = v[m], gid[m], rows[m]
                rank = lambda x: (1, 0.0) if x != x else (0, x)
                for val, g, r in zip(xv.tolist(), xg.tolist(), xr.tolist()):
                    h = out[g]
                    if h < 0:
                        out[g] = r
                        continue
                    a, b = rank(val), rank(vals[h].item())
                    if (a > b if kind == ARGMAX else a < b) or (a == b and r < h):
                        out[g] = r
                per.append((out, (vc > 0) if has_nulls else None))
                continue
            if kind == COUNT_ALL:
                per.append((np.bincount(gid, minlength=ng).astype(np.int32), None))
                continue
            if kind == COUNT_VALID:
                per.append((vc.astype(np.int32), None))
                continue
            out = np.zeros(ng, dtype=rdt)
            xv, xg = v[m], gid[m]
            with np.errstate(over="ignore", invalid="ignore"):
                if kind in (SUM, MEAN):
                    # MEAN = SUM / COUNT_VALID with SUM in its own target type (hash_compound_agg_finalizer.cu:95-131):
                    # integer sources accumulate in (wrapping) int64, floats in their type (float32 kept as float64 here)
                    sdt = result_dtype(SUM, vals.dtype)
                    acc = np.zeros(ng, dtype=np.float64 if sdt.kind == "f" else sdt)
                    np.add.at(acc, xg, xv.astype(acc.dtype))
                    out = (acc.astype(np.float64) / np.maximum(vc, 1)).astype(rdt) if kind == MEAN else acc.astype(rdt)
                elif kind == PRODUCT:
                    acc = np.ones(ng, dtype=np.float64 if rdt.kind == "f" else rdt)
                    np.multiply.at(acc, xg, xv.astype(acc.dtype))
                    out = acc.astype(rdt)
                elif kind == MIN:
                    # NaN ranks above +inf (fmin drops it while a number is there); MAX's np.maximum propagates it
                    big = np.full(ng, np.nan if rdt.kind == "f" else (np.iinfo(rdt).max if rdt != np.bool_ else True), dtype=rdt)
                    np.fmin.at(big, xg, xv)
                    out = big
                elif kind == MAX:
                    small = np.full(ng, -np.inf if rdt.kind == "f" else (np.iinfo(rdt).min if rdt != np.bool_ else False), dtype=rdt)
                    np.maximum.at(small, xg, xv)
                    out = small
                else:
                    raise ValueError("unsupported aggregation")
            ov = (vc > 0) if has_nulls else None
            per.append((out, ov))
        results.append(per)
    return out_keys, results


def scan(key_cols, requests, null_handling=EXCLUDE):
    """cudf::groupby::scan: rows in stable sorted key order; inclusive scan restarted per group."""
    from . import reduce as ored

    rows, gid, _ = _group_ids(key_cols, null_handling == INCLUDE)
    out_keys = [(np.asarray(v)[rows], None if m is None else np.asarray(m)[rows]) for v, m in key_cols]
    starts = np.nonzero(np.concatenate([[True], gid[1:] != gid[:-1]]))[0] if len(gid) else np.empty(0, np.int64)
    bounds = list(starts) + [len(rows)]
    results = []
    for (vals, valid), kinds in requests:
        vals = np.asarray(vals)
        v = vals[rows]
        m = None if valid is None else np.asarray(valid, dtype=bool)[rows]
        per = []
        for kind in kinds:
            rdt = result_dtype(kind, vals.dtype)
            out = np.zeros(len(rows), dtype=rdt)
            for b, e in zip(bounds[:-1], bounds[1:]):
                seg = v[b:e].astype(rdt) if kind not in (COUNT_VALID, COUNT_ALL) else v[b:e]
                r, _ = ored.scan(seg, None if m is None else m[b:e], kind, True, ored.EXCLUDE)
                out[b:e] = r
            per.append((out, m if kind not in (COUNT_VALID, COUNT_ALL) else None))
        results.append(per)
    return out_keys, results

"""Per-operation measurements behind bench.py's `ops` object: hash inner_join (BASELINE configs[2], index pairs and the
payload materialisation with 50 % nulls), groupby (configs[3]), scan / reduce / segmented reduce (SURVEY §8d C4b) and the
keys-only sort.  Every entry carries rows/s, a `roofline` object (algorithmic bytes of SURVEY §8d against the measured
HBM peak) and, where BASELINE.md §3 names one, a `cpu_baseline` (pandas on a bounded 1e7-row sample of the same
generator, timed on the host cores).  Data set-up uses torch ops; the timed region is the library through the
pylibcudf-named shim."""
from __future__ import annotations

import ctypes as C
import os
import time

SEED = 0x5EED0001


def _fill(_lib, t, n, stream_id, kind=0, modulus=0, seed=SEED):
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(t.data_ptr()), n, seed, stream_id << 40, kind, modulus, _lib.stream_arg(None)))
    return t


def _warm(torch, fn, warmup=2, limit=8):
    """At least `warmup` untimed calls, then more (up to `limit`) until two consecutive calls agree within 3 %: the first calls of
    an operation grow the stream-ordered memory pool, which is allocator warm-up, not the operation."""
    prev = None
    for i in range(limit):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        del out
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1)
        if i + 1 >= warmup and prev is not None and abs(t - prev) <= 0.03 * max(t, prev):
            break
        prev = t


def _time(torch, fn, steps=3, warmup=2):
    if warmup:
        _warm(torch, fn, warmup)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = fn()
        del out
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


# ------------------------------------------------------------------------------------------------
# CPU baselines (pandas; BASELINE.md §3) — the cpu_baseline leg may use oracle.datagen (same generator as the GPU fill)
# ------------------------------------------------------------------------------------------------
def _best(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def cpu_baselines(rows: int) -> dict:
    import numpy as np
    import pandas as pd

    from oracle import datagen

    out = {}
    cores = os.cpu_count()
    # join: 10 % of probe rows match exactly once; float64 payloads with 50 % nulls (NaN)
    rk = datagen.fill(rows, SEED, 1 << 40, 0)
    lk = datagen.fill(rows, SEED, 6 << 40, 0)
    u = datagen.fill(rows, SEED, 5 << 40, 1)
    sel = datagen.fill(rows, SEED, 4 << 40, 2, rows)
    hit = u < 0.10
    lk[hit] = rk[sel[hit]]
    pay = datagen.fill(rows, SEED, 8 << 40, 1)
    pay[~datagen.fill(rows, SEED, 3 << 40, 4)] = np.nan
    L = pd.DataFrame({"k": lk, "lp": pay})
    R = pd.DataFrame({"k": rk, "rp": pay[::-1].copy()})
    t = _best(lambda: pd.merge(L, R, on="k", how="inner"))
    out["inner_join"] = {"value": rows / t, "unit": "probe rows/s", "cores": 1, "kind": "port", "ms": t * 1e3,
                         "sample": f"pandas {pd.__version__} merge(how='inner') of {rows} x {rows} int64 keys, 10 % match rate, float64 payloads "
                                   f"with 50 % NaN, best of 3; host has {cores} logical cores"}
    del L, R, lk, rk, sel, hit, u
    # groupby: k = x mod 1e6, sum(float64) + count(int32)
    G = 1_000_000
    gk = datagen.fill(rows, SEED, 9 << 40, 2, G)
    v2 = datagen.fill(rows, SEED, 10 << 40, 3)
    df = pd.DataFrame({"k": gk, "v": datagen.fill(rows, SEED, 8 << 40, 1), "c": v2})
    t = _best(lambda: df.groupby("k").agg(v=("v", "sum"), c=("c", "count")))
    out["groupby"] = {"value": rows / t, "unit": "rows/s", "cores": 1, "kind": "port", "ms": t * 1e3,
                      "sample": f"pandas groupby('k').agg(sum(float64), count(int32)) on {rows} rows, {G} groups, best of 3; host has {cores} logical cores"}
    del df
    x = datagen.fill(rows, SEED, 7 << 40, 0)
    t = _best(lambda: np.cumsum(x))
    out["scan"] = {"value": rows / t, "unit": "rows/s", "cores": 1, "kind": "port", "ms": t * 1e3, "sample": f"numpy cumsum of {rows} int64, best of 3"}
    t = _best(lambda: np.sum(x))
    out["reduce"] = {"value": rows / t, "unit": "rows/s", "cores": 1, "kind": "port", "ms": t * 1e3, "sample": f"numpy sum of {rows} int64, best of 3"}
    # stream compaction: {int64, float64 with 50 % NaN} frame, 50 % boolean mask; drop_duplicates of the groupby key
    u = datagen.fill(rows, SEED, 8 << 40, 1)
    df = pd.DataFrame({"x": x, "p": np.where(datagen.fill(rows, SEED, 3 << 40, 4), u, np.nan)})
    keep = u < 0.5
    t = _best(lambda: df[keep])
    out["apply_boolean_mask"] = {"value": rows / t, "unit": "rows/s", "cores": 1, "kind": "port", "ms": t * 1e3,
                                 "sample": f"pandas boolean indexing of {rows} rows (int64 + float64 with 50 % NaN), 50 % mask, best of 3"}
    t = _best(lambda: df.dropna(subset=["p"]))
    out["drop_nulls"] = {"value": rows / t, "unit": "rows/s", "cores": 1, "kind": "port", "ms": t * 1e3,
                         "sample": f"pandas dropna(subset=['p']) of {rows} rows, 50 % NaN, best of 3"}
    ks = pd.Series(gk)
    t = _best(lambda: ks.drop_duplicates())
    out["distinct"] = {"value": rows / t, "unit": "rows/s", "cores": 1, "kind": "port", "ms": t * 1e3,
                       "sample": f"pandas Series.drop_duplicates of {rows} int64 keys with {G} values, best of 3"}
    return out


# ------------------------------------------------------------------------------------------------
# GPU measurements
# ------------------------------------------------------------------------------------------------
def run(plc, _lib, n, peak_gbs, cpu_rows=10_000_000, with_cpu=True):
    import torch

    res = {}
    dev = "cuda"
    cpu = cpu_baselines(cpu_rows) if with_cpu else {}

    def phases(*names):
        return {k_: _lib.profile_get(k_)[0] / max(_lib.profile_get(k_)[1], 1) for k_ in names if _lib.profile_get(k_)[1]}

    def entry(ms, rows, alg_bytes, cpu_key=None, unit="rows/s", **kw):
        gbs = alg_bytes / (ms / 1e3) / 1e9
        e = dict(ms=ms, value=rows / (ms / 1e3), unit=unit,
                 roofline={"bound": "hbm", "achieved": gbs, "peak": peak_gbs, "unit": "GB/s", "frac": gbs / peak_gbs,
                           "algorithmic_bytes": alg_bytes, "peak_source": "MEASURED_PEAKS.json hbm_gbs (or the H100 SXM data sheet's 3.35 TB/s)"}, **kw)
        if cpu_key and cpu_key in cpu:
            e["cpu_baseline"] = cpu[cpu_key]
        return e

    def release():
        """Hand every cached block back to the driver (torch's caching allocator and the library's pool): the next operation
        starts from the same memory state whatever ran before it (deleted tensors still cached by torch otherwise slow the
        allocations of the next operation's temporaries)."""
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        _lib.check(_lib.lib.b2_trim_pool())

    def profiled(fn, steps=3, warmup=2):
        _warm(torch, fn, warmup)
        _lib.lib.b2_profile_reset()
        _lib.lib.b2_profile_enable(1)
        ms = _time(torch, fn, steps=steps, warmup=0)
        _lib.lib.b2_profile_enable(0)
        return ms

    # ---- scan / reduce / segmented reduce (int64 and float64) ----
    release()
    x = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 7)
    f = _fill(_lib, torch.empty(n, dtype=torch.float64, device=dev), n, 8, kind=1)
    ci, cf = plc.Column.from_torch(x), plc.Column.from_torch(f)
    agg = plc.aggregation
    res["scan_sum_int64"] = entry(_time(torch, lambda: plc.reduce.scan(ci, agg.sum(), plc.reduce.ScanType.INCLUSIVE)), n, 16 * n, "scan")
    res["scan_sum_float64"] = entry(_time(torch, lambda: plc.reduce.scan(cf, agg.sum(), plc.reduce.ScanType.INCLUSIVE)), n, 16 * n)
    res["reduce_sum_int64"] = entry(_time(torch, lambda: plc.reduce.reduce(ci, agg.sum(), plc.DataType(plc.TypeId.INT64))), n, 8 * n, "reduce")
    res["reduce_sum_float64"] = entry(_time(torch, lambda: plc.reduce.reduce(cf, agg.sum(), plc.DataType(plc.TypeId.FLOAT64))), n, 8 * n)
    ti = plc.Table([ci])
    ms = profiled(lambda: plc.sorting.sort(ti, [plc.Order.ASCENDING], []))
    res["sort_single_int64_keys_only"] = entry(ms, n, 136 * n, note="cudf::sort of one int64 column; contract bytes: histogram 8 + 8 passes x 16 B/row",
                                               phases_ms=phases("histogram", "onesweep", "segment_fix"))
    ms = profiled(lambda: plc.sorting.sorted_order(ti, [plc.Order.ASCENDING], []))
    res["sorted_order_int64"] = entry(ms, n, 196 * n, note="cudf::sorted_order; contract bytes: histogram 8 + 20 + 7 x 24 B/row",
                                      phases_ms=phases("histogram", "onesweep", "segment_fix"))
    del ti
    S = 1_000_000
    offs = torch.linspace(0, n, S + 1, device=dev).to(torch.int32)
    co = plc.Column.from_torch(offs)
    res["segmented_reduce_sum_float64_1e6_segments"] = entry(
        _time(torch, lambda: plc.reduce.segmented_reduce(cf, co, agg.sum(), plc.DataType(plc.TypeId.FLOAT64))), n, 8 * n + 4 * (S + 1) + 8 * S)
    del x, ci, offs, co
    release()

    # ---- groupby (BASELINE configs[3]): int64 key with 1e6 groups, sum(float64) + count(int32) ----
    G = 1_000_000
    k = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 9, kind=2, modulus=G)
    v2 = _fill(_lib, torch.empty(n, dtype=torch.int32, device=dev), n, 10, kind=3)
    gb = plc.groupby.GroupBy(plc.Table([plc.Column.from_torch(k)]))
    reqs = [plc.groupby.GroupByRequest(cf, [agg.sum()]), plc.groupby.GroupByRequest(plc.Column.from_torch(v2), [agg.count()])]
    ms = profiled(lambda: gb.aggregate(reqs))
    keys_out, _ = gb.aggregate(reqs)
    res["groupby_sum_count_1e6_groups"] = entry(ms, n, 16 * n + 20 * G, "groupby", groups=keys_out.num_rows(),
                                                phases_ms=phases("groupby_partition", "groupby_aggregate"),
                                                note="partition pass (one-sweep, mix64 top byte, value carried) + shared-memory aggregation per partition chunk")
    del k, v2, gb, reqs, keys_out
    release()

    # ---- stream compaction: {int64, float64 with 50 % nulls} table filtered by a 50 % BOOL8 mask / by its nulls; distinct on the
    # groupby workload's key column (1e6 values) ----
    x = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 7)
    vmask = _fill(_lib, torch.empty((n + 31) // 32, dtype=torch.int32, device=dev), n, 3, kind=4)
    pcol = plc.Column.from_torch(f, mask=vmask)
    tbl = plc.Table([plc.Column.from_torch(x), pcol])
    bm = f < 0.5
    mcol = plc.Column.from_torch(bm)
    sc = plc.stream_compaction
    sw = 16  # bytes per row of the two columns
    ms = profiled(lambda: sc.apply_boolean_mask(tbl, mcol))
    s_ = sc.apply_boolean_mask(tbl, mcol).num_rows()
    res["apply_boolean_mask_50pct"] = entry(ms, n, n * (1 + sw) + s_ * sw + n // 8 + s_ // 8, "apply_boolean_mask", kept=s_,
                                            phases_ms=phases("compact", "gather"),
                                            note="int64 + float64 (50 % nulls) table, 50 % BOOL8 mask; contract bytes: n(1 + 16) + 16s + validity in and out")
    ms = profiled(lambda: sc.drop_nulls(tbl, [1]))
    s_ = sc.drop_nulls(tbl, [1]).num_rows()
    res["drop_nulls_50pct"] = entry(ms, n, n // 8 + n * sw + s_ * sw + s_ // 8, kept=s_, cpu_key="drop_nulls", phases_ms=phases("compact", "gather"),
                                    note="same table, key = the float64 column; contract bytes: validity n/8 + 16n + 16s + s/8")
    del tbl, pcol, mcol, bm, vmask, x
    release()
    k = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 9, kind=2, modulus=G)
    kt = plc.Table([plc.Column.from_torch(k)])
    args = (sc.DuplicateKeepOption.KEEP_ANY, plc.NullEquality.EQUAL, plc.NanEquality.ALL_EQUAL)
    ms = profiled(lambda: sc.distinct(kt, [0], *args))
    d = sc.distinct(kt, [0], *args).num_rows()
    res["distinct_1e6_keys"] = entry(ms, n, 8 * n + 2 * n + 4 * d + 8 * d, "distinct", distinct_rows=d,
                                     phases_ms=phases("distinct_insert", "distinct_mark", "compact", "gather"),
                                     note="KEEP_ANY on the groupby key column; contract bytes: keys 8n + flags 2n + map 4d + keys out 8d")
    del k, kt
    release()

    # ---- inner join (BASELINE configs[2]): |R| = |L| = n, 10 % of probe rows match exactly once; payload gather with 50 % nulls ----
    try:
        rk = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 1)
        lk = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 6)          # fresh keys (match prob ~ 0)
        u = _fill(_lib, torch.empty(n, dtype=torch.float64, device=dev), n, 5, kind=1)
        sel = _fill(_lib, torch.empty(n, dtype=torch.int64, device=dev), n, 4, kind=2, modulus=n)
        hit = u < 0.10
        del u
        lk[hit] = rk[sel[hit]]
        del sel, hit
        release()
        L, R = plc.Table([plc.Column.from_torch(lk)]), plc.Table([plc.Column.from_torch(rk)])
        slots = 1 << (2 * n - 1).bit_length()
        ms = profiled(lambda: plc.join.inner_join(L, R, plc.NullEquality.EQUAL), steps=3, warmup=2)
        li, ri = plc.join.inner_join(L, R, plc.NullEquality.EQUAL)
        M = li.size()
        alg = 16 * slots + 24 * n + 24 * n + 8 * M
        res["inner_join_10pct"] = entry(ms, n, alg, "inner_join", unit="probe rows/s", matches=M,
                                        phases_ms=phases("join_build", "join_count", "join_retrieve", "rjoin_partition", "rjoin_join"),
                                        note="contract bytes (SURVEY §8d C3): 16 B x 2|R| slots + 24|R| + 24|L| + 8M")
        # both join paths forced on the same inputs (B2_JOIN_RADIX_ROWS: 0 = open-addressing table in HBM, <rows> = partitioned
        # shared-memory join for inputs of at least that many rows; unset = the library's default choice, measured above)
        prev = os.environ.get("B2_JOIN_RADIX_ROWS")
        for label, val in (("inner_join_10pct_hash_table_path", "0"), ("inner_join_10pct_partitioned_path", "1000000")):
            os.environ["B2_JOIN_RADIX_ROWS"] = val
            try:
                release()
                rms = profiled(lambda: plc.join.inner_join(L, R, plc.NullEquality.EQUAL), steps=2, warmup=1)
                li2, _ri2 = plc.join.inner_join(L, R, plc.NullEquality.EQUAL)
                res[label] = entry(rms, n, alg, unit="probe rows/s", matches=li2.size(), same_match_count=bool(li2.size() == M),
                                   phases_ms=phases("join_build", "join_count", "join_retrieve", "rjoin_partition", "rjoin_join"))
                del li2, _ri2
            except Exception as ex:
                res[label] = {"error": repr(ex)[:200]}
        if prev is None:
            os.environ.pop("B2_JOIN_RADIX_ROWS", None)
        else:
            os.environ["B2_JOIN_RADIX_ROWS"] = prev
        # materialisation: gather both payload columns (float64, 50 % nulls) through the index columns
        release()
        pay = f
        nwords = (n + 31) // 32
        mask = _fill(_lib, torch.empty(nwords, dtype=torch.int32, device=dev), n, 3, kind=4)
        pcol = plc.Column.from_torch(pay, mask=mask)
        pt = plc.Table([pcol])
        gms = _time(torch, lambda: (plc.copying.gather(pt, li, plc.OutOfBoundsPolicy.DONT_CHECK), plc.copying.gather(pt, ri, plc.OutOfBoundsPolicy.DONT_CHECK)), steps=2, warmup=1)
        res["inner_join_materialise_payloads"] = entry(gms, M, 2 * M * (4 + 8 + 8) + 2 * M // 4, unit="output rows/s", null_fraction=pcol.null_count() / n,
                                                       note="gather of one float64 payload column per side (50 % nulls) through the join's index columns")
    except MemoryError as ex:  # not enough HBM next to the inputs
        res["inner_join_10pct"] = {"error": str(ex)[:200]}
    return res

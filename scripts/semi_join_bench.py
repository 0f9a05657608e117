"""Left semi / anti join at 1e9 left int64 rows on one GPU, printed as one JSON line (card name and power limit included).

(a) small filter: right = 1e6 distinct keys (the even numbers below 2e6), left keys = splitmix64 mod 2e6, so about half of the
    left rows are kept. The set (2^21 slots x 16 B = 32 MB) fits in L2.
(b) BASELINE configs[2] shape: |R| = |L| = 1e9, 10 % of the left rows copy one right key (the generator of bench_extra's
    inner_join_10pct). The set (2^31 slots = 32 GB) lives in HBM. The same inputs then go through inner_join, the workaround
    a caller without a semi join has; the set is released before that call, so the two never hold device memory together.

Every shape is warmed up; times are best-of-k host clocks around calls that end in a device synchronise, and the
filtered_join_build / compact split comes from the library's profiling scopes in separate calls. Contract bytes: build
8|R| + 16S (initialising the S-slot set) and probe 8n + 4m (keys in, ids out) + 8m (the copy into the right-sized column);
(b) adds one 32-byte sector per probe (32n), since its set does not fit in L2. The CPU baseline is pandas' Series.isin at
1e7 left rows on one host core.

usage: python scripts/semi_join_bench.py [--rows N] [--reps K] [--skip-b]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SEED = 0x5EED0001  # BASELINE / bench_extra seed; streams are `first` offsets of stream_id << 40
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().splitlines() or ["unknown, unknown"])[0].split(", ")
    return name, power


def best_ms(torch, fn, reps):
    fn()  # warm-up: module load, pool growth
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
        del r
    return min(out)


def scopes(torch, _lib, fn, names):
    """ms per launch of each profiling scope over one profiled call (a run of its own: the events slow the host)."""
    torch.cuda.synchronize()
    _lib.lib.b2_profile_reset()
    _lib.lib.b2_profile_enable(1)
    r = fn()
    torch.cuda.synchronize()
    _lib.lib.b2_profile_enable(0)
    del r
    return {k: _lib.profile_get(k)[0] / max(_lib.profile_get(k)[1], 1) for k in names if _lib.profile_get(k)[1]}


def pandas_isin(left, right, reps=3):
    import pandas as pd

    s, r = pd.Series(left), pd.Series(right)
    s.isin(r)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        s.isin(r)
        ts.append(time.perf_counter() - t0)
    return min(ts) * 1e3


def set_slots(rows, load_factor=0.5):
    """Slots of the filter set (filtered_join.cu set_slots)."""
    above = 1 << int(rows).bit_length()
    cap = min(above * 8, 1 << 31)
    want = max(rows + 1, math.ceil(rows / load_factor))
    s = 1
    while s < cap and s < want:
        s <<= 1
    return s


def measure(torch, plc, _lib, L, R, r_rows, n, reps, per_probe_sector):
    """Build once, then semi and anti over the same left table."""
    out = {}
    EQ = plc.NullEquality.EQUAL
    S = set_slots(r_rows)
    build_bytes = 8 * r_rows + 16 * S
    out["build_ms"] = best_ms(torch, lambda: plc.join.FilteredJoin(R, EQ), max(1, reps // 2))
    out["build_split_ms"] = scopes(torch, _lib, lambda: plc.join.FilteredJoin(R, EQ), ["filtered_join_build"])
    out["build_contract_bytes"] = build_bytes
    out["build_frac_of_hbm"] = build_bytes / (out["build_ms"] / 1e3) / HBM_PEAK
    fj = plc.join.FilteredJoin(R, EQ)
    torch.cuda.synchronize()
    for kind in ("semi", "anti"):
        fn = getattr(fj, f"{kind}_join")
        m = fn(L).size()
        ms = best_ms(torch, lambda: fn(L), reps)
        probe_bytes = 8 * n + 4 * m + 8 * m + (32 * n if per_probe_sector else 0)
        out[kind] = {"ms_per_call": ms, "kept_rows": m, "split_ms": scopes(torch, _lib, lambda: fn(L), ["compact"]),
                     "contract_bytes": probe_bytes, "achieved_GBps": probe_bytes / (ms / 1e3) / 1e9,
                     "frac_of_hbm": probe_bytes / (ms / 1e3) / HBM_PEAK,
                     "rows_per_s": n / (ms / 1e3)}
    del fj
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-b", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch

    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    import __graft_entry__ as g

    g.build()
    import cudf_b200.pylibcudf as plc
    from cudf_b200 import _lib
    from oracle import datagen

    dev = torch.device("cuda:0")
    n = args.rows

    def fill(t, stream_id, kind=0, modulus=0):
        _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(t.data_ptr()), t.numel(), SEED, stream_id << 40, kind, modulus,
                                               _lib.stream_arg(None)))
        return t

    def release():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        _lib.check(_lib.lib.b2_trim_pool())

    name, power = card()
    res = {"card": name, "power_limit": power, "left_rows": n, "hbm_peak_GBps": HBM_PEAK / 1e9}

    # ---- (a) small filter --------------------------------------------------------------------------------------------
    rk = torch.arange(0, 2_000_000, 2, dtype=torch.int64, device=dev)
    lk = fill(torch.empty(n, dtype=torch.int64, device=dev), 6, kind=2, modulus=2_000_000)
    L, R = plc.Table([plc.Column.from_torch(lk)]), plc.Table([plc.Column.from_torch(rk)])
    a = measure(torch, plc, _lib, L, R, rk.numel(), n, args.reps, False)
    cn = 10_000_000
    a["pandas_isin_1e7_ms"] = pandas_isin(datagen.fill(cn, SEED, 6 << 40, 2, 2_000_000), np.arange(0, 2_000_000, 2))
    a["pandas_isin_1e7_rows_per_s"] = cn / (a["pandas_isin_1e7_ms"] / 1e3)
    res["a_small_filter"] = a
    del L, R, lk, rk
    release()

    # ---- (b) |R| = 1e9, 10 % of the left rows match once ---------------------------------------------------------------
    if not args.skip_b:
        rk = fill(torch.empty(n, dtype=torch.int64, device=dev), 1)
        lk = fill(torch.empty(n, dtype=torch.int64, device=dev), 6)
        u = fill(torch.empty(n, dtype=torch.float64, device=dev), 5, kind=1)
        sel = fill(torch.empty(n, dtype=torch.int64, device=dev), 4, kind=2, modulus=n)
        hit = u < 0.10
        del u
        lk[hit] = rk[sel[hit]]
        del sel, hit
        release()
        L, R = plc.Table([plc.Column.from_torch(lk)]), plc.Table([plc.Column.from_torch(rk)])
        b = measure(torch, plc, _lib, L, R, n, n, max(2, args.reps - 1), True)
        release()  # the 32 GB set is gone before the inner join allocates
        EQ = plc.NullEquality.EQUAL
        b["inner_join_ms"] = best_ms(torch, lambda: plc.join.inner_join(L, R, EQ), 2)
        li, _ = plc.join.inner_join(L, R, EQ)
        b["inner_join_pairs"] = li.size()
        del li
        release()
        cl = datagen.fill(cn, SEED, 6 << 40, 0)
        cr = datagen.fill(cn, SEED, 1 << 40, 0)
        pick = datagen.fill(cn, SEED, 5 << 40, 1) < 0.10
        cl[pick] = cr[datagen.fill(cn, SEED, 4 << 40, 2, cn)[pick]]
        b["pandas_isin_1e7_ms"] = pandas_isin(cl, cr)
        b["pandas_isin_1e7_rows_per_s"] = cn / (b["pandas_isin_1e7_ms"] / 1e3)
        b["semi_vs_inner_join_speedup"] = b["inner_join_ms"] / b["semi"]["ms_per_call"]
        b["semi_with_build_vs_inner_join_speedup"] = b["inner_join_ms"] / (b["semi"]["ms_per_call"] + b["build_ms"])
        res["b_configs2_shape"] = b
        del L, R, lk, rk
        release()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

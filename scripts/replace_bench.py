"""Replacement at 1e9 rows on one GPU, printed as one JSON line (card name and power limit included).

(a) replace_nulls with a scalar, int64 with 50 % nulls: 8 B in, 8 B out, 1/8 B of mask in (16.125 B/row);
(b) replace_nulls with a column, int64 with 50 % nulls, a replacement without nulls: 8 + 8 B in, 8 B out, 1/8 B of mask in
    (24.125 B/row);
(c) PRECEDING fill, int64 with 50 % random nulls: 8 B in, 8 B out, 1/8 B of mask in and out (16.25 B/row);
(d) PRECEDING fill, int64 with long null runs (one valid row in 4096): 8 B out and 1/8 B of mask in and out; a run reads its
    one value, so about 8.25 B/row;
(e) find_and_replace_all, int64, k = 16 (table in shared memory): 16 B/row;
(f) find_and_replace_all, int64, k = 20 000 (past the shared-memory budget: the table is searched in L2): 16 B/row;
(g) clamp, float64 without nulls: 16 B/row;
(h) normalize_nans_and_zeros, float64 without nulls: 16 B/row.

Times are best-of-k host clocks around calls that end in a device synchronise, after a warm-up call of the same shape; a call
includes the output allocation (pooled) and, for find_and_replace_all, building its table. Achieved bandwidth is contract bytes
over that time; HBM_PEAK is the data sheet's figure, for the share of peak.

usage: python scripts/replace_bench.py [--rows N] [--reps K]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch

    import __graft_entry__ as g

    assert torch.cuda.is_available(), "replace_bench needs a GPU"
    g.build()
    import cudf_b200.pylibcudf as plc

    n = args.rows
    R, T = plc.replace, plc.TypeId
    gen = torch.Generator(device="cuda").manual_seed(7)
    res = {"bench": "replace", "rows": n, "reps": args.reps}
    res["card"], res["power_limit"] = card()

    def record(name, fn, bytes_per_row):
        ms = best_ms(torch, fn, args.reps)
        gbs = bytes_per_row * n / (ms * 1e-3) / 1e9
        res[name] = {"ms": round(ms, 3), "contract_bytes_per_row": bytes_per_row, "GB_s": round(gbs, 1),
                     "share_of_hbm_peak": round(gbs * 1e9 / HBM_PEAK, 3)}

    i64 = plc.DataType(T.INT64)
    words = (n + 31) // 32
    a = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=gen, device="cuda")
    m = torch.randint(-(2**31), 2**31, (words,), dtype=torch.int64, generator=gen, device="cuda").to(torch.int32)
    ca = plc.Column.from_torch(a, mask=m)
    record("replace_nulls_scalar_int64", lambda: R.replace_nulls(ca, plc.Scalar.from_py(-1, i64)), 16.125)
    b = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=gen, device="cuda")
    cb = plc.Column.from_torch(b)
    record("replace_nulls_column_int64", lambda: R.replace_nulls(ca, cb), 24.125)
    del cb, b
    record("fill_preceding_int64_random", lambda: R.replace_nulls(ca, R.ReplacePolicy.PRECEDING), 16.25)
    runs = torch.zeros(words, dtype=torch.int32, device="cuda")
    runs[::128] = 1  # one valid row in 4096
    cr = plc.Column.from_torch(a, mask=runs)
    record("fill_preceding_int64_runs", lambda: R.replace_nulls(cr, R.ReplacePolicy.PRECEDING), 8.25)
    del cr, ca, runs, m

    x = torch.randint(0, 64, (n,), dtype=torch.int64, generator=gen, device="cuda")
    cx = plc.Column.from_torch(x)
    for k in (16, 20_000):
        old = plc.Column.from_torch(torch.randint(0, 64 if k == 16 else 3 * k, (k,), dtype=torch.int64, generator=gen, device="cuda"))
        new = plc.Column.from_torch(torch.randint(-(2**40), 2**40, (k,), dtype=torch.int64, generator=gen, device="cuda"))
        record(f"find_and_replace_all_int64_k{k}", lambda: R.find_and_replace_all(cx, old, new), 16)
    del cx, x, a

    f64 = plc.DataType(T.FLOAT64)
    f = torch.randn(n, dtype=torch.float64, generator=gen, device="cuda")
    cf = plc.Column.from_torch(f)
    record("clamp_float64", lambda: R.clamp(cf, plc.Scalar.from_py(-1.0, f64), plc.Scalar.from_py(1.0, f64)), 16)
    record("normalize_nans_and_zeros_float64", lambda: R.normalize_nans_and_zeros(cf), 16)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

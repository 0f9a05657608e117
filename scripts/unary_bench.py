"""Unary operations and casts at 1e9 rows on one GPU, printed as one JSON line (card name and power limit included).

(a) float64 SQRT: 8 B in, 8 B out per row (16 B/row);
(b) float64 SIN: 16 B/row, and about 20-40 FP64 operations per row: may be bound by FP64 throughput rather than HBM;
(c) int32 -> float64 cast: 4 B in, 8 B out (12 B/row);
(d) int64 -> float64 cast with 50 % nulls: 8 + 8 B, and 1/8 B of mask in and out (16.25 B/row);
(e) TIMESTAMP_NANOSECONDS -> TIMESTAMP_MILLISECONDS: 8 + 8 B (16 B/row), one floor division per row;
(f) is_null of a nullable column: 1/8 B of mask in, 1 B out (1.125 B/row).

Times are best-of-k host clocks around calls that end in a device synchronise, after a warm-up call of the same shape; a call
includes the output allocation (pooled). Achieved bandwidth is contract bytes over that time; HBM_PEAK is the data sheet's
figure, for the share of peak.

usage: python scripts/unary_bench.py [--rows N] [--reps K]
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

    assert torch.cuda.is_available(), "unary_bench needs a GPU"
    g.build()
    import cudf_b200.pylibcudf as plc

    n = args.rows
    U, T = plc.unary, plc.TypeId
    gen = torch.Generator(device="cuda").manual_seed(7)
    res = {"bench": "unary", "rows": n, "reps": args.reps}
    res["card"], res["power_limit"] = card()

    def record(name, fn, bytes_per_row):
        ms = best_ms(torch, fn, args.reps)
        gbs = bytes_per_row * n / (ms * 1e-3) / 1e9
        res[name] = {"ms": round(ms, 3), "contract_bytes_per_row": bytes_per_row, "GB_s": round(gbs, 1),
                     "share_of_hbm_peak": round(gbs * 1e9 / HBM_PEAK, 3)}

    f64 = plc.DataType(T.FLOAT64)
    x = torch.rand(n, dtype=torch.float64, generator=gen, device="cuda") * 100
    cx = plc.Column.from_torch(x)
    record("sqrt_float64", lambda: U.unary_operation(cx, U.UnaryOperator.SQRT), 16)
    record("sin_float64", lambda: U.unary_operation(cx, U.UnaryOperator.SIN), 16)
    del cx, x

    i = torch.randint(-(2**31), 2**31, (n,), dtype=torch.int64, generator=gen, device="cuda").to(torch.int32)
    ci = plc.Column.from_torch(i)
    record("cast_int32_float64", lambda: U.cast(ci, f64), 12)
    del ci, i

    words = n // 32 + 1
    a = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=gen, device="cuda")
    m = torch.randint(-(2**31), 2**31, (words,), dtype=torch.int64, generator=gen, device="cuda").to(torch.int32)
    ca = plc.Column.from_torch(a, mask=m)
    record("cast_int64_float64_nulls", lambda: U.cast(ca, f64), 16.25)
    ct = plc.Column.from_torch(a, dtype=plc.DataType(T.TIMESTAMP_NANOSECONDS))
    record("cast_timestamp_ns_ms", lambda: U.cast(ct, plc.DataType(T.TIMESTAMP_MILLISECONDS)), 16)
    del ca, ct, a

    b = torch.empty(n, dtype=torch.int8, device="cuda")
    cb = plc.Column.from_torch(b, mask=m)
    record("is_null", lambda: U.is_null(cb), 1.125)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

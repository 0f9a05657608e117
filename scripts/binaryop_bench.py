"""Binary operations at 1e9 rows on one GPU, printed as one JSON line (card name and power limit included).

(a) int64 ADD of two null-free columns: 8 + 8 B in, 8 B out per row (24 B/row);
(b) float64 MUL of two columns with 50 % nulls each: 8 + 8 B in, 8 B out, and 1/8 B of mask per operand and for the output
    (24.375 B/row);
(c) float64 GREATER against a scalar, null-free: 8 B in, 1 B out (9 B/row) — the predicate of a filter.

Times are best-of-k host clocks around calls that end in a device synchronise, after a warm-up call of the same shape; a call
includes the output allocation (pooled) and, for (b), the read-back of the null count when the result is wrapped. Achieved
bandwidth is contract bytes over that time; HBM_PEAK is the data sheet's figure, for the share of peak.

usage: python scripts/binaryop_bench.py [--rows N] [--reps K]
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

    assert torch.cuda.is_available(), "binaryop_bench needs a GPU"
    g.build()
    import cudf_b200.pylibcudf as plc

    n = args.rows
    B, T = plc.binaryop, plc.TypeId
    gen = torch.Generator(device="cuda").manual_seed(7)
    res = {"bench": "binaryop", "rows": n, "reps": args.reps}
    res["card"], res["power_limit"] = card()

    def record(name, fn, bytes_per_row):
        ms = best_ms(torch, fn, args.reps)
        gbs = bytes_per_row * n / (ms * 1e-3) / 1e9
        res[name] = {"ms": round(ms, 3), "contract_bytes_per_row": bytes_per_row, "GB_s": round(gbs, 1),
                     "share_of_hbm_peak": round(gbs * 1e9 / HBM_PEAK, 3)}

    a = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=gen, device="cuda")
    b = torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=gen, device="cuda")
    ca, cb = plc.Column.from_torch(a), plc.Column.from_torch(b)
    record("add_int64", lambda: B.binary_operation(ca, cb, B.BinaryOperator.ADD, plc.DataType(T.INT64)), 24)
    del ca, cb, a, b

    words = n // 32 + 1
    x = torch.rand(n, dtype=torch.float64, generator=gen, device="cuda")
    y = torch.rand(n, dtype=torch.float64, generator=gen, device="cuda")
    mx = torch.randint(-(2**31), 2**31, (words,), dtype=torch.int64, generator=gen, device="cuda").to(torch.int32)
    my = torch.randint(-(2**31), 2**31, (words,), dtype=torch.int64, generator=gen, device="cuda").to(torch.int32)
    cx, cy = plc.Column.from_torch(x, mask=mx), plc.Column.from_torch(y, mask=my)
    record("mul_float64_nulls", lambda: B.binary_operation(cx, cy, B.BinaryOperator.MUL, plc.DataType(T.FLOAT64)), 24.375)
    del cx, cy, y, mx, my

    cx = plc.Column.from_torch(x)
    s = plc.Scalar.from_py(0.5, plc.DataType(T.FLOAT64))
    record("greater_float64_scalar", lambda: B.binary_operation(cx, s, B.BinaryOperator.GREATER, plc.DataType(T.BOOL8)), 9)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

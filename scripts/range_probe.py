"""Phase probe of the range sort: where one range's time goes.   python scripts/range_probe.py [--rows N] [--out DIR]

Compiles `radix_sort.cu` with -DB2_RANGE_PROBE into a temporary copy of the library (the other objects come from the in-tree
build, so run build() first), runs `sort_by_key(T, T)` of --rows int64 splitmix64 keys twice to warm up and once probed, and
prints the mean and p90 of every phase of `range_sort_kernel` over all its CTAs: thread 0 takes a clock64() stamp behind the
barrier that ends each phase. Cycles are turned into microseconds with the probed call's `segment_fix` scope, which holds only
the range sort. Each SM's CTAs run one after another, so the probe also prints how much of an SM's span its CTAs cover.
The library is loaded on its own (not through cudf_b200._lib), so the shipped library is never touched. `--build-only SO` builds
it without a GPU; `--lib SO` then runs that build instead of compiling again."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "cudf_b200"))
import build as b2build  # noqa: E402  (cudf_b200/build.py: flags and object directory, without loading the library)

PHASES = ["key load waited", "histogram", "scan", "scatter", "walk", "payload waited", "write issued"]


class ColumnView(C.Structure):
    _fields_ = [("type_id", C.c_int32), ("size", C.c_int32), ("data", C.c_void_p), ("null_mask", C.c_void_p),
                ("null_count", C.c_int32), ("offset", C.c_int32)]


class TableView(C.Structure):
    _fields_ = [("columns", C.POINTER(ColumnView)), ("num_columns", C.c_int32)]


def probe_library(tmp: Path) -> Path:
    objs = [p for p in sorted(b2build.OBJ.glob("*.o")) if p.stem != "radix_sort"]
    if not objs:
        raise SystemExit("run build() first: the probe links the in-tree objects")
    obj = tmp / "radix_sort_probe.o"
    subprocess.run([b2build.NVCC, *b2build.FLAGS, "-DB2_RANGE_PROBE", "-c", str(b2build.CSRC / "radix_sort.cu"), "-o", str(obj)],
                   check=True)
    so = tmp / "libcudf_b200_probe.so"
    subprocess.run([b2build.NVCC, "-shared", "-o", str(so), str(obj), *map(str, objs), "-lcudart", "-ldl"], check=True)
    return so


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--out", default=None, help="directory for range_probe.json")
    ap.add_argument("--lib", default=None, help="a probe library built earlier by --build-only")
    ap.add_argument("--build-only", default=None, metavar="SO", help="build the probe library to SO and exit")
    a = ap.parse_args()
    if a.build_only:
        with tempfile.TemporaryDirectory() as tmp:
            Path(a.build_only).write_bytes(probe_library(Path(tmp)).read_bytes())
        return
    if a.lib:
        lib = C.CDLL(str(Path(a.lib).resolve()), mode=C.RTLD_LOCAL)
    else:
        with tempfile.TemporaryDirectory() as tmp:
            lib = C.CDLL(str(probe_library(Path(tmp))), mode=C.RTLD_LOCAL)
    lib.b2_last_error.restype = C.c_char_p

    def check(st):
        if st != 0:
            raise RuntimeError(lib.b2_last_error().decode())

    n = a.rows
    torch.cuda.set_device(0)
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    check(lib.b2_fill_splitmix64(C.c_void_p(keys.data_ptr()), C.c_int64(n), C.c_uint64(0x5EED0001), C.c_int64(0), 0,
                                 C.c_uint64(0), None))
    col = ColumnView(4, n, keys.data_ptr(), None, 0, 0)
    tv = TableView(C.pointer(col), 1)
    tot_ms, launches = C.c_double(), C.c_int64()

    def call():
        out = C.c_void_p()
        check(lib.b2_sort_by_key(C.byref(tv), C.byref(tv), None, 0, None, 0, 0, None, C.byref(out)))
        torch.cuda.synchronize()
        lib.b2_table_free(out)

    for _ in range(2):
        call()
    check(lib.b2_range_probe_reset())
    lib.b2_profile_reset()
    lib.b2_profile_enable(1)
    call()
    lib.b2_profile_enable(0)
    check(lib.b2_profile_get(b"segment_fix", C.byref(tot_ms), C.byref(launches)))
    stamps, ctas = C.c_int(), C.c_int()
    buf = np.zeros((10, 1 << 17), dtype=np.int64)
    check(lib.b2_range_probe_read(buf.ctypes.data_as(C.POINTER(C.c_longlong)), C.byref(stamps), C.byref(ctas)))
    t = buf[: stamps.value]
    smid, m = buf[stamps.value], buf[stamps.value + 1]
    live = m > 0
    t, smid, m = t[:, live], smid[live], m[live]
    d = np.diff(t, axis=0).astype(np.float64)  # [phase][cta] cycles
    cta = (t[-1] - t[0]).astype(np.float64)
    spans, busy = [], []
    for s in np.unique(smid):
        sel = smid == s
        spans.append(float(t[-1, sel].max() - t[0, sel].min()))
        busy.append(float(cta[sel].sum()) / spans[-1])
    cyc_per_us = float(np.median(spans)) / (tot_ms.value * 1e3)
    name = torch.cuda.get_device_name(0)
    print(f"{name}; {n} rows, {int(live.sum())} ranges of {m.mean():.0f} rows (max {m.max()}); range sort {tot_ms.value:.2f} ms "
          f"in {launches.value} launch(es); {cyc_per_us:.0f} cycles/us; CTAs cover {np.mean(busy):.3f} of their SM's span")
    rows = {}
    print(f"| phase | mean us | p90 us | share |")
    print("|---|---|---|---|")
    for i, p in enumerate(PHASES):
        mu, p90 = d[i].mean() / cyc_per_us, np.percentile(d[i], 90) / cyc_per_us
        rows[p] = {"mean_us": mu, "p90_us": p90, "share": float(d[i].mean() / cta.mean())}
        print(f"| {p} | {mu:.2f} | {p90:.2f} | {rows[p]['share']:.3f} |")
    print(f"| whole range | {cta.mean() / cyc_per_us:.2f} | {np.percentile(cta, 90) / cyc_per_us:.2f} | 1 |")
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "range_probe.json").write_text(json.dumps(
            {"device": name, "rows": n, "ranges": int(live.sum()), "range_sort_ms": tot_ms.value, "cycles_per_us": cyc_per_us,
             "sm_busy": float(np.mean(busy)), "phases": rows, "range_us_mean": float(cta.mean() / cyc_per_us)}, indent=1))


if __name__ == "__main__":
    main()

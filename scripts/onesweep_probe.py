"""Phase probe of the one-sweep pass: where one tile's time goes.   python scripts/onesweep_probe.py [--rows N] [--out DIR]

Compiles `radix_sort.cu` with -DB2_ONESWEEP_PROBE into a temporary copy of the library (the other objects come from the in-tree
build, so run build() first), runs `sort_by_key(T, T)` of --rows int64 splitmix64 keys twice to warm up and once probed, and
prints the mean and p90 of every phase of `onesweep_kernel`, separately for the first pass (raw keys in) and the second: ranking
thread 0 of the CTA that runs a tile takes a clock64() stamp at each phase boundary, and the first look-back lane one when its
look-back is done. Cycles are turned into microseconds with the probed call's `onesweep` scope, which holds both passes. The probe
also prints how much of each SM's span its tiles cover (the rest is CTA turnover, or a CTA waiting with no tile).
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

# stamp i ends phase i - 1; stamp 8 (look-back done) is taken by a look-back lane, so it is reported on its own
STAMPS = ["entry", "tile id known", "keys landed", "S1 (counts)", "S1b (scan)", "S2", "ranked and staged", "S4",
          "look-back done", "keys written", "payload landed", "payload written"]
PHASES = [(0, 1, "tile claim"), (1, 2, "key wait"), (2, 3, "counts (S1)"), (3, 4, "scan (S1b)"), (4, 5, "offsets (S2)"),
          (5, 6, "ranking and staging"), (6, 7, "payload issue + S4"), (7, 9, "key scatter"), (9, 10, "payload wait + staging"),
          (10, 11, "payload write issued")]


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
    subprocess.run([b2build.NVCC, *b2build.FLAGS, "-DB2_ONESWEEP_PROBE", "-c", str(b2build.CSRC / "radix_sort.cu"), "-o", str(obj)],
                   check=True)
    so = tmp / "libcudf_b200_probe.so"
    subprocess.run([b2build.NVCC, "-shared", "-o", str(so), str(obj), *map(str, objs), "-lcudart", "-ldl"], check=True)
    return so


def pass_table(t, smid):
    """t: [stamp][tile] cycles of one pass's probed tiles; returns per-phase cycles, the tile spans and each SM's covered share."""
    tile = (t[11] - t[0]).astype(np.float64)
    phases = {name: (t[b] - t[a]).astype(np.float64) for a, b, name in PHASES}
    phases["look-back (S2 to look-back done)"] = (t[8] - t[5]).astype(np.float64)
    spans, busy = [], []
    for s in np.unique(smid):
        sel = smid == s
        spans.append(float(t[11, sel].max() - t[0, sel].min()))
        busy.append(float(tile[sel].sum()) / spans[-1])
    return phases, tile, spans, busy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--out", default=None, help="directory for onesweep_probe.json")
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
    check(lib.b2_onesweep_probe_reset())
    lib.b2_profile_reset()
    lib.b2_profile_enable(1)
    call()
    lib.b2_profile_enable(0)
    check(lib.b2_profile_get(b"onesweep", C.byref(tot_ms), C.byref(launches)))
    stamps, tiles = C.c_int(), C.c_int()
    buf = np.zeros((2, len(STAMPS) + 1, 1 << 17), dtype=np.int64)
    check(lib.b2_onesweep_probe_read(buf.ctypes.data_as(C.POINTER(C.c_longlong)), C.byref(stamps), C.byref(tiles)))
    assert stamps.value == len(STAMPS) and tiles.value == buf.shape[2]
    res = []
    for slot in range(2):
        live = buf[slot, 11] > 0  # tiles that ran to the end (not trivial passes, not past-the-end claims)
        res.append(pass_table(buf[slot, :-1][:, live], buf[slot, -1][live]) + (int(live.sum()),))
    cyc_per_us = (float(np.median(res[0][2])) + float(np.median(res[1][2]))) / (tot_ms.value * 1e3)
    name = torch.cuda.get_device_name(0)
    print(f"{name}; {n} rows; both passes {tot_ms.value:.2f} ms in {launches.value} launch(es); {cyc_per_us:.0f} cycles/us")
    out = {"device": name, "rows": n, "onesweep_ms": tot_ms.value, "cycles_per_us": cyc_per_us, "passes": []}
    for slot, (phases, tile, spans, busy, nt) in enumerate(res):
        print(f"\npass {slot + 1}: {nt} tiles; tiles cover {np.mean(busy):.3f} of their SM's span; SM span "
              f"{np.median(spans) / cyc_per_us / 1e3:.2f} ms")
        print("| phase | mean us | p90 us |")
        print("|---|---|---|")
        rows = {}
        for p, d in phases.items():
            rows[p] = {"mean_us": d.mean() / cyc_per_us, "p90_us": np.percentile(d, 90) / cyc_per_us}
            print(f"| {p} | {rows[p]['mean_us']:.2f} | {rows[p]['p90_us']:.2f} |")
        rows["whole tile"] = {"mean_us": tile.mean() / cyc_per_us, "p90_us": np.percentile(tile, 90) / cyc_per_us}
        print(f"| whole tile (entry to payload written) | {rows['whole tile']['mean_us']:.2f} | {rows['whole tile']['p90_us']:.2f} |")
        out["passes"].append({"tiles": nt, "sm_busy": float(np.mean(busy)), "sm_span_ms": float(np.median(spans)) / cyc_per_us / 1e3,
                              "phases": rows})
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / "onesweep_probe.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

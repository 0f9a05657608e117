"""Static resource table of the shipped kernels (no GPU needed): registers, static shared memory and stack per kernel from
`cuobjdump --dump-resource-usage`, plus the SASS mnemonics that identify a mechanism (UBLKCP = cp.async.bulk / 1-D TMA, ATOMS = shared
atomics, REDUX, MATCH, BAR with a named id).   python scripts/kernel_resources.py"""
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "cudf_b200" / "libcudf_b200.so"
INTEREST = ["onesweep_kernel", "histogram_kernel", "segment_fix_kernel", "plan_kernel", "rj_join_kernel", "pgb_agg_kernel",
            "scan_kernel", "reduce_kernel", "segreduce_kernel", "gather_kernel", "range_count_kernel", "build_kernel", "groupby_kernel",
            "compact_kernel", "scatter_staged_kernel", "peer_copy_kernel"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


res = subprocess.run(["cuobjdump", "--dump-resource-usage", str(LIB)], capture_output=True, text=True).stdout
rows = []
cur = None
for line in res.splitlines():
    m = re.match(r"\s*Function (\S+):", line)
    if m:
        cur = m.group(1)
        continue
    m = re.match(r"\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
    if m and cur:
        rows.append((cur, int(m.group(1)), int(m.group(2)), int(m.group(3))))
        cur = None
dm = demangle([r[0] for r in rows])
sass = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True).stdout
mnem = {}
cur = None
for line in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1)
        mnem[cur] = {}
        continue
    if cur:
        for key in ("UBLKCP", "ATOMS", "ATOMG", "REDG", "REDUX", "MATCH", "SYNCS", "LDG.E.128", "STG.E.128", "LDS.128", "BAR.SYNC", "BAR.ARV", "VOTE", "SHFL"):
            if re.search(r"\b" + re.escape(key), line):
                mnem[cur][key] = mnem[cur].get(key, 0) + 1
print("# Static resources of the shipped kernels (sm_90a; `scripts/kernel_resources.py`, no GPU involved)\n")
print("Registers / stack / static shared memory from `cuobjdump --dump-resource-usage cudf_b200/libcudf_b200.so`; dynamic shared memory is set at")
print("launch (one-sweep with 8-byte keys: 76.9 KB at 384 x 16 -> two CTAs of 448 threads per SM, 117.8 KB at 512 x 20 -> one CTA of 576;")
print("`rj_join_kernel`: 160 KB, one CTA of 1024; `pgb_agg_kernel`: 160 KB, one CTA of 1024). Mnemonic counts are static occurrences in the")
print("SASS (UBLKCP = `cp.async.bulk`, the 1-D TMA path, only in the 512 x 20 payload-carrying one-sweep instantiation and in")
print("`range_sort_kernel`; SYNCS = mbarrier operations).\n")
print("| Kernel | regs | stack | static smem | SASS mnemonics (static count) |")
print("|---|---|---|---|---|")
for name, reg, stack, sh in sorted(rows, key=lambda r: dm[r[0]]):
    d = dm[name]
    if not any(k in d for k in INTEREST):
        continue
    short = re.sub(r"\(anonymous namespace\)::", "", d)
    short = re.sub(r"^void ", "", short)
    short = short.split("(")[0] if "<" not in short else short[: short.rindex(">") + 1] if ">" in short else short
    short = short.replace("b2::", "")
    ms = ", ".join(f"{k} {v}" for k, v in sorted(mnem.get(name, {}).items()))
    print(f"| `{short[:150]}` | {reg} | {stack} | {sh} | {ms} |")

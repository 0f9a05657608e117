"""include/cudf/replace.hpp: tests/cpp/replace_smoke.cpp compiles against the library (CPU), runs on the kernel
emulator (CPU, linked against tests/emu's library and its runtime) and runs on the GPU."""
import os
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "cpp" / "replace_smoke.cpp"
MARK = "REPLACE_CPP_OK"


def _compile(out: Path, emu: bool) -> Path:
    if emu:
        from tests.emu.build_emu import LIB

        lib_dir, lib, inc = LIB.parent, "-l:" + LIB.name, [f"-I{ROOT / 'tests' / 'emu' / 'include'}"]
    else:
        import __graft_entry__ as g

        g.build()
        lib_dir, lib, inc = ROOT / "cudf_b200", "-lcudf_b200", ["-I/usr/local/cuda/include"]
    cmd = ["g++", "-std=c++17", *inc, f"-I{ROOT / 'include'}", str(SRC), "-o", str(out), f"-L{lib_dir}", lib, f"-Wl,-rpath,{lib_dir}"]
    if not emu:
        cmd += ["-L/usr/local/cuda/lib64", "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return out


def test_cpp_replace_compiles(tmp_path):
    assert _compile(tmp_path / "replace_smoke", emu=False).exists()


@pytest.mark.skipif(shutil.which("g++") is None, reason="the emulator build needs g++")
def test_cpp_replace_runs_on_emulator(tmp_path):
    from tests.emu.build_emu import build

    build()
    exe = _compile(tmp_path / "replace_smoke_emu", emu=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300, env=dict(os.environ))
    assert MARK in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cpp_replace_runs(tmp_path):
    exe = _compile(tmp_path / "replace_smoke", emu=False)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert MARK in r.stdout, r.stdout + r.stderr

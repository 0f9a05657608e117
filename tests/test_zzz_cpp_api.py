"""The cudf:: C++ header surface (include/cudf/*.hpp) compiles against the C ABI (CPU) and runs (GPU)."""
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _build(out_dir: Path) -> Path:
    """Compile tests/cpp/api_smoke.cpp into `out_dir` (the source tree may be read-only) and return the executable."""
    import __graft_entry__ as g

    g.build()
    exe = out_dir / "api_smoke"
    cmd = ["g++", "-std=c++17", f"-I{ROOT / 'include'}", "-I/usr/local/cuda/include", str(ROOT / "tests/cpp/api_smoke.cpp"), "-o", str(exe),
           f"-L{ROOT / 'cudf_b200'}", "-lcudf_b200", "-L/usr/local/cuda/lib64", "-lcudart", f"-Wl,-rpath,{ROOT / 'cudf_b200'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_cpp_headers_compile(tmp_path):
    assert _build(tmp_path).exists()


@pytest.mark.gpu
def test_cpp_api_runs(tmp_path):
    exe = _build(tmp_path)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert "CPP_API_OK" in r.stdout, r.stdout + r.stderr

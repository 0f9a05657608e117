"""CPU: the replacement parity cases of tests/test_replace_gpu.py at reduced sizes on the kernel emulator (tests/emu):
replace_kernel's generic and vector paths, the staged and global lookup tables and fill_kernel's look-back across tiles. One
subprocess per case, because tests/emu/harness.install() rebinds the package's ctypes entry points."""
import pytest

from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (fixture)
from tests.test_replace_gpu import PARITY

CODE = r"""
from tests.test_replace_gpu import PARITY
{body}
print('REPLACE_OK')
"""


@pytest.mark.parametrize("name", list(PARITY))
def test_emu_parity(emu_lib, name):  # noqa: F811
    run(CODE.format(body=f"PARITY[{name!r}](plc, True)"), "REPLACE_OK")

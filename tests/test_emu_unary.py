"""CPU: the unary-operation parity cases of tests/test_unary_gpu.py at reduced sizes on the kernel emulator (tests/emu):
unary_kernel's generic and vector paths, validity_kernel, every operator and cast family, nulls and sliced views. One subprocess
per case, because tests/emu/harness.install() rebinds the package's ctypes entry points."""
import pytest

from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (fixture)
from tests.test_unary_gpu import PARITY

CODE = r"""
from tests.test_unary_gpu import PARITY, test_golden
{body}
print('UNARY_OK')
"""


@pytest.mark.parametrize("name", list(PARITY))
def test_emu_parity(emu_lib, name):  # noqa: F811
    run(CODE.format(body=f"PARITY[{name!r}](plc, True)"), "UNARY_OK")


def test_emu_golden(emu_lib):  # noqa: F811
    run(CODE.format(body="test_golden(plc)"), "UNARY_OK")

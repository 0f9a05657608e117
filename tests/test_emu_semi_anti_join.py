"""CPU: the semi / anti join parity cases of tests/test_semi_anti_join_gpu.py at reduced sizes on the kernel emulator
(tests/emu): fj_build_kernel and compact_kernel with the contains predicate, packed and wide keys. One subprocess per case,
because tests/emu/harness.install() rebinds the package's ctypes entry points."""
import pytest

from tests.test_emu_kernels import emu_lib, run  # noqa: F401  (fixture)
from tests.test_semi_anti_join_gpu import CASES, PARITY

CODE = r"""
from tests.test_semi_anti_join_gpu import PARITY, test_golden
from tests.golden.semi_anti_join_cases import CASES
{body}
print('SEMI_ANTI_OK')
"""


@pytest.mark.parametrize("name", list(PARITY))
def test_emu_parity(emu_lib, name):  # noqa: F811
    run(CODE.format(body=f"PARITY[{name!r}](plc, True)"), "SEMI_ANTI_OK")


def test_emu_golden(emu_lib):  # noqa: F811
    assert CASES
    run(CODE.format(body="for c in CASES:\n    test_golden(plc, c)"), "SEMI_ANTI_OK")

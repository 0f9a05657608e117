"""Binary operations at 1e9 rows on one 80 GB H100: int64 ADD of two columns and float64 GREATER against a scalar with 50 % nulls,
checked against the oracle at a seeded sample of rows, with the null count checked over every row. Runs late (file name)
because each case moves tens of GB."""
import numpy as np
import pytest

from tests import binaryop_oracle as ob

pytestmark = pytest.mark.gpu

N = 1_000_000_000


def _free(torch):
    from cudf_b200 import _lib

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.check(_lib.lib.b2_trim_pool())


def test_add_int64_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(41)
    a = torch.randint(-(2**62), 2**62, (N,), dtype=torch.int64, generator=g, device="cuda")
    b = torch.randint(-(2**62), 2**62, (N,), dtype=torch.int64, generator=g, device="cuda")
    i64 = plc.DataType(plc.TypeId.INT64)
    out = plc.binaryop.binary_operation(plc.Column.from_torch(a), plc.Column.from_torch(b), plc.binaryop.BinaryOperator.ADD, i64)
    assert out.size() == N and out.null_count() == 0 and not out.nullable()
    got = out.to_torch()
    pos = torch.randint(0, N, (1 << 20,), generator=g, device="cuda")
    exp, _, _, _ = ob.binop(ob.ADD, (a[pos].cpu().numpy(), None, ob.INT64), (b[pos].cpu().numpy(), None, ob.INT64), ob.INT64)
    assert np.array_equal(got[pos].cpu().numpy(), exp)
    assert bool((got[-4096:] == a[-4096:] + b[-4096:]).all())  # the last tile
    del out, got, a, b
    _free(torch)


def test_greater_float64_scalar_half_nulls_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(43)
    x = torch.rand(N, dtype=torch.float64, generator=g, device="cuda")
    words = torch.randint(-(2**31), 2**31, (N // 32,), dtype=torch.int64, generator=g, device="cuda").to(torch.int32)
    col = plc.Column.from_torch(x, mask=words)
    f64, b8 = plc.DataType(plc.TypeId.FLOAT64), plc.DataType(plc.TypeId.BOOL8)
    out = plc.binaryop.binary_operation(col, plc.Scalar.from_py(0.5, f64), plc.binaryop.BinaryOperator.GREATER, b8)
    # every row: the output's nulls are the input's, counted here independently of the library
    shifts = torch.arange(32, dtype=torch.int32, device="cuda")
    valid_rows = sum(int(((words[i:i + (1 << 24)].unsqueeze(1) >> shifts) & 1).sum()) for i in range(0, N // 32, 1 << 24))
    assert out.null_count() == N - valid_rows
    assert 0.49 < valid_rows / N < 0.51
    got_v = out.to_torch()
    got_m = out.null_mask()
    mask_words = torch.as_tensor(plc.DeviceSpan(got_m.ptr, got_m.nelems, np.int32, out), device="cuda")
    assert bool((mask_words[: N // 32] == words).all())
    pos = torch.randint(0, N, (1 << 20,), generator=g, device="cuda")
    vbits = ((words[pos // 32] >> (pos % 32).to(torch.int32)) & 1).bool().cpu().numpy()
    exp, exp_valid, _, _ = ob.binop(ob.GREATER, (x[pos].cpu().numpy(), vbits, ob.FLOAT64), (np.asarray(0.5), True, ob.FLOAT64), ob.BOOL8)
    gv = got_v[pos].cpu().numpy()
    assert np.array_equal(exp_valid, vbits)
    assert np.array_equal(gv[vbits], exp[vbits])
    del out, got_v, x, words, col
    _free(torch)

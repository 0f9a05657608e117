"""Unary operations at 1e9 rows on one 80 GB H100: an int64 -> float64 cast with nulls through a view at a non-zero offset,
is_null of a nullable column and float64 SQRT, checked against the oracle at a seeded sample of rows (the cast's mask and
is_null over every row). Runs late (file name) because each case moves tens of GB."""
import numpy as np
import pytest

from tests import unary_oracle as ou

pytestmark = pytest.mark.gpu

N = 1_000_000_000


def _free(torch):
    from cudf_b200 import _lib

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.check(_lib.lib.b2_trim_pool())


def _bits(words, rows, torch):
    """validity of `rows` (a CUDA int64 tensor) from little-endian mask words"""
    return ((words[rows // 32] >> (rows % 32).to(torch.int32)) & 1).bool()


def test_cast_int64_to_float64_offset_nulls_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(51)
    off = 37
    a = torch.randint(-(2**62), 2**62, (N + off,), dtype=torch.int64, generator=g, device="cuda")
    words = torch.randint(-(2**31), 2**31, ((N + off) // 32 + 1,), dtype=torch.int64, generator=g, device="cuda").to(torch.int32)
    col = plc.Column.from_torch(a, mask=words, offset=off, size=N)
    out = plc.unary.cast(col, plc.DataType(plc.TypeId.FLOAT64))
    assert out.size() == N and out.null_count() == col.null_count() and out.nullable()
    # every row's validity: the output mask is the input's, realigned to offset 0
    m = out.null_mask()
    got_words = torch.as_tensor(plc.DeviceSpan(m.ptr, m.nelems, np.int32, out), device="cuda")
    for i in range(0, N, 1 << 26):
        rows = torch.arange(i, min(N, i + (1 << 26)), device="cuda")
        assert bool((_bits(got_words, rows, torch) == _bits(words, rows + off, torch)).all())
    got = out.to_torch()
    pos = torch.randint(0, N, (1 << 20,), generator=g, device="cuda")
    vbits = _bits(words, pos + off, torch).cpu().numpy()
    exp, _, _ = ou.cast((a[pos + off].cpu().numpy(), vbits, ou.INT64), ou.FLOAT64)
    assert np.array_equal(got[pos].cpu().numpy()[vbits], exp[vbits])
    del out, got, col, a, words
    _free(torch)


def test_is_null_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(53)
    x = torch.empty(N, dtype=torch.int8, device="cuda")
    words = torch.randint(-(2**31), 2**31, (N // 32,), dtype=torch.int64, generator=g, device="cuda").to(torch.int32)
    out = plc.unary.is_null(plc.Column.from_torch(x, mask=words))
    assert out.size() == N and not out.nullable()
    got = out.to_torch()
    for i in range(0, N, 1 << 26):
        rows = torch.arange(i, min(N, i + (1 << 26)), device="cuda")
        assert bool((got[rows] == ~_bits(words, rows, torch)).all())
    del out, got, x, words
    _free(torch)


def test_sqrt_float64_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(57)
    x = torch.rand(N, dtype=torch.float64, generator=g, device="cuda") * 1e6
    out = plc.unary.unary_operation(plc.Column.from_torch(x), plc.unary.UnaryOperator.SQRT)
    assert out.size() == N and out.null_count() == 0 and not out.nullable()
    got = out.to_torch()
    pos = torch.cat([torch.randint(0, N, (1 << 20,), generator=g, device="cuda"), torch.arange(N - 4096, N, device="cuda")])
    exp, _, _ = ou.unary(ou.SQRT, (x[pos].cpu().numpy(), None, ou.FLOAT64))
    assert np.array_equal(got[pos].cpu().numpy(), exp)
    del out, got, x
    _free(torch)

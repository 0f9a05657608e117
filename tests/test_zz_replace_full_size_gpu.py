"""Replacement at 1e9 rows on one 80 GB H100: the PRECEDING and FOLLOWING fills of an int64 column with 50 % random nulls and
with one null run of 5e8 rows, checked on every row against a torch reference on the device (the nearest valid row index by
cummax / cummin, then a gather); a scalar fill; find_and_replace_all with a table past the shared-memory budget, checked at a
seeded sample of rows. Runs late (file name) because each case moves tens of GB."""
import numpy as np
import pytest

from tests import replace_oracle as orp

pytestmark = pytest.mark.gpu

N = 1_000_000_000
CHUNK = 1 << 26


def _free(torch):
    from cudf_b200 import _lib

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.check(_lib.lib.b2_trim_pool())


def _bits(words, rows, torch):
    """validity of `rows` (a CUDA int64 tensor) from little-endian mask words"""
    return ((words[rows // 32] >> (rows % 32).to(torch.int32)) & 1).bool()


def _mask_words(out, plc, torch):
    m = out.null_mask()
    return torch.as_tensor(plc.DeviceSpan(m.ptr, m.nelems, np.int32, out), device="cuda")


def _check_fill(plc, torch, a, words, policy):
    col = plc.Column.from_torch(a, mask=words)
    out = plc.replace.replace_nulls(col, plc.replace.ReplacePolicy(policy))
    # the reference: the nearest valid row index at or before (after) each row
    idx = torch.arange(N, device="cuda")
    for i in range(0, N, CHUNK):
        rows = idx[i:i + CHUNK]
        rows.masked_fill_(~_bits(words, rows.clone(), torch), -1 if policy == orp.PRECEDING else N)
    if policy == orp.PRECEDING:
        src = torch.cummax(idx, 0).values
    else:
        src = torch.cummin(idx.flip(0), 0).values.flip(0)
    del idx
    ok = (src >= 0) & (src < N)
    assert out.null_count() == int((~ok).sum())
    got = out.to_torch()
    got_words = _mask_words(out, plc, torch)
    for i in range(0, N, CHUNK):
        rows = torch.arange(i, min(N, i + CHUNK), device="cuda")
        o = ok[i:i + CHUNK]
        assert bool((_bits(got_words, rows, torch) == o).all())
        assert bool((got[i:i + CHUNK][o] == a[src[i:i + CHUNK][o]]).all())
    del out, got, src, ok, got_words, col
    _free(torch)


@pytest.mark.parametrize("policy", [0, 1])
def test_fill_random_nulls_1e9(plc, policy):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(61 + policy)
    a = torch.randint(-(2**62), 2**62, (N,), dtype=torch.int64, generator=g, device="cuda")
    words = torch.randint(-(2**31), 2**31, (N // 32,), dtype=torch.int64, generator=g, device="cuda").to(torch.int32)
    words[0] = 0  # a leading and a trailing null run
    words[-1] = 0
    _check_fill(plc, torch, a, words, policy)
    del a, words
    _free(torch)


@pytest.mark.parametrize("policy", [0, 1])
def test_fill_long_run_1e9(plc, policy):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(67 + policy)
    a = torch.randint(-(2**62), 2**62, (N,), dtype=torch.int64, generator=g, device="cuda")
    words = torch.randint(-(2**31), 2**31, (N // 32,), dtype=torch.int64, generator=g, device="cuda").to(torch.int32)
    words[N // 32 // 4: 3 * (N // 32) // 4] = 0  # one null run of 5e8 rows
    _check_fill(plc, torch, a, words, policy)
    del a, words
    _free(torch)


def test_scalar_fill_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(71)
    a = torch.randint(-(2**62), 2**62, (N,), dtype=torch.int64, generator=g, device="cuda")
    words = torch.randint(-(2**31), 2**31, (N // 32,), dtype=torch.int64, generator=g, device="cuda").to(torch.int32)
    out = plc.replace.replace_nulls(plc.Column.from_torch(a, mask=words), plc.Scalar.from_py(-5, plc.DataType(plc.TypeId.INT64)))
    assert out.size() == N and not out.nullable() and out.null_count() == 0
    got = out.to_torch()
    for i in range(0, N, CHUNK):
        rows = torch.arange(i, min(N, i + CHUNK), device="cuda")
        v = _bits(words, rows, torch)
        assert bool((got[rows] == torch.where(v, a[rows], -5)).all())
    del out, got, a, words
    _free(torch)


def test_find_and_replace_all_large_k_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(73)
    k = 20_000  # 20 000 keys of 8 bytes and their positions are past the 48 KiB shared-memory budget
    a = torch.randint(0, 3 * k, (N,), dtype=torch.int64, generator=g, device="cuda")
    old = torch.randint(0, 3 * k, (k,), dtype=torch.int64, generator=g, device="cuda")
    new = torch.randint(-(2**40), 2**40, (k,), dtype=torch.int64, generator=g, device="cuda")
    out = plc.replace.find_and_replace_all(plc.Column.from_torch(a), plc.Column.from_torch(old), plc.Column.from_torch(new))
    assert out.size() == N and not out.nullable()
    got = out.to_torch()
    pos = torch.cat([torch.randint(0, N, (1 << 20,), generator=g, device="cuda"), torch.arange(N - 4096, N, device="cuda")])
    exp, _ = orp.find_and_replace_all((a[pos].cpu().numpy(), None, 4), (old.cpu().numpy(), None, 4), (new.cpu().numpy(), None, 4))
    assert np.array_equal(got[pos].cpu().numpy(), exp)
    del out, got, a, old, new
    _free(torch)

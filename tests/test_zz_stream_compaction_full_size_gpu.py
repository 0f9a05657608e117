"""Stream compaction at the bench's size (1e9 rows) on one 80 GB H100: apply_boolean_mask against torch.nonzero at a seeded
sample of positions, and distinct's row count. Runs late (file name) because each case moves tens of GB."""
import pytest

pytestmark = pytest.mark.gpu

N = 1_000_000_000


def _free(torch):
    from cudf_b200 import _lib

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _lib.check(_lib.lib.b2_trim_pool())


def test_apply_boolean_mask_1e9(plc):
    import torch

    _free(torch)
    g = torch.Generator(device="cuda").manual_seed(31)
    vals = torch.arange(N, dtype=torch.int64, device="cuda")   # value = row id: the output is the kept row ids
    mask = torch.rand(N, generator=g, device="cuda") < 0.5     # 50 % true
    _free(torch)
    out = plc.stream_compaction.apply_boolean_mask(plc.Table([plc.Column.from_torch(vals)]), plc.Column.from_torch(mask))
    got = out.columns()[0].to_torch()
    count = int(mask.sum())
    assert got.numel() == count
    kept = torch.nonzero(mask).squeeze(1)
    pos = torch.randint(0, count, (1 << 16,), generator=g, device="cuda")
    assert bool((got[pos] == kept[pos]).all())
    assert bool((got[1:] > got[:-1]).all())  # stable: strictly increasing row ids
    del out, got, kept, vals, mask
    _free(torch)


def test_distinct_1e9_rows_1e6_keys(plc):
    import torch

    _free(torch)
    G = 1_000_000
    k = (torch.arange(N, dtype=torch.int64, device="cuda") * 2654435761) % G
    _free(torch)
    sc = plc.stream_compaction
    out = sc.distinct(plc.Table([plc.Column.from_torch(k)]), [0], sc.DuplicateKeepOption.KEEP_ANY, plc.NullEquality.EQUAL,
                      plc.NanEquality.ALL_EQUAL)
    got = out.columns()[0].to_torch()
    assert got.numel() == G
    assert bool((torch.sort(got).values == torch.arange(G, device="cuda")).all())
    del out, got, k
    _free(torch)

"""Semi / anti join at full size on the GPU: 2^27 rows per side compared exactly with the oracle, and 1e9 left rows against
a 1e6-row filter checked for completeness, order and disjointness on the device and for membership on 2^20 sampled rows."""
import ctypes as C

import numpy as np
import pytest

from oracle import datagen
from tests import semi_anti_oracle as osa

pytestmark = pytest.mark.gpu

SEED = 0x5EED0001


def _fill(torch, _lib, n, stream_id, modulus):
    t = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.b2_fill_splitmix64(C.c_void_p(t.data_ptr()), n, SEED, stream_id << 40, 2, modulus, _lib.stream_arg(None)))
    return t


def test_semi_anti_2p27_exact(plc):
    import torch

    from cudf_b200 import _lib

    n = 1 << 27
    lk, rk = _fill(torch, _lib, n, 6, 1 << 28), _fill(torch, _lib, n, 1, 1 << 28)  # about 39 % of the left keys occur on the right
    fj = plc.join.FilteredJoin(plc.Table([plc.Column.from_torch(rk)]), plc.NullEquality.EQUAL)
    L = plc.Table([plc.Column.from_torch(lk)])
    semi, anti = fj.semi_join(L).to_numpy()[0], fj.anti_join(L).to_numpy()[0]
    hl, hr = datagen.fill(n, SEED, 6 << 40, 2, 1 << 28), datagen.fill(n, SEED, 1 << 40, 2, 1 << 28)
    assert np.array_equal(hl, lk.cpu().numpy())
    assert np.array_equal(semi, osa.left_semi_join([(hl, None)], [(hr, None)]))
    assert np.array_equal(anti, osa.left_anti_join([(hl, None)], [(hr, None)]))


def test_semi_anti_1e9_left_rows(plc):
    import torch

    from cudf_b200 import _lib

    n, mod = 1_000_000_000, 2_000_000
    lk = _fill(torch, _lib, n, 6, mod)
    rk = torch.arange(0, mod, 2, dtype=torch.int64, device="cuda")  # 1e6 distinct keys: the even left keys are kept
    fj = plc.join.FilteredJoin(plc.Table([plc.Column.from_torch(rk)]), plc.NullEquality.EQUAL)
    L = plc.Table([plc.Column.from_torch(lk)])
    semi, anti = fj.semi_join(L).to_torch(), fj.anti_join(L).to_torch()
    del lk
    assert semi.numel() + anti.numel() == n
    for ids in (semi, anti):
        assert bool((ids[1:] > ids[:-1]).all())
    member = torch.zeros(n, dtype=torch.bool, device="cuda")
    member[semi.long()] = True
    assert not bool(member[anti.long()].any())  # disjoint; with the counts above, together they are every row
    pos = np.sort(np.random.default_rng(43).choice(n, 1 << 20, replace=False)).astype(np.uint64)
    with np.errstate(over="ignore"):
        vals = (datagen.splitmix64(pos + np.uint64(SEED + (6 << 40))) % np.uint64(mod)).astype(np.int64)
    exp = osa.contains([(vals, None)], [(np.arange(0, mod, 2, dtype=np.int64), None)])
    got = member[torch.from_numpy(pos.astype(np.int64)).cuda()].cpu().numpy()
    assert np.array_equal(got, exp)

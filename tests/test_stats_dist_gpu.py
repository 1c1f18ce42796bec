"""GPU: the sharded NumPy-order mean/std (gsx_pairwise_leaves_dist / _finish) equals np.mean / np.std of the
concatenated vector bit for bit -- ranks emulated in one process (the slot all-reduce is a plain sum here)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("sizes", [(1000, 1000), (4097, 1, 0, 300, 129), (100_003, 50_000, 77), (5, 3), (3_000_001, 7, 999_992),
                                   (128, 128, 128, 128), (127, 130),
                                   (0, 300, 500), (400, 129, 0), (5, 20, 0, 17, 3, 11, 0, 9)])
def test_sharded_mean_std_matches_numpy(sizes, cuda, gsx_lib):
    import torch
    from gsx._abi import lib, check
    from gsx._abi import _ptr, _stream
    rng = np.random.default_rng(sum(sizes))
    n = int(sum(sizes))
    a = (rng.random(n, dtype=np.float32) * np.float32(3.0)).astype(np.float32)
    a[rng.integers(0, n, max(1, n // 50))] = 0.0
    world = len(sizes)
    bases = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    slabs = [torch.from_numpy(a[bases[r]:bases[r + 1]].copy()).to(cuda) for r in range(world)]
    halo = torch.zeros(world * 128, dtype=torch.float32, device=cuda)
    for r in range(world):
        m = min(128, sizes[r])
        if m:
            halo[r * 128: r * 128 + m] = slabs[r][:m]
    bases_dev = torch.from_numpy(bases).to(cuda)
    nslot = lib.gsx_pairwise_slots(n)
    meanstd = torch.zeros(2, dtype=torch.float32, device=cuda)
    for sq in (0, 1):
        total = torch.zeros(nslot, dtype=torch.float32, device=cuda)
        for r in range(world):
            slot = torch.empty(nslot, dtype=torch.float32, device=cuda)
            check(lib.gsx_pairwise_leaves_dist(_ptr(slabs[r]), int(bases[r]), sizes[r], n, sq, _ptr(meanstd), _ptr(halo),
                                               _ptr(bases_dev), world, _ptr(slot), _stream()))
            total += slot
        check(lib.gsx_pairwise_finish(_ptr(total), n, sq, _ptr(meanstd), _stream()))
    got = meanstd.cpu().numpy()
    assert got[0].view(np.uint32) == np.mean(a).view(np.uint32)
    assert got[1].view(np.uint32) == np.std(a).view(np.uint32)

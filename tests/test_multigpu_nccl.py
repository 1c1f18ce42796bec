"""GPU (>= 2 devices): the sharded drivers over NCCL reproduce the single-GPU results bit for bit.
Skipped on a machine with one GPU; run on two or more with `python -m pytest tests/test_multigpu_nccl.py -m gpu`."""
import os
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def _slab(rank, world, n_per, ragged):
    """Equal slabs, or ragged ones (rank 0 gets 1/3 more, the last rank the rest) over the same union cloud."""
    if not ragged:
        return rank * n_per, (rank + 1) * n_per
    total = n_per * world
    cuts = [0] + [min(total, (r + 1) * n_per + n_per // 3) for r in range(world - 1)] + [total]
    return cuts[rank], cuts[rank + 1]


def _worker(rank, world, port, n_per, q):
    sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device(f"cuda:{rank}"))
    from gsx import dist as gd, sor, density, synth
    xyz = synth.xyz(n_per * world, "mixed")
    local = torch.from_numpy(xyz[rank * n_per:(rank + 1) * n_per].copy()).cuda()
    res = {}
    for mode in ("i32wrap", "i64"):
        mask, means = gd.sor_filter_sharded(local, 16, 2.0, mode, return_means=True)
        res[f"sor_{mode}"] = (mask.cpu().numpy(), means.cpu().numpy())
        mask2, means2 = gd.sor_filter_distributed(local, 16, 2.0, mode, return_means=True)
        res[f"sor2_{mode}"] = (mask2.cpu().numpy(), means2.cpu().numpy())
        a, b = _slab(rank, world, n_per, True)          # ragged slabs: all-reduce routing, spill-over leaves
        rag = torch.from_numpy(xyz[a:b].copy()).cuda()
        mask3, means3 = gd.sor_filter_distributed(rag, 16, 2.0, mode, return_means=True)
        res[f"sor3_{mode}"] = (mask3.cpu().numpy(), means3.cpu().numpy())
    dm, info = gd.density_filter_sharded(local, sensitivity=0.5, keep_multicluster=True)
    res["density"] = (dm.cpu().numpy(), info["clusters"])
    if rank == 0:  # single-GPU truth on the union cloud
        full = torch.from_numpy(xyz).cuda()
        for mode in ("i32wrap", "i64"):
            m, md = sor.sor_filter(full, 16, 2.0, hash_mode=mode, return_means=True)
            res[f"truth_sor_{mode}"] = (m.cpu().numpy(), md.cpu().numpy())
        m, info = density.density_filter(full, sensitivity=0.5, keep_multicluster=True)
        res["truth_density"] = (m.cpu().numpy(), info["clusters"])
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_equals_single_gpu(gsx_lib):
    import torch
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 2)   # 2 ranks exercise every collective; keeps GPU time low
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    n_per = 300_000
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n_per, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, out = q.get(timeout=600)
        res[r] = out
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    for mode in ("i32wrap", "i64"):
        tm, tmd = res[0][f"truth_sor_{mode}"]
        gm = np.concatenate([res[r][f"sor_{mode}"][0] for r in range(world)])
        gmd = np.concatenate([res[r][f"sor_{mode}"][1] for r in range(world)])
        assert np.array_equal(gmd.view(np.uint32), tmd.view(np.uint32)), mode
        assert np.array_equal(gm, tm), mode
        gm2 = np.concatenate([res[r][f"sor2_{mode}"][0] for r in range(world)])
        gmd2 = np.concatenate([res[r][f"sor2_{mode}"][1] for r in range(world)])
        assert np.array_equal(gmd2.view(np.uint32), tmd.view(np.uint32)), ("distributed build", mode)
        assert np.array_equal(gm2, tm), ("distributed build", mode)
        gm3 = np.concatenate([res[r][f"sor3_{mode}"][0] for r in range(world)])
        gmd3 = np.concatenate([res[r][f"sor3_{mode}"][1] for r in range(world)])
        assert np.array_equal(gmd3.view(np.uint32), tmd.view(np.uint32)), ("distributed build, ragged slabs", mode)
        assert np.array_equal(gm3, tm), ("distributed build, ragged slabs", mode)
    td, tc = res[0]["truth_density"]
    gd_ = np.concatenate([res[r]["density"][0] for r in range(world)])
    assert np.array_equal(gd_, td) and all(res[r]["density"][1] == tc for r in range(world))

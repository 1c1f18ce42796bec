"""CPU, world_size 2, gloo: the sharded SOR driver (gsx/dist.py) reproduces the single-process
result bit for bit.  Device ops are replaced by the CPU oracle here (test only)."""
import os
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parent.parent



def _leaves(n):
    """Leaves (off, m) of NumPy's float32 pairwise-sum tree over n elements, in offset order."""
    out = []

    def rec(off, m):
        if m <= 128:
            out.append((off, m))
            return
        n2 = m // 2
        n2 -= n2 % 8
        rec(off, n2)
        rec(off + n2, m - n2)
    rec(0, n)
    return out


def _combine(vals, n):
    """Bottom-up float32 combination of the leaf sums (same tree)."""
    it = iter(vals)

    def rec(m):
        if m <= 128:
            return np.float32(next(it))
        n2 = m // 2
        n2 -= n2 % 8
        a = rec(n2)
        b = rec(m - n2)
        return np.float32(a + b)
    return rec(n)


class StatsOpsMixin:
    """NumPy stand-ins of gsx_pairwise_leaves_dist / gsx_pairwise_finish / threshold (driver logic under test)."""

    def slots(self, n_global):
        return len(_leaves(n_global))

    def leaves(self, a_local, base, n_global, sq, meanstd, halo, bases_dev, world, slot):
        a = a_local.numpy()
        bases = bases_dev.numpy()
        h = halo.numpy().reshape(world, 128)
        mean = np.float32(meanstd.numpy()[0])
        s = slot.numpy()
        s[:] = 0
        for i, (off, m) in enumerate(_leaves(n_global)):
            if not (base <= off < base + len(a)):
                continue
            blk = np.empty(m, np.float32)
            for e in range(m):
                g = off + e
                if g < base + len(a):
                    blk[e] = a[g - base]
                else:
                    r = int(np.searchsorted(bases, g, side="right") - 1)
                    blk[e] = h[r, g - bases[r]]
            if sq:
                blk = (blk - mean) * (blk - mean)
            s[i] = np.add.reduce(blk)

    def finish_stats(self, slot, n_global, sq, meanstd):
        tot = _combine(slot.numpy(), n_global)
        v = np.float32(tot / np.float32(n_global))
        meanstd.numpy()[1 if sq else 0] = np.sqrt(v) if sq else v

    def threshold(self, means_local, meanstd, threshold_factor):
        ms = meanstd.numpy()
        thr = np.float32(ms[0] + np.float32(threshold_factor) * ms[1])
        return torch.from_numpy(means_local.numpy() < thr)


class OracleOps(StatsOpsMixin):
    """Stand-in for the CUDA ops so the collective logic can run on CPU."""

    def build(self, xyz_all):
        import oracle
        pos = xyz_all.numpy()
        lo, cell = oracle.sor_cell_size(pos)
        from oracle.sor import sor_hash_table
        order, cs, cc = sor_hash_table(pos, lo, cell)
        return dict(pos=pos, lo=lo, cell=cell, order=order, cs=cs, cc=cc)

    def mean_dists_range(self, grid, k, hash_mode, out, qb, qe):
        import ctypes
        import oracle
        from oracle import _p
        n = len(grid["pos"])
        spos = np.ascontiguousarray(grid["pos"][grid["order"]])
        md = np.zeros(n, np.float32)
        oracle.lib().orc_sor_mean_dists(_p(spos, ctypes.c_float), _p(grid["cs"], ctypes.c_int32),
                                        _p(grid["cc"], ctypes.c_int32), _p(md, ctypes.c_float), float(grid["lo"][0]),
                                        float(grid["lo"][1]), float(grid["lo"][2]), ctypes.c_float(grid["cell"]), n, n,
                                        min(k, 50), {"i32wrap": 0, "i64": 1}[hash_mode or "i32wrap"], None)
        o = out.numpy()
        o[grid["order"][qb:qe]] = md[qb:qe]   # only this rank's range of sorted positions

    def mask_from_means(self, means, threshold_factor):
        import oracle
        return torch.from_numpy(oracle.threshold_mask(means.numpy(), threshold_factor))


def _worker(rank, world, port, sizes, q):
    sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["OMP_NUM_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsx import dist as gd, synth
    xyz = synth.xyz(sum(sizes), "mixed")
    off = sum(sizes[:rank])
    local = torch.from_numpy(xyz[off:off + sizes[rank]].copy())
    mask, means = gd.sor_filter_sharded(local, 16, 2.0, "i32wrap", return_means=True, ops=OracleOps())
    q.put((rank, mask.numpy(), means.numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("sizes", [(20_000, 20_000), (25_000, 15_001)])
def test_sor_sharded_equals_single(sizes):
    import oracle
    from gsx import synth
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, sizes, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict()
    for _ in range(2):
        r, m, md = q.get(timeout=300)
        res[r] = (m, md)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    xyz = synth.xyz(sum(sizes), "mixed")
    want = oracle.sor_taichi_mean_dists(xyz, 16, "i32wrap")
    wmask = oracle.threshold_mask(want, 2.0)
    got = np.concatenate([res[0][1], res[1][1]])
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(np.concatenate([res[0][0], res[1][0]]), wmask)


def test_query_range_partition():
    from gsx.dist import query_range
    for n in (1, 7, 1000, 10_000_019):
        for w in (1, 2, 4, 8):
            edges = [query_range(n, r, w) for r in range(w)]
            assert edges[0][0] == 0 and edges[-1][1] == n
            assert all(edges[i][1] == edges[i + 1][0] for i in range(w - 1))


def _voxels(a, voxel):
    """floor(a / f32(voxel)) as int64; NaN gives INT64_MIN, as on x86 and in the device kernels."""
    with np.errstate(invalid="ignore"):
        return np.floor(np.asarray(a, np.float32) / np.float32(voxel)).astype(np.int64)


class OracleDensityOps:
    """NumPy stand-in for the CUDA density ops (collective logic under test, CPU/gloo)."""

    def minmax(self, xyz):
        """Like the device min/max (fminf/fmaxf), NaN rows are left out of the box."""
        if xyz.shape[0] == 0:
            return torch.tensor([float("inf")] * 3 + [float("-inf")] * 3, dtype=torch.float32)
        a = xyz.numpy()
        return torch.from_numpy(np.r_[np.fmin.reduce(a, axis=0), np.fmax.reduce(a, axis=0)].astype(np.float32))

    def voxel_range(self, mm, voxel):
        q0, q1 = _voxels(mm[:3], voxel), _voxels(mm[3:], voxel)
        return q0, q1 - q0 + 1

    def grid_count(self, xyz, voxel, q0, dim, grid):
        q = _voxels(xyz.numpy(), voxel)
        inb = np.all((q >= q0) & (q <= q0 + dim - 1), axis=1)
        r = q[inb] - q0
        flat = (r[:, 0] * dim[1] + r[:, 1]) * dim[2] + r[:, 2]
        grid += torch.from_numpy(np.bincount(flat, minlength=grid.numel()).astype(np.int32))

    def grid_dense(self, grid, q0, dim, min_points, n_total):
        g = grid.numpy().reshape(tuple(int(d) for d in dim))
        idx = np.argwhere(g >= max(min_points, 1))
        return idx + q0, g[tuple(idx.T)], int((g > 0).sum())

    def member_mask(self, xyz, voxel, keep):
        q = _voxels(xyz.numpy(), voxel)
        ks = set(map(tuple, keep))
        return torch.from_numpy(np.array([tuple(v) in ks for v in q]))


def _density_worker(rank, world, port, sizes, q):
    sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsx import dist as gd, synth
    xyz = synth.xyz(sum(sizes), "mixed")
    off = sum(sizes[:rank])
    local = torch.from_numpy(xyz[off:off + sizes[rank]].copy())
    out = {}
    for sens, multi in ((0.5, True), (0.9, False)):
        mask, info = gd.density_filter_sharded(local, sensitivity=sens, keep_multicluster=multi,
                                               ops=OracleDensityOps())
        out[(sens, multi)] = (mask.numpy(), info)
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("sizes", [(30_000, 20_000), (30_000, 0, 20_000)])
def test_density_sharded_equals_single(sizes):
    """Includes a rank with an EMPTY slab: it must take part in every collective (no hang)."""
    import oracle
    from gsx import synth
    world = len(sizes)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000) + world
    procs = [ctx.Process(target=_density_worker, args=(r, world, port, sizes, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, out = q.get(timeout=300)
        res[r] = out
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    xyz = synth.xyz(sum(sizes), "mixed")
    for key in res[0]:
        want, info = oracle.density_mask(xyz, sensitivity=key[0], keep_multicluster=key[1])
        got = np.concatenate([res[r][key][0] for r in range(world)])
        assert np.array_equal(got, want), key
        assert all(res[r][key][1]["clusters"] == info["clusters"] for r in range(world))


def _nan_cloud(n, nan_rows):
    """The mixed cloud with NaN in x (every third row also in y and z) at `nan_rows` rows spread over the cloud."""
    from gsx import synth
    xyz = synth.xyz(n, "mixed").copy()
    rows = np.linspace(0, n - 1, nan_rows).astype(np.int64)
    xyz[rows, 0] = np.nan
    xyz[rows[::3], 1:] = np.nan
    return xyz


def _density_nan_worker(rank, world, port, sizes, nan_rows, q):
    sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsx import dist as gd
    from gsx._abi import GsxError
    off = sum(sizes[:rank])
    out = {}
    for k in nan_rows:
        local = torch.from_numpy(_nan_cloud(sum(sizes), k)[off:off + sizes[rank]].copy())
        try:
            mask, info = gd.density_filter_sharded(local, sensitivity=0.5, keep_multicluster=True,
                                                   ops=OracleDensityOps())
            out[k] = (mask.numpy(), info["clusters"])
        except GsxError as e:
            out[k] = str(e)
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_density_sharded_nan_rows():
    """Rows with a NaN coordinate fall outside the global box.  Below min_points of them (275 here) the mask equals
    the oracle's, which puts them in a voxel of their own; at 400, split 200 / 200 so that no single slab reaches
    min_points, every rank refuses."""
    import oracle
    sizes, world = (30_000, 20_000), 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_density_nan_worker, args=(r, world, port, sizes, (100, 400), q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, out = q.get(timeout=300)
        res[r] = out
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    xyz = _nan_cloud(sum(sizes), 100)
    with np.errstate(invalid="ignore"):
        want, info = oracle.density_mask(xyz, sensitivity=0.5, keep_multicluster=True)
    assert np.array_equal(np.concatenate([res[r][100][0] for r in range(world)]), want)
    assert all(res[r][100][1] == info["clusters"] for r in range(world))
    assert not want[np.isnan(xyz).any(axis=1)].any()
    nan_rows = np.isnan(_nan_cloud(sum(sizes), 400)).any(axis=1)
    assert nan_rows[:30_000].sum() < 275 and nan_rows[30_000:].sum() < 275
    for r in range(world):
        assert isinstance(res[r][400], str) and "non-finite" in res[r][400]


class OracleBuildOps:
    """NumPy stand-ins for the CUDA stages of the distributed grid build (gsx.dist._GsxSorOps)."""

    def minmax(self, xyz_local):
        if xyz_local.shape[0] == 0:
            return torch.tensor([float("inf")] * 3 + [float("-inf")] * 3, dtype=torch.float32)
        return torch.cat([xyz_local.min(dim=0).values, xyz_local.max(dim=0).values])
    P = (73856093, 19349663, 83492791)

    def _hash(self, pos, bmin, cell, n_global):
        gi = np.floor((pos - bmin) / np.float32(cell)).astype(np.int32).astype(np.int64)
        return ((gi[:, 0] * self.P[0]) ^ (gi[:, 1] * self.P[1]) ^ (gi[:, 2] * self.P[2])) % n_global

    def cell_size(self, mm, n_global):
        lo, hi = mm[:3], mm[3:]
        vol = np.prod(hi - lo)
        if vol <= 0:
            vol = 1.0
        avg = max(1e-8, vol / n_global)
        return max(float((avg * 32) ** (1.0 / 3.0)), 1e-4)

    def local_run(self, xyz_local, idx_base, n_global, world, bmin, cell):
        pos = xyz_local.numpy()
        owner = self._hash(pos, bmin, cell, n_global) * world // n_global
        order = np.argsort(owner, kind="stable")
        pos4 = np.empty((len(pos), 4), np.float32)
        pos4[:, :3] = pos[order]
        pos4[:, 3] = (idx_base + order).astype(np.int32).view(np.float32)
        cuts = np.searchsorted(owner[order], np.arange(world + 1))
        return torch.from_numpy(pos4), torch.from_numpy(cuts.astype(np.int64))

    def merge_into(self, pos4_r, n_global, bmin, cell, out, flags_out=None, bucket_range=None):
        if pos4_r.shape[0] == 0:
            return
        p = pos4_r.numpy()
        h = self._hash(p[:, :3], bmin, cell, n_global)
        if bucket_range is not None:
            assert np.all((h >= bucket_range[0]) & (h < bucket_range[1]))     # only the owner's buckets arrive
        order = np.argsort(h, kind="stable")
        out.copy_(torch.from_numpy(p[order]))
        if flags_out is not None:   # bit 0: bucket start, bit 1: cell change (first point of the segment: both)
            hs = h[order]
            cells = np.floor((p[order][:, :3] - bmin) / np.float32(cell)).astype(np.int32)
            start = np.r_[True, hs[1:] != hs[:-1]]
            newc = np.r_[True, np.any(cells[1:] != cells[:-1], axis=1)] | start
            flags_out.copy_(torch.from_numpy((start.astype(np.uint8) | (newc.astype(np.uint8) << 1))))

    def new_grid_storage(self, n_global, dev):
        return None, torch.empty((n_global, 4), dtype=torch.float32)

    def finish(self, ws, spos_full, n_global, bmin, cell, flags_full=None):
        sp = spos_full.numpy()
        if flags_full is not None:   # the exchanged flags describe the globally sorted array
            h = self._hash(np.ascontiguousarray(sp[:, :3]), bmin, cell, n_global)
            assert np.array_equal((flags_full.numpy() & 1).astype(bool), np.r_[True, h[1:] != h[:-1]])
        return dict(spos=sp.copy(), bmin=bmin, cell=cell, n=n_global)


class OracleQueryOps(OracleOps):
    def mean_dists_range(self, grid, k, hash_mode, out, qb, qe):
        import ctypes
        import oracle
        from oracle import _p
        n = grid["n"]
        sp = np.ascontiguousarray(grid["spos"][:, :3])
        orig = grid["spos"][:, 3].copy().view(np.int32)
        h = OracleBuildOps()._hash(sp, grid["bmin"], grid["cell"], n).astype(np.int32)
        assert np.all(h[1:] >= h[:-1])                       # the all-gathered array is globally hash-sorted
        uniq, first, cnt = np.unique(h, return_index=True, return_counts=True)
        cs = np.full(n, -1, np.int32)
        cc = np.zeros(n, np.int32)
        cs[uniq], cc[uniq] = first, cnt
        md = np.zeros(n, np.float32)
        b = grid["bmin"]
        oracle.lib().orc_sor_mean_dists(_p(sp, ctypes.c_float), _p(cs, ctypes.c_int32), _p(cc, ctypes.c_int32),
                                        _p(md, ctypes.c_float), float(b[0]), float(b[1]), float(b[2]),
                                        ctypes.c_float(grid["cell"]), n, n, min(k, 50),
                                        {"i32wrap": 0, "i64": 1}[hash_mode or "i32wrap"], None)
        out.numpy()[orig[qb:qe]] = md[qb:qe]

    def mean_dists_strided(self, grid, k, hash_mode, out, stride, phase):
        n = grid["n"]
        full = torch.zeros(n, dtype=torch.float32)
        self.mean_dists_range(grid, k, hash_mode, full, 0, n)           # all queries, then keep this rank's batches
        orig = grid["spos"][:, 3].copy().view(np.int32)
        pos = np.arange(n)
        mine = ((pos // 16) % stride) == phase
        out.numpy()[orig[mine]] = full.numpy()[orig[mine]]


class OracleDistOps(OracleQueryOps, OracleBuildOps):
    pass


def _dist_build_worker(rank, world, port, sizes, q):
    sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["OMP_NUM_THREADS"] = "2"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsx import dist as gd, synth
    xyz = synth.xyz(sum(sizes), "mixed")
    off = sum(sizes[:rank])
    local = torch.from_numpy(xyz[off:off + sizes[rank]].copy())
    mask, means = gd.sor_filter_distributed(local, 16, 2.0, "i64", return_means=True, ops=OracleDistOps())
    q.put((rank, mask.numpy(), means.numpy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("sizes", [(15_000, 15_000), (20_000, 9_999), (7_000, 7_000, 7_001), (9_000, 0, 100, 5_000)])
def test_distributed_build_driver_equals_single(sizes):
    """The host logic of gsx.dist.sor_filter_distributed (one-shot size/box exchange, owner partition, all-to-all with
    split lists, ragged segment exchange, own-segment queries, routing of the means to the slab owners, distributed
    NumPy-order statistics; equal, ragged, tiny and EMPTY slabs) with NumPy stages: bit-identical to the oracle."""
    import oracle
    from gsx import synth
    world = len(sizes)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() % 2000) + world
    procs = [ctx.Process(target=_dist_build_worker, args=(r, world, port, sizes, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(world):
        r, m, md = q.get(timeout=300)
        res[r] = (m, md)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    xyz = synth.xyz(sum(sizes), "mixed")
    want = oracle.sor_taichi_mean_dists(xyz, 16, "i64")
    got = np.concatenate([res[r][1] for r in range(world)])
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(np.concatenate([res[r][0] for r in range(world)]), oracle.threshold_mask(want, 2.0))

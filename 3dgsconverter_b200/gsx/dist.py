"""Multi-GPU (one process per GPU, torch.distributed) versions of the hot path.

SOR (Taichi semantics) is global by construction: the bucket table is a hash of size N_global, and neighbouring
cells hash to arbitrary buckets, so a halo exchange cannot reproduce it (SURVEY 8e).  Scheme of
`sor_filter_distributed` (every rank holds a contiguous slab of the cloud, slabs may be ragged or empty):

  1. ONE all-gather of {n_local, local min/max} (56 B per rank) -> slab bases, N_global, global box -> cell size;
  2. A: stable partition of the slab by BUCKET OWNER (rank o owns the buckets [ceil(o N/G), ceil((o+1) N/G)) ),
     one radix pass; ONE all-gather of the G x G count matrix -> send/recv splits and every owner's segment
     size and base (2 host syncs in total -- they size the buffers);
  3. all-to-all of float4 {x, y, z, global index} (16 B/pt, each point crosses NVLink once);
  4. B: every owner sorts what it received by (bucket, in-cell Morton code) STRAIGHT INTO its slot of the
     global hash-sorted array; the slots are exchanged with one grouped batch of point-to-point sends
     (an all-gather with ragged segment sizes and no staging copy);
  5. C: bucket table, bucket boxes and chunk/super boxes from the sorted array (two streaming passes, replicated);
  6. the sorted order is cut into batches of 16 queries dealt round-robin over the ranks (cost-balanced: every rank
     samples the whole hash range); each rank writes its mean distances at the global original indices of a
     zero-filled vector;
  7. reduce-scatter(sum) of that vector to the slab owners -- every entry has exactly one writer, so x+0 is exact
     (half the traffic of the all-reduce of round 1); ragged slabs fall back to all-reduce + slice;
  8. NumPy-order mean/std of the GLOBAL vector without gathering it: every rank sums the pairwise-tree leaves that
     start in its slab (spill-over from a 128-element halo), the 2^d leaf sums are all-reduced (a few MB),
     the inner nodes are combined replicated; threshold on the local slab.
The mask of every slab is bit-identical to the single-GPU filter on the concatenated cloud
(tests/test_dist_gloo.py on CPU with NumPy stages, tests/test_multigpu_nccl.py and bench.py's `parity` on GPUs).

Density: all-reduce(min/max) -> global voxel box -> rank-local int32 histogram -> ONE all-reduce(sum) of the grid ->
identical host cluster selection on every rank -> local membership mask.
K-Means (SOG chunks) shards by problem: chunks are independent, no data-path collective.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


# ============================================================================ helpers
def _all_gather_rows(x: torch.Tensor, group=None):
    """All-gather a [n_local, C] tensor with possibly different n_local per rank."""
    world = dist.get_world_size(group)
    n_local = torch.tensor([x.shape[0]], dtype=torch.int64, device=x.device)
    sizes = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(sizes, n_local, group=group)
    sizes = [int(s.item()) for s in sizes]
    if len(set(sizes)) == 1:
        out = torch.empty((world * sizes[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x.contiguous(), group=group)
        return out, sizes
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    pad[: x.shape[0]] = x
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([p[:s] for p, s in zip(parts, sizes)], dim=0), sizes


def query_range(n_total: int, rank: int, world: int):
    """Contiguous split of the hash-sorted query positions (replicated-build path)."""
    return (n_total * rank) // world, (n_total * (rank + 1)) // world


def _owner_bounds(n_global: int, world: int):
    """First bucket of every owner: rank o owns the buckets [ceil(o*N/G), ceil((o+1)*N/G))."""
    return [(o * n_global + world - 1) // world for o in range(world + 1)]


def _global_rank(group, r):
    return dist.get_global_rank(group, r) if group is not None else r


def exchange_segments(bufs, seg_sizes, rank: int, group=None):
    """All-gather with ragged segment sizes, in place: every `buf` [sum(seg_sizes), ...] of `bufs` (one tensor or a
    list with the same row partition) already holds this rank's segment at its offset; ONE grouped batch of
    point-to-point operations sends the segments to every peer and receives the peers' segments straight into their
    slots (NCCL runs the batch as one group = an all-to-all pattern over NVSwitch)."""
    if isinstance(bufs, torch.Tensor):
        bufs = [bufs]
    world = len(seg_sizes)
    bases = np.concatenate([[0], np.cumsum(seg_sizes)]).astype(np.int64)
    ops = []
    for step in range(1, world):
        dst = (rank + step) % world
        src = (rank - step) % world
        for buf in bufs:
            if seg_sizes[rank] > 0:
                ops.append(dist.P2POp(dist.isend, buf[bases[rank]: bases[rank + 1]], _global_rank(group, dst), group))
            if seg_sizes[src] > 0:
                ops.append(dist.P2POp(dist.irecv, buf[bases[src]: bases[src + 1]], _global_rank(group, src), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()


def route_to_slabs(full: torch.Tensor, sizes, rank: int, group=None) -> torch.Tensor:
    """`full` [N_global]: every entry written by exactly one rank (0 elsewhere).  Returns this rank's slab of the
    element-wise sum.  Equal slabs on NCCL: reduce-scatter (half the bytes of an all-reduce); otherwise all-reduce."""
    if len(set(sizes)) == 1 and sizes[0] > 0 and dist.get_backend(group) == "nccl":
        out = torch.empty(sizes[0], dtype=full.dtype, device=full.device)
        dist.reduce_scatter_tensor(out, full, op=dist.ReduceOp.SUM, group=group)
        return out
    dist.all_reduce(full, op=dist.ReduceOp.SUM, group=group)
    off = int(sum(sizes[:rank]))
    return full[off: off + sizes[rank]]


# ============================================================================ SOR: device stages (replaceable in tests)
class _GsxSorOps:
    """Device stages of the distributed SOR (CPU/gloo tests substitute NumPy stand-ins)."""

    def minmax(self, xyz_local):
        """float32[6] {min xyz, max xyz} of the slab on its device; +/-inf for an empty slab."""
        from . import sor
        from ._abi import lib, check
        from .sor import _ptr, _stream
        dev = xyz_local.device
        n = xyz_local.shape[0]
        if n == 0:
            return torch.tensor([float("inf")] * 3 + [float("-inf")] * 3, dtype=torch.float32, device=dev)
        ws = torch.empty(32768, dtype=torch.uint8, device=dev)  # reduction scratch (24 KiB)
        out = torch.empty(8, dtype=torch.float32, device=dev)
        check(lib.gsx_sor_minmax(_ptr(xyz_local), n, _ptr(out), _ptr(ws), ws.numel(), _stream()), "gsx_sor_minmax")
        return out[:6]

    def cell_size(self, mm: np.ndarray, n_global: int) -> float:
        import ctypes as C
        from ._abi import lib
        return float(lib.gsx_sor_cell_size(mm.ctypes.data_as(C.POINTER(C.c_float)), n_global))

    def local_run(self, xyz_local, idx_base, n_global, world, bmin, cell):
        """A: stable partition of the slab by bucket owner.  Returns (pos4 [n,4] float32, cuts int64[world+1])."""
        import ctypes as C
        from . import sor
        from ._abi import lib, check
        from .sor import _ptr, _stream
        dev = xyz_local.device
        n_local = xyz_local.shape[0]
        ws_l = sor.workspace(max(n_local, 1), dev)
        pos4 = torch.empty((n_local, 4), dtype=torch.float32, device=dev)
        cuts = torch.zeros(world + 1, dtype=torch.int64, device=dev)
        check(lib.gsx_sor_dist_local_run(_ptr(xyz_local), n_local, idx_base, n_global, world,
                                         bmin.ctypes.data_as(C.POINTER(C.c_float)), cell, _ptr(pos4), _ptr(cuts),
                                         _ptr(ws_l), ws_l.numel(), _stream()), "gsx_sor_dist_local_run")
        return pos4, cuts

    def merge_into(self, pos4_r, n_global, bmin, cell, out, flags_out=None, bucket_range=None):
        """B: sort the received points of this rank's bucket range by (bucket, in-cell Morton) into `out`; with
        `flags_out` (uint8 per point) also the bucket-start / cell-change flags stage C consumes."""
        import ctypes as C
        from . import sor
        from ._abi import lib, check
        from .sor import _ptr, _stream
        m = pos4_r.shape[0]
        if m == 0:
            return
        ws_m = sor.workspace(m, pos4_r.device)
        lo, hi = bucket_range if bucket_range is not None else (0, n_global)
        check(lib.gsx_sor_dist_merge(_ptr(pos4_r), m, n_global, int(lo), int(hi),
                                     bmin.ctypes.data_as(C.POINTER(C.c_float)), cell, _ptr(out), _ptr(flags_out), _ptr(ws_m),
                                     ws_m.numel(), _stream()), "gsx_sor_dist_merge")

    def new_grid_storage(self, n_global, dev):
        """Workspace of the final grid and a [n_global,4] view of its sorted-position array (exchange target)."""
        from ._abi import lib
        ws = torch.empty(lib.gsx_sor_grid_workspace_bytes(n_global), dtype=torch.uint8, device=dev)  # no sort buffers
        off = lib.gsx_sor_spos_offset(n_global)
        return ws, ws[off: off + n_global * 16].view(torch.float32).view(n_global, 4)

    def finish(self, ws, spos_full, n_global, bmin, cell, flags_full=None):
        """C: table, boxes and bucket boxes from the globally sorted array (and the owners' flags, if exchanged)."""
        import ctypes as C
        from . import sor
        from ._abi import lib, check
        from .sor import _ptr, _stream
        check(lib.gsx_sor_build_from_sorted(_ptr(spos_full), _ptr(flags_full), n_global,
                                            bmin.ctypes.data_as(C.POINTER(C.c_float)), cell, _ptr(ws), ws.numel(),
                                            _stream()), "gsx_sor_build_from_sorted")
        return sor.SorGrid(n_global, ws, bmin, cell)

    # replicated-build path
    def build(self, xyz_all):
        from . import sor
        return sor.build_grid(xyz_all)

    def mean_dists_range(self, grid, k, hash_mode, out, qb, qe):
        from . import sor
        sor.mean_dists(grid, k, hash_mode, out=out, q_range=(qb, qe))

    def mean_dists_strided(self, grid, k, hash_mode, out, stride, phase):
        from . import sor
        sor.mean_dists_strided(grid, k, hash_mode, out, stride, phase)

    def mask_from_means(self, means, threshold_factor):
        from . import sor
        return sor.threshold_mask(means, sor.mean_std(means), threshold_factor)

    # distributed statistics
    def leaves(self, a_local, base, n_global, sq, meanstd, halo, bases_dev, world, slot):
        from ._abi import lib, check
        from .sor import _ptr, _stream
        check(lib.gsx_pairwise_leaves_dist(_ptr(a_local), base, a_local.numel(), n_global, sq, _ptr(meanstd), _ptr(halo),
                                           _ptr(bases_dev), world, _ptr(slot), _stream()), "gsx_pairwise_leaves_dist")

    def slots(self, n_global):
        from ._abi import lib
        return int(lib.gsx_pairwise_slots(n_global))

    def finish_stats(self, slot, n_global, sq, meanstd):
        from ._abi import lib, check
        from .sor import _ptr, _stream
        check(lib.gsx_pairwise_finish(_ptr(slot), n_global, sq, _ptr(meanstd), _stream()), "gsx_pairwise_finish")

    def threshold(self, means_local, meanstd, threshold_factor):
        from . import sor
        if means_local.numel() == 0:
            return torch.zeros(0, dtype=torch.bool, device=means_local.device)
        return sor.threshold_mask(means_local, meanstd, threshold_factor)


_GsxOps = _GsxSorOps          # names of round 1 (tests inject subclasses of these)
_GsxBuildOps = _GsxSorOps


def mean_std_distributed(a_local: torch.Tensor, sizes, rank: int, group=None, ops=None) -> torch.Tensor:
    """np.mean / np.std (float32 pairwise order) of the concatenation of every rank's `a_local`, without gathering
    it: tensor [mean, std] on the device, the same bits on every rank as gsx_mean_std_f32 on the whole vector."""
    ops = ops or _GsxSorOps()
    world = len(sizes)
    dev = a_local.device
    n_global = int(sum(sizes))
    bases = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    head = torch.zeros(128, dtype=torch.float32, device=dev)
    m = min(128, a_local.numel())
    if m:
        head[:m] = a_local[:m]
    halo = torch.empty(world * 128, dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(halo, head, group=group)
    bases_dev = torch.from_numpy(bases).to(dev)
    slot = torch.empty(ops.slots(n_global), dtype=torch.float32, device=dev)
    meanstd = torch.zeros(2, dtype=torch.float32, device=dev)
    for sq in (0, 1):
        ops.leaves(a_local, int(bases[rank]), n_global, sq, meanstd, halo, bases_dev, world, slot)
        dist.all_reduce(slot, op=dist.ReduceOp.SUM, group=group)
        ops.finish_stats(slot, n_global, sq, meanstd)
    return meanstd


class _Stamps:
    """Optional CUDA-event stamps at the stage boundaries (bench.py's per-stage and NCCL-time break-down)."""

    def __init__(self, enabled, dev):
        self.on = bool(enabled) and dev.type == "cuda"
        self.ev = []

    def mark(self, name):
        if self.on:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.ev.append((name, e))

    def result(self):
        if not self.on or len(self.ev) < 2:
            return {}
        torch.cuda.synchronize()
        out = {}
        for (_, a), (name, b) in zip(self.ev[:-1], self.ev[1:]):
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        return out


def build_grid_distributed(xyz_local: torch.Tensor, group=None, ops=None, stamps=None):
    """Hash grid of the UNION cloud without replicating the sort (steps 1-5 of the module docstring).
    Returns (grid over n_global points, slab sizes, segment sizes of the owners)."""
    ops = ops or _GsxSorOps()
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = xyz_local.device
    n_local = xyz_local.shape[0]
    st = stamps or _Stamps(False, dev)
    st.mark("start")
    # 1. slab sizes + global bounding box in one exchange (float64 carries the int and the float32s exactly)
    head = torch.empty(7, dtype=torch.float64, device=dev)
    head[0] = float(n_local)
    head[1:] = ops.minmax(xyz_local).to(torch.float64)
    heads = torch.empty(world * 7, dtype=torch.float64, device=dev)
    dist.all_gather_into_tensor(heads, head, group=group)
    heads = heads.cpu().numpy().reshape(world, 7)                 # host sync 1
    sizes = [int(v) for v in heads[:, 0]]
    n_global = int(sum(sizes))
    idx_base = int(sum(sizes[:rank]))
    if n_global == 0:
        raise ValueError("sor: empty cloud")
    mm = np.concatenate([heads[:, 1:4].min(axis=0), heads[:, 4:7].max(axis=0)]).astype(np.float32)
    cell = ops.cell_size(mm, n_global)
    if cell != cell:
        from ._abi import GsxError
        raise GsxError("sor: non-finite coordinates")
    bmin = mm[:3].copy()
    st.mark("sync")
    # 2. A: stable partition by bucket owner; the G x G count matrix gives every split and segment size
    pos4, cuts = ops.local_run(xyz_local, idx_base, n_global, world, bmin, cell)
    send = (cuts[1:] - cuts[:-1]).contiguous()
    st.mark("build_A_partition")
    counts = torch.empty(world * world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(counts, send, group=group)
    counts = counts.cpu().numpy().reshape(world, world)           # host sync 2: counts[r][o] = r sends to owner o
    send_l = [int(v) for v in counts[rank]]
    recv_l = [int(v) for v in counts[:, rank]]
    seg_sizes = [int(v) for v in counts.sum(axis=0)]
    m = seg_sizes[rank]
    seg_base = int(sum(seg_sizes[:rank]))
    st.mark("sync")
    # 3. each point crosses NVLink once, to the owner of its bucket
    pos4_r = torch.empty((m, 4), dtype=torch.float32, device=dev)
    dist.all_to_all_single(pos4_r, pos4, recv_l, send_l, group=group)
    st.mark("nccl_all_to_all")
    # 4. B: owner sort straight into the slot, then the ragged all-gather of the slots
    ws, spos_full = ops.new_grid_storage(n_global, dev)
    flags_full = torch.empty(n_global, dtype=torch.uint8, device=dev)   # bit 0 bucket start, bit 1 cell change
    ob = _owner_bounds(n_global, world)
    ops.merge_into(pos4_r, n_global, bmin, cell, spos_full[seg_base: seg_base + m], flags_full[seg_base: seg_base + m],
                   bucket_range=(ob[rank], ob[rank + 1]))
    st.mark("build_B_owner_sort")
    exchange_segments([spos_full, flags_full], seg_sizes, rank, group)
    st.mark("nccl_segments")
    # 5. C: table, boxes, bucket boxes -- replicated, two streaming passes over n_global (no re-hash: owners' flags)
    grid = ops.finish(ws, spos_full, n_global, bmin, cell, flags_full)
    st.mark("build_C_table_boxes")
    return grid, sizes, seg_sizes


def sor_filter_distributed(xyz_local: torch.Tensor, k: int = 25, threshold_factor: float = 1.0,
                           hash_mode: str | None = None, group=None, return_means: bool = False, ops=None,
                           build_ops=None, timings: dict | None = None):
    """SOR keep-mask of this rank's slab, bit-identical to the single-GPU filter on the union cloud."""
    ops = ops or _GsxSorOps()
    rank = dist.get_rank(group)
    dev = xyz_local.device
    st = _Stamps(timings is not None, dev)
    grid, sizes, seg_sizes = build_grid_distributed(xyz_local, group, ops=build_ops or ops, stamps=st)
    n = int(sum(sizes))
    means_full = torch.zeros(n, dtype=torch.float32, device=dev)
    # batches of 16 consecutive sorted positions dealt round-robin over the ranks: every rank samples the whole hash
    # range, so the expensive clustered buckets do not all land on the owner of their hash range
    ops.mean_dists_strided(grid, k, hash_mode, means_full, dist.get_world_size(group), rank)
    st.mark("knn")
    means_local = route_to_slabs(means_full, sizes, rank, group)
    st.mark("nccl_route_means")
    meanstd = mean_std_distributed(means_local, sizes, rank, group, ops=ops)
    mask = ops.threshold(means_local, meanstd, threshold_factor)
    st.mark("stats_mask")
    if timings is not None:
        timings.update(st.result())
    return (mask, means_local) if return_means else mask


sor_filter_sharded_v2 = sor_filter_distributed   # round-1 name


def sor_filter_sharded(xyz_local: torch.Tensor, k: int = 25, threshold_factor: float = 1.0,
                       hash_mode: str | None = None, group=None, return_means: bool = False, ops=None):
    """Replicated-build variant (all-gather the raw xyz, every rank builds the whole grid, sharded queries, one
    all-reduce): kept as the simple reference implementation of the sharded filter and for A/B timing."""
    ops = ops or _GsxSorOps()
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    xyz_all, sizes = _all_gather_rows(xyz_local, group)
    n = xyz_all.shape[0]
    grid = ops.build(xyz_all)
    qb, qe = query_range(n, rank, world)
    means = torch.zeros(n, dtype=torch.float32, device=xyz_all.device)
    ops.mean_dists_range(grid, k, hash_mode, means, qb, qe)
    dist.all_reduce(means, op=dist.ReduceOp.SUM, group=group)
    mask_all = ops.mask_from_means(means, threshold_factor)
    off = sum(sizes[:rank])
    sl = slice(off, off + sizes[rank])
    return (mask_all[sl], means[sl]) if return_means else mask_all[sl]


def sor_filter_auto(xyz_local, k=25, threshold_factor=1.0, hash_mode=None, group=None, return_means=False,
                    timings=None):
    """The distributed build is the default for every world size; GSX_DIST_BUILD=0 selects the replicated one."""
    import os
    if os.environ.get("GSX_DIST_BUILD", "1") == "0":
        return sor_filter_sharded(xyz_local, k, threshold_factor, hash_mode, group=group, return_means=return_means)
    return sor_filter_distributed(xyz_local, k, threshold_factor, hash_mode, group=group, return_means=return_means,
                                  timings=timings)


# ============================================================================ K-Means
def kmeans_chunks_sharded(X_chunks, K: int, max_iter: int, inits, group=None, runner=None):
    """SOG shN schedule across ranks: chunk p goes to rank p % world; no collective on the data path.
    X_chunks / inits: lists (only the entries owned by this rank need to be real tensors).
    Returns {chunk index: (C, labels, counts)} for the chunks this rank owns."""
    from . import kmeans as gk
    runner = runner or gk.kmeans_lloyd
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    out = {}
    for p in range(len(X_chunks)):
        if p % world == rank:
            out[p] = runner(X_chunks[p], K, max_iter, inits[p])
    return out


# ============================================================================ density
class _GsxDensityOps:
    """Device ops of the sharded density filter (replaceable in CPU/gloo tests)."""

    def minmax(self, xyz):
        if xyz.shape[0] == 0:
            return torch.tensor([float("inf")] * 3 + [float("-inf")] * 3, dtype=torch.float32, device=xyz.device)
        if xyz.is_cuda:
            return _GsxSorOps().minmax(xyz)
        return torch.cat([xyz.min(dim=0).values, xyz.max(dim=0).values])

    def voxel_range(self, mm, voxel):
        from . import density
        return density.voxel_range(mm, voxel)

    def grid_count(self, xyz, voxel, q0, dim, grid):
        from . import density
        density.grid_count(xyz, voxel, q0, dim, grid)

    def grid_dense(self, grid, q0, dim, min_points, n_total):
        from . import density
        return density.grid_dense(grid, q0, dim, min_points, n_total)

    def member_mask(self, xyz, voxel, keep):
        from . import density
        return density.member_mask(xyz, voxel, keep)


def density_filter_sharded(xyz_local: torch.Tensor, voxel_size=1.0, threshold_percentage=0.32, sensitivity=None,
                           keep_multicluster=False, group=None, ops=None):
    """Density keep-mask of this rank's slab, identical to the single-GPU filter on the union cloud.
    all-reduce(min/max) of 6 floats -> global voxel box -> rank-local int32 histogram -> ONE all-reduce(sum)
    of the grid -> identical (tiny) host cluster selection on every rank -> local membership mask.
    Empty slabs take part in every collective (min/max = +/-inf, zero histogram)."""
    from . import density
    ops = ops or _GsxDensityOps()
    if sensitivity is not None:
        voxel_size, threshold_percentage = density.slider(sensitivity)
    dev = xyz_local.device
    n_here = xyz_local.shape[0]
    n_local = torch.tensor([n_here], dtype=torch.int64, device=dev)
    dist.all_reduce(n_local, group=group)
    n_total = int(n_local.item())
    empty_info = dict(clusters=0, max_len=0, dense=0, voxels=0)
    if n_total == 0:
        return torch.zeros(0, dtype=torch.bool, device=dev), empty_info
    mm = ops.minmax(xyz_local)
    lo, hi = mm[:3].clone(), mm[3:].clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=group)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=group)
    q0, dim = ops.voxel_range(torch.cat([lo, hi]).cpu().numpy(), voxel_size)
    ncell = int(dim[0]) * int(dim[1]) * int(dim[2])
    if ncell > density.GRID_CELL_LIMIT:
        # sparse far-flung cloud: replicate (all-gather) and run the single-GPU hash-table path on every rank
        xyz_all, sizes = _all_gather_rows(xyz_local, group)
        mask_all, info = density.density_filter(xyz_all, voxel_size, threshold_percentage, None, keep_multicluster)
        off = sum(sizes[: dist.get_rank(group)])
        return mask_all[off: off + n_here], info
    grid = torch.zeros(ncell, dtype=torch.int32, device=dev)
    if n_here:
        ops.grid_count(xyz_local, voxel_size, q0, dim, grid)
    dist.all_reduce(grid, op=dist.ReduceOp.SUM, group=group)
    min_points = int(n_total * (threshold_percentage / 100.0))  # data_processor.py:48 on the global count
    vox, cnt, n_unique = ops.grid_dense(grid, q0, dim, min_points, n_total)
    if len(vox) == 0:
        return torch.zeros(n_here, dtype=torch.bool, device=dev), dict(empty_info, voxels=n_unique)
    keep, n_kept, max_len = density.select_clusters(vox, keep_multicluster)
    if n_here:
        mask = ops.member_mask(xyz_local, voxel_size, keep)
    else:
        mask = torch.zeros(0, dtype=torch.bool, device=dev)
    return mask, dict(clusters=n_kept, max_len=max_len, dense=len(vox), voxels=n_unique)


# ============================================================================ the whole chain on a sharded cloud
class ShardedFilterChain:
    """converter.py:194-236 (bbox -> alpha -> density -> SOR) on a cloud sharded over the ranks: every rank keeps
    its slab's working set (xyz, opacity, surviving local row indices) in HBM; bbox / alpha need no communication,
    density and SOR are the global filters above.  Masks equal the single-GPU chain on the concatenated cloud."""

    def __init__(self, xyz_local: torch.Tensor, opacity_local: torch.Tensor | None = None, group=None):
        from .pipeline import FilterChain
        self.group = group
        self.chain = FilterChain(xyz_local, opacity_local, device=xyz_local.device)

    @property
    def count(self):
        return self.chain.count

    def global_count(self) -> int:
        t = torch.tensor([self.chain.count], dtype=torch.int64, device=self.chain.xyz.device)
        dist.all_reduce(t, group=self.group)
        return int(t.item())

    def crop_by_bbox(self, *bbox):
        return self.chain.crop_by_bbox(*bbox)

    def alpha(self, min_opacity_u8):
        return self.chain.alpha(min_opacity_u8)

    def density(self, voxel_size=1.0, threshold_percentage=0.32, sensitivity=None, keep_multicluster=False):
        mask, info = density_filter_sharded(self.chain.xyz, voxel_size, threshold_percentage, sensitivity,
                                            keep_multicluster, group=self.group)
        if info["dense"] == 0 or info["clusters"] == 0:
            self.chain.clear()
        else:
            self.chain._apply(mask)
        return self.chain.count, info

    def sor(self, k=25, threshold_factor=1.0, hash_mode=None, timings=None):
        mask = sor_filter_auto(self.chain.xyz, k, threshold_factor, hash_mode, group=self.group, timings=timings)
        self.chain._apply(mask)
        return self.chain.count

    def local_indices(self) -> torch.Tensor:
        """Surviving rows of this rank's slab (device int64)."""
        if self.chain.idx is None:
            return torch.arange(self.chain.n0, device=self.chain.xyz.device)
        return self.chain.idx.to(torch.int64)

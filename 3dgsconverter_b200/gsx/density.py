"""Density filter: device voxel histogram + membership mask, host cluster selection.

Mirrors ``DataProcessor.apply_density_filter`` (data_processor.py:11-117).  The connected-component
step runs on the host over the (tiny) dense-voxel list and reproduces the reference's discovery order
(Python ``set`` over lexicographically inserted tuples, stable sort by size) because it decides ties.
"""
from __future__ import annotations

import ctypes as C
from collections import deque

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream
from .sor import _check_xyz


def slider(sensitivity: float):
    """data_processor.py:17-28: --density_sensitivity -> (voxel_size, threshold_percentage)."""
    voxel = max(0.1, 2.0 - (sensitivity * 1.8))
    thr = 0.1 + (sensitivity * 0.9)
    return voxel, thr


def dense_voxels(xyz: torch.Tensor, voxel_size: float, min_points: int):
    """Voxels with count >= min_points, sorted lexicographically (the order np.unique gives the
    reference, data_processor.py:43,51-52).  Returns (vox int64[M,3], counts int32[M], n_unique_voxels)."""
    _check_xyz(xyz)
    n = xyz.shape[0]
    thr = max(int(min_points), 1)
    cap = n // thr + 1
    nbytes = lib.gsx_density_workspace_bytes(n, cap)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=xyz.device)
    vox = np.empty((cap, 3), dtype=np.int64)
    cnt = np.empty(cap, dtype=np.int32)
    nd = C.c_int64(0)
    nv = C.c_int64(0)
    check(lib.gsx_density_voxel_count(_ptr(xyz), n, float(np.float32(voxel_size)), int(min_points),
                                      vox.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), cap,
                                      C.byref(nd), C.byref(nv), _ptr(ws), ws.numel(), _stream()),
          "gsx_density_voxel_count")
    m = nd.value
    vox, cnt = vox[:m], cnt[:m]
    order = np.lexsort((vox[:, 2], vox[:, 1], vox[:, 0]))
    return vox[order], cnt[order], nv.value, ws


def select_clusters(dense_vox: np.ndarray, keep_multicluster: bool):
    """6-connected components over the dense voxels; keep the largest (or all >= 5 % of it).
    data_processor.py:59-106.  Returns (kept voxels int64[M,3], kept_clusters, max_len)."""
    dense = set(map(tuple, dense_vox))  # insertion in lexicographic order, like the reference (:59)
    seen: set = set()
    comps: list = []
    for seed in dense:  # set iteration order decides which of two equally large clusters is "first"
        if seed in seen:
            continue
        comp = [seed]
        seen.add(seed)
        todo = deque(comp)
        while todo:
            x, y, z = todo.popleft()
            for nb in ((x - 1, y, z), (x + 1, y, z), (x, y - 1, z), (x, y + 1, z), (x, y, z - 1), (x, y, z + 1)):
                if nb in dense and nb not in seen:
                    seen.add(nb)
                    comp.append(nb)
                    todo.append(nb)
        comps.append(comp)
    if not comps:
        return np.empty((0, 3), np.int64), 0, 0
    comps.sort(key=len, reverse=True)  # stable: ties keep discovery order
    max_len = len(comps[0])
    need = max_len * 0.05 if keep_multicluster else max_len
    kept, n_kept = [], 0
    for comp in comps:
        if len(comp) >= need:
            kept.extend(comp)
            n_kept += 1
            if not keep_multicluster:
                break
    return np.asarray(kept, dtype=np.int64).reshape(-1, 3), n_kept, max_len


def member_mask(xyz: torch.Tensor, voxel_size: float, keep_vox: np.ndarray, ws: torch.Tensor | None = None):
    """data_processor.py:111-112: point kept <=> its voxel is one of keep_vox."""
    _check_xyz(xyz)
    n = xyz.shape[0]
    keep_vox = np.ascontiguousarray(keep_vox, dtype=np.int64).reshape(-1, 3)
    need = max(64, 1 << int(np.ceil(np.log2(max(2 * len(keep_vox), 1))))) * 16 + 256   # two-word keys if far apart
    if len(keep_vox):   # room for the bitmap form of the set (one bit per voxel of the kept voxels' box, <= 16 MiB)
        bits = int(np.prod((keep_vox.max(axis=0) - keep_vox.min(axis=0) + 1).astype(np.float64)))
        if bits <= (1 << 27):
            need = max(need, bits // 8 + 256)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=xyz.device)
    mask = torch.empty(n, dtype=torch.uint8, device=xyz.device)
    check(lib.gsx_density_member_mask(_ptr(xyz), n, float(np.float32(voxel_size)), keep_vox.ctypes.data_as(C.c_void_p),
                                      len(keep_vox), _ptr(mask), _ptr(ws), ws.numel(), _stream()),
          "gsx_density_member_mask")
    return mask.view(torch.bool)


def density_filter(xyz: torch.Tensor, voxel_size=1.0, threshold_percentage=0.32, sensitivity=None,
                   keep_multicluster=False):
    """Keep-mask of apply_density_filter on a device tensor.  Returns (mask bool[N], info dict)."""
    if sensitivity is not None:
        voxel_size, threshold_percentage = slider(sensitivity)
    n = xyz.shape[0]
    min_points = int(n * (threshold_percentage / 100.0))  # data_processor.py:48
    vox, cnt, n_unique, ws = dense_voxels(xyz, voxel_size, min_points)
    if len(vox) == 0:
        return torch.zeros(n, dtype=torch.bool, device=xyz.device), dict(clusters=0, max_len=0, dense=0,
                                                                         voxels=n_unique)
    keep, n_kept, max_len = select_clusters(vox, keep_multicluster)
    mask = member_mask(xyz, voxel_size, keep, ws)
    return mask, dict(clusters=n_kept, max_len=max_len, dense=len(vox), voxels=n_unique)


# ------------------------------------------------------------------ staged / sharded form
GRID_CELL_LIMIT = 1 << 28   # 1 GiB of int32 counters


def voxel_range(minmax: np.ndarray, voxel_size: float):
    """Voxel-space origin and extent of a bounding box (floor(x / f32(voxel)) is monotone)."""
    mm = np.ascontiguousarray(minmax, dtype=np.float32)
    q0 = (C.c_int64 * 3)()
    dim = (C.c_int64 * 3)()
    lib.gsx_density_voxel_range(mm.ctypes.data_as(C.POINTER(C.c_float)), float(np.float32(voxel_size)), q0, dim)
    return np.array(q0[:], dtype=np.int64), np.array(dim[:], dtype=np.int64)


def grid_count(xyz: torch.Tensor, voxel_size: float, q0: np.ndarray, dim: np.ndarray, grid: torch.Tensor):
    """Accumulate this slab's voxel histogram into `grid` (int32, prod(dim) cells, caller-zeroed)."""
    _check_xyz(xyz)
    oob = torch.zeros(1, dtype=torch.int64, device=xyz.device)
    q0c = (C.c_int64 * 3)(*[int(v) for v in q0])
    dimc = (C.c_int64 * 3)(*[int(v) for v in dim])
    check(lib.gsx_density_grid_count(_ptr(xyz), xyz.shape[0], float(np.float32(voxel_size)), q0c, dimc, _ptr(grid),
                                     _ptr(oob), _stream()), "gsx_density_grid_count")
    return oob


def grid_dense(grid: torch.Tensor, q0: np.ndarray, dim: np.ndarray, min_points: int, n_total: int):
    """Dense voxels (count >= max(min_points,1)) of an (all-reduced) grid, lexicographically sorted."""
    thr = max(int(min_points), 1)
    cap = n_total // thr + 1
    ws = torch.empty(cap * 28 + 4096, dtype=torch.uint8, device=grid.device)
    vox = np.empty((cap, 3), dtype=np.int64)
    cnt = np.empty(cap, dtype=np.int32)
    nd, nv = C.c_int64(0), C.c_int64(0)
    q0c = (C.c_int64 * 3)(*[int(v) for v in q0])
    dimc = (C.c_int64 * 3)(*[int(v) for v in dim])
    check(lib.gsx_density_grid_dense(_ptr(grid), q0c, dimc, int(min_points), vox.ctypes.data_as(C.c_void_p),
                                     cnt.ctypes.data_as(C.c_void_p), cap, C.byref(nd), C.byref(nv), _ptr(ws),
                                     ws.numel(), _stream()), "gsx_density_grid_dense")
    vox, cnt = vox[: nd.value], cnt[: nd.value]
    order = np.lexsort((vox[:, 2], vox[:, 1], vox[:, 0]))
    return vox[order], cnt[order], nv.value

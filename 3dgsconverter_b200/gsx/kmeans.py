"""Lloyd K-Means on device buffers: host plumbing over gsx_kmeans_* (gpu_ops.py:27-46,178-191)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ._abi import lib, check, KM_ASSIGN
from ._abi import _ptr, _stream


def tensor_core_supported(K: int, D: int) -> bool:
    return bool(lib.gsx_kmeans_tensor_core_supported(int(K), int(D)))


def kmeans_lloyd_batched(X: torch.Tensor, row_off, K: int, max_iter: int, init: torch.Tensor,
                         assign: str | None = None, want_stats: bool = False):
    """`nprob` independent problems stored back to back in X[*,D] (rows row_off[p]:row_off[p+1]),
    each with K centroids.  init: float32 [nprob,K,D] (consumed as the start, not modified).
    assign: "auto" (None), "strict" or "tensor" -- the labels are bit-identical in every mode.
    Returns (C [nprob,K,D], labels int32 [N] (problem-local ids), counts int32 [nprob,K]) (+ tensor-core stats)."""
    if not X.is_cuda or X.dtype != torch.float32 or not X.is_contiguous() or X.dim() != 2:
        raise ValueError("X must be a contiguous float32 CUDA tensor [N,D]")
    row_off = np.ascontiguousarray(row_off, dtype=np.int64)
    nprob = len(row_off) - 1
    D = X.shape[1]
    mode = KM_ASSIGN[assign or "auto"]
    Cc = init.to(device=X.device, dtype=torch.float32).reshape(nprob, K, D).contiguous().clone()
    labels = torch.zeros(X.shape[0], dtype=torch.int32, device=X.device)
    counts = torch.zeros(nprob * K, dtype=torch.int32, device=X.device)
    stats = torch.zeros(4, dtype=torch.int64, device=X.device) if want_stats else None
    ws = torch.empty(lib.gsx_kmeans_workspace_bytes(X.shape[0], nprob, K, D), dtype=torch.uint8, device=X.device)
    check(lib.gsx_kmeans_lloyd_device(_ptr(X), row_off.ctypes.data_as(C.POINTER(C.c_int64)), nprob, K, D, max_iter,
                                      _ptr(Cc), _ptr(labels), _ptr(counts), _ptr(ws), ws.numel(), mode, _ptr(stats),
                                      _stream()), "gsx_kmeans_lloyd_device")
    if want_stats:
        v = stats.cpu().numpy()
        return Cc, labels, counts.reshape(nprob, K), dict(strict_evals=int(v[0]), multi_candidate_points=int(v[1]),
                                                          full_scans=int(v[2]))
    return Cc, labels, counts.reshape(nprob, K)


def kmeans_lloyd(X: torch.Tensor, K: int, max_iter: int, init: torch.Tensor, assign: str | None = None):
    """Single problem.  Returns (C [K,D], labels [N], counts [K])."""
    Cc, labels, counts = kmeans_lloyd_batched(X, [0, X.shape[0]], K, max_iter, init.reshape(1, K, -1), assign)
    return Cc[0], labels, counts[0]


def tc_debug_scores(X: torch.Tensor, Cc: torch.Tensor) -> torch.Tensor:
    """Raw tensor-core scores of the first 128 rows of X against the centroids Cc [K,D] (test hook)."""
    K, D = Cc.shape
    npad = (K + 31) // 32 * 32
    out = torch.zeros((128, npad), dtype=torch.float32, device=X.device)
    ws = torch.zeros(4096, dtype=torch.uint8, device=X.device)
    check(lib.gsx_kmeans_tc_debug_scores(_ptr(X), X.shape[0], _ptr(Cc.contiguous()), K, D, _ptr(out), _ptr(ws), ws.numel(),
                                         _stream()), "gsx_kmeans_tc_debug_scores")
    return out


def kmeans_host(data: np.ndarray, K: int, max_iter: int, init: np.ndarray, assign: str | None = None):
    """Host-buffer entry (copies inside libgsx): binding target for gpu_ops.kmeans' GPU path.
    Returns (C [K,D], labels int32[N])."""
    Cc, labels = kmeans_host_batched(data, [0, len(data)], K, max_iter, init, assign)
    return Cc[0], labels


def kmeans_host_batched(base: np.ndarray, row_off, K: int, max_iter: int, init: np.ndarray, assign: str | None = None):
    """Host-buffer entry for several problems stored back to back in `base` [N,D] (the SOG shN chunk schedule):
    one upload, one batched launch per phase.  init float32 [nprob,K,D].  Returns (C [nprob,K,D], labels int32[N])."""
    X = np.ascontiguousarray(base, dtype=np.float32)
    row_off = np.ascontiguousarray(row_off, dtype=np.int64)
    nprob = len(row_off) - 1
    D = X.shape[1]
    Cc = np.ascontiguousarray(init, dtype=np.float32).reshape(nprob, K, D).copy()
    labels = np.zeros(int(row_off[-1]), dtype=np.int32)
    check(lib.gsx_kmeans_host_batched(X.ctypes.data_as(C.c_void_p), row_off.ctypes.data_as(C.POINTER(C.c_int64)), nprob, K,
                                      D, max_iter, Cc.ctypes.data_as(C.c_void_p), labels.ctypes.data_as(C.c_void_p),
                                      KM_ASSIGN[assign or "auto"]), "gsx_kmeans_host_batched")
    return Cc, labels


def device_free_bytes() -> int:
    f, t = C.c_int64(0), C.c_int64(0)
    check(lib.gsx_device_memory(C.byref(f), C.byref(t)), "gsx_device_memory")
    return int(f.value)

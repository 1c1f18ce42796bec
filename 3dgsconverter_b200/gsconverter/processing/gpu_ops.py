"""Drop-in for ``gsconverter/processing/gpu_ops.py`` backed by libgsx.so (hand-written sm_90a CUDA).

Same importable surface as the reference (gpu_ops.py:8-46,193-263):

    HAS_TAICHI                      bool   -- name kept because data_processor.py:144 and
                                              formats/sog.py:524 read it; True <=> the gsx CUDA backend
                                              is usable (a CUDA device is present)
    kmeans(data, k, max_iter=10, tolerance=1e-4, use_gpu=True, verbose=False) -> (centroids, labels)
    filter_sor_gpu(data_np, k=25, threshold_factor=1.0, verbose=False)        -> bool mask | None

Differences that are deliberate: there is NO silent CPU fallback.  libgsx.so missing => ImportError at
import; a failing CUDA call => GsxError propagates (the reference swallowed it and ran scikit-learn).
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

import numpy as np

try:
    import gsx  # noqa: F401
except ImportError:  # dropped into a foreign tree: locate the backend next to this repo or via GSX_HOME
    _home = os.environ.get("GSX_HOME") or str(Path(__file__).resolve().parents[2])
    if _home not in sys.path:
        sys.path.insert(0, _home)
    import gsx  # noqa: F401  (ImportError here is fatal on purpose: no CPU fallback)

from gsx import backend_available

HAS_TAICHI = backend_available()


def _hash_mode():
    # "i32wrap" reproduces the Taichi kernel's default-int arithmetic (SURVEY F8); "i64" is the intended hash.
    return os.environ.get("GSX_SOR_HASH", "i32wrap")


# ---------------------------------------------------------------------------------------------------------------
# Batch-ahead for the SOG shN loop (formats/sog.py:536-549).  The reference clusters the SH block chunk by chunk:
#     for i in range(num_chunks): c, l = gpu_ops.kmeans(sh_data_flat[start:end], this_k, max_iter=10)
# Every chunk is a row-range VIEW of one float32 array and nothing else touches the global NumPy RNG inside the loop.
# So when the first chunk arrives (a view starting at row 0 of a larger base array) the whole schedule is known: the
# SH block is uploaded ONCE, the init rows of every chunk are drawn in call order from the global RNG, and all chunks
# run in ONE batched launch (gsx_kmeans_lloyd_device with nprob problems).  The following calls return their cached
# result after checking that they are exactly the predicted call (same base array, rows, k, max_iter) AND that the
# global RNG is in exactly the state the reference would have left it in (state after the previous chunk's draw);
# the RNG is then advanced to the state after this chunk's draw.  Any deviation drops the cache and falls back to
# the per-call path -- results and RNG stream are identical to chunk-by-chunk execution either way.
_BATCH = None
BATCH_AHEAD = os.environ.get("GSX_KMEANS_BATCH_AHEAD", "1") == "1"
batch_stats = {"batched_launches": 0, "served_from_batch": 0, "single_calls": 0, "dropped": 0}


def _chunk_view(data):
    base = data.base
    if not isinstance(base, np.ndarray) or base.ndim != 2 or data.ndim != 2:
        return None
    if base.dtype != np.float32 or data.dtype != np.float32 or base.shape[1] != data.shape[1]:
        return None
    if not (base.flags.c_contiguous and data.flags.c_contiguous):
        return None
    off = data.ctypes.data - base.ctypes.data
    rowb = base.shape[1] * 4
    if off < 0 or off % rowb or off // rowb + data.shape[0] > base.shape[0]:
        return None
    return base, off // rowb


def _rng_same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _run_batch(base, plan, max_iter):
    """One upload of the rows involved, one batched launch per distinct K (gsx_kmeans_host_batched).
    plan: [(start, end, k, init | None)]."""
    from gsx import kmeans as _km
    results = [None] * len(plan)
    by_k = {}
    for i, (s, e, k, init) in enumerate(plan):
        if init is not None:
            by_k.setdefault(k, []).append(i)
    for k, idxs in by_k.items():
        runs = []   # maximal runs of consecutive chunks: back-to-back rows of the block
        for i in idxs:
            if runs and runs[-1][-1] == i - 1:
                runs[-1].append(i)
            else:
                runs.append([i])
        for run in runs:
            s0, e1 = plan[run[0]][0], plan[run[-1]][1]
            offs = [plan[i][0] - s0 for i in run] + [e1 - s0]
            Cn, Ln = _km.kmeans_host_batched(base[s0:e1], offs, k, int(max_iter), np.stack([plan[i][3] for i in run]))
            for j, i in enumerate(run):
                results[i] = (np.ascontiguousarray(Cn[j]), np.ascontiguousarray(Ln[offs[j]: offs[j + 1]]))
            batch_stats["batched_launches"] += 1
    return results


def _try_batched(data, k, max_iter):
    """Serve this call from (or start) a batch-ahead plan; None = take the per-call path."""
    global _BATCH
    info = _chunk_view(data)
    if info is None:
        if _BATCH is not None:
            _BATCH, batch_stats["dropped"] = None, batch_stats["dropped"] + 1
        return None
    base, start = info
    n = data.shape[0]
    b = _BATCH
    if b is not None:
        i = b["next"]
        ok = (b["base"] is base and b["ptr"] == base.ctypes.data and b["shape"] == base.shape and i < len(b["plan"])
              and b["plan"][i][:3] == (start, start + n, k) and b["max_iter"] == max_iter
              and _rng_same(np.random.get_state(), b["states"][i]))
        if ok:
            np.random.set_state(b["states"][i + 1])
            res = b["results"][i]
            b["results"][i] = None
            b["next"] = i + 1
            if b["next"] == len(b["plan"]):
                _BATCH = None
            batch_stats["served_from_batch"] += 1
            return res
        _BATCH, batch_stats["dropped"] = None, batch_stats["dropped"] + 1
    N = base.shape[0]
    if start != 0 or n >= N or k >= n:
        return None
    nch = -(-N // n)
    if not (2 <= nch <= 64):
        return None
    try:
        from gsx import kmeans as _km
        if base.nbytes * 1.25 + (64 << 20) > _km.device_free_bytes():
            return None   # the block does not fit next to its workspace: chunk by chunk
    except Exception:
        return None
    states = [np.random.get_state()]
    plan = []
    for i in range(nch):
        s, e = i * n, min((i + 1) * n, N)
        ki = min(e - s, k)                                  # sog.py:542 this_k = min(len(chunk), k_per_chunk)
        if ki >= e - s:                                      # gpu_ops.py:30-31 passthrough: no draw, no clustering
            plan.append((s, e, ki, None))
        else:
            plan.append((s, e, ki, base[s:e][np.random.choice(e - s, ki, replace=False)].astype(np.float32)))
        states.append(np.random.get_state())
    results = _run_batch(base, plan, max_iter)
    for i, (s, e, ki, init) in enumerate(plan):
        if init is None:
            results[i] = (base[s:e].copy(), np.arange(e - s, dtype=np.int32))
    np.random.set_state(states[1])
    _BATCH = dict(base=base, ptr=base.ctypes.data, shape=base.shape, plan=plan, states=states, results=results,
                  max_iter=max_iter, next=1)
    res = results[0]
    results[0] = None
    batch_stats["served_from_batch"] += 1
    return res


def kmeans(data: np.ndarray, k: int, max_iter=10, tolerance=1e-4, use_gpu=True, verbose=False):
    """gpu_ops.py:27-46.  ``tolerance`` is accepted and ignored, as in the reference (F9)."""
    n, d = data.shape
    if k >= n:  # gpu_ops.py:30-31
        return data.copy(), np.arange(n, dtype=np.int32)
    if not use_gpu:
        # explicit request for the reference's CPU algorithm (gpu_ops.py:34-38, 48-52): scikit-learn
        # MiniBatchKMeans, unseeded -- a different algorithm, outside the parity contract.
        from sklearn.cluster import MiniBatchKMeans
        km = MiniBatchKMeans(n_clusters=k, max_iter=max_iter, batch_size=min(4096 * 4, len(data)), n_init="auto",
                             compute_labels=True)
        km.fit(data)
        return km.cluster_centers_.astype(np.float32), km.labels_.astype(np.int32)
    if not HAS_TAICHI:
        raise RuntimeError("gsx: no CUDA device available and CPU fallback is disabled by design")
    from gsx import kmeans as _km
    if BATCH_AHEAD and d >= 2:
        r = _try_batched(data, int(k), int(max_iter))
        if r is not None:
            return r
    batch_stats["single_calls"] += 1
    x = data.astype(np.float32, copy=False)   # (the reference copies, gpu_ops.py:181; same values, 140 MB less traffic)
    # exactly the reference's draw from the global NumPy RNG (gpu_ops.py:182) so np.random.seed reproduces
    init = x[np.random.choice(n, k, replace=False)].astype(np.float32)
    centroids, labels = _km.kmeans_host(x, int(k), int(max_iter), init)
    return centroids, labels


def filter_sor_gpu(data_np: np.ndarray, k: int = 25, threshold_factor: float = 1.0, verbose=False):
    """gpu_ops.py:193-263: keep-mask of the statistical outlier removal, or None if no backend."""
    if not HAS_TAICHI:
        return None
    n, d = data_np.shape
    if d != 3:
        raise ValueError("Requires 3D data")
    from gsx import sor as _sor
    if os.environ.get("GSX_SOR_SEMANTICS", "taichi") == "ckdtree":
        # opt-in: the arithmetic of the reference's CPU path (data_processor.py:155-180, exact float64 KNN)
        return _sor.ckdtree_filter_host(data_np, int(k), float(threshold_factor))
    return _sor.sor_filter_host(data_np, int(k), float(threshold_factor), hash_mode=_hash_mode())

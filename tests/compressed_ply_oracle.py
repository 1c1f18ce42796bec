"""NumPy restatement of the PlayCanvas compressed PLY writer's arithmetic (CompressedPlyFormat.write,
formats/compressed_ply.py:126-250 of 3dgsconverter) for a given splat order, vectorised over all chunks, plus the
inputs of tests/golden/g10_reference_compressed_ply_small.npz and the packed-word comparison the tests use.

Float32 semantics of NumPy 2: Python float constants are weak scalars (rounded to float32 first)."""
from __future__ import annotations

import hashlib

import numpy as np

SH_C0 = 0.28209479177387814
SQRT2_2 = 0.7071067811865476
CHUNK = 256
CHUNK_FIELDS = ("min_x", "min_y", "min_z", "max_x", "max_y", "max_z",
                "min_scale_x", "min_scale_y", "min_scale_z", "max_scale_x", "max_scale_y", "max_scale_z",
                "min_r", "min_g", "min_b", "max_r", "max_g", "max_b")
VERTEX_FIELDS = ("packed_position", "packed_rotation", "packed_scale", "packed_color")


def _per_splat(v, n):
    return np.repeat(v, CHUNK)[:n]


def _unorm(v, lo, hi, t):
    """clip(floor((v - min) / (max - min) * t + 0.5), 0, t), or 0 where the chunk's float32 extent is < f32(1e-5)."""
    n = len(v)
    lo_s, hi_s = _per_splat(lo, n), _per_splat(hi, n)
    ext = hi_s - lo_s
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.clip(np.floor((v - lo_s) / ext * t + 0.5), 0, t)
    return np.where(ext < np.float32(1e-5), 0, q).astype(np.uint32)


def _pack_quat(q):
    q = [x.astype(np.float32) for x in q]
    ss = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]   # serial order of np.linalg.norm over 4 values
    d = np.sqrt(ss) + 1e-10
    q = np.stack([x / d for x in q], axis=1)
    largest = np.argmax(np.abs(q), axis=1)
    sign = np.sign(q[np.arange(len(q)), largest])
    res = largest.astype(np.uint32)
    for i in range(4):
        comp = np.clip(np.floor((q[:, i] * sign * SQRT2_2 + 0.5) * 1023 + 0.5), 0, 1023).astype(np.uint32)
        res = np.where(largest != i, (res << 10) | comp, res)
    return res


def sh_names(a: np.ndarray, order=None):
    """compressed_ply.py:141-169: the f_rest_i kept for the last index (44 .. 0) with a value != 0."""
    names = a.dtype.names
    last = -1
    for i in range(44, -1, -1):
        f = f"f_rest_{i}"
        if f in names and np.any(a[f] != 0):
            last = i
            break
    need = 45 if last >= 24 else 24 if last >= 9 else 9 if last >= 0 else 0
    return [f"f_rest_{i}" for i in range(need) if f"f_rest_{i}" in names]


def encode(a: np.ndarray, order) -> tuple:
    """(chunk_data, vertex_data, sh_data or None) of CompressedPlyFormat.write for the records `a` in `order`."""
    s = a[np.asarray(order, np.int64)]
    n = len(s)
    starts = np.arange(0, n, CHUNK)

    def bounds(v):
        if n == 0:
            return np.empty(0, np.float32), np.empty(0, np.float32)
        return np.minimum.reduceat(v, starts), np.maximum.reduceat(v, starts)

    pos = [s[f] for f in ("x", "y", "z")]
    scl = [np.clip(s[f"scale_{i}"], -20, 20) for i in range(3)]
    rgb = [s[f"f_dc_{i}"] * SH_C0 + 0.5 for i in range(3)]
    bp, bs, bc = [bounds(v) for v in pos], [bounds(v) for v in scl], [bounds(v) for v in rgb]
    chunk = np.zeros(len(starts), dtype=[(f, "f4") for f in CHUNK_FIELDS])
    for group, b in (("", bp), ("scale_", bs)):
        for i, ax in enumerate("xyz"):
            chunk[f"min_{group}{ax}"], chunk[f"max_{group}{ax}"] = b[i]
    for i, ch in enumerate("rgb"):
        chunk[f"min_{ch}"], chunk[f"max_{ch}"] = bc[i]

    vertex = np.zeros(n, dtype=[(f, "u4") for f in VERTEX_FIELDS])
    vertex["packed_position"] = (_unorm(pos[0], *bp[0], 2047) << 21) | (_unorm(pos[1], *bp[1], 1023) << 11) | \
        _unorm(pos[2], *bp[2], 2047)
    vertex["packed_scale"] = (_unorm(scl[0], *bs[0], 2047) << 21) | (_unorm(scl[1], *bs[1], 1023) << 11) | \
        _unorm(scl[2], *bs[2], 2047)
    vertex["packed_rotation"] = _pack_quat([s[f"rot_{i}"] for i in range(4)])
    with np.errstate(over="ignore"):
        alpha = 1.0 / (1.0 + np.exp(-s["opacity"]))
    na = np.clip(np.floor(alpha * 255 + 0.5), 0, 255).astype(np.uint32)
    vertex["packed_color"] = (_unorm(rgb[0], *bc[0], 255) << 24) | (_unorm(rgb[1], *bc[1], 255) << 16) | \
        (_unorm(rgb[2], *bc[2], 255) << 8) | na

    names = sh_names(s)
    sh = None
    if names:
        sh = np.zeros(n, dtype=[(f, "u1") for f in names])
        for f in names:
            sh[f] = np.clip((s[f] / 8.0 + 0.5) * 256, 0, 255).astype(np.uint8)
    return chunk, vertex, sh


def assert_packed_equal(got: tuple, want: tuple):
    """Chunk rows (as uint32), the four packed words of every splat and the SH bytes, all bit-exact."""
    gc, gv, gs = got
    wc, wv, ws = want
    assert gc.dtype.names == wc.dtype.names and len(gc) == len(wc)
    bad = np.flatnonzero(np.ascontiguousarray(gc).view(np.uint32) != np.ascontiguousarray(wc).view(np.uint32))
    assert bad.size == 0, f"chunk rows differ at flat index {bad[:10]}"
    assert gv.dtype.names == wv.dtype.names and len(gv) == len(wv)
    for f in VERTEX_FIELDS[:4]:
        bad = np.flatnonzero(gv[f] != wv[f])
        assert bad.size == 0, f"{f} differs at {bad[:10]}: {gv[f][bad[:5]]} vs {wv[f][bad[:5]]}"
    if ws is None:
        assert gs is None
    else:
        assert gs is not None and gs.dtype.names == ws.dtype.names
        assert np.array_equal(np.ascontiguousarray(gs).view(np.uint8), np.ascontiguousarray(ws).view(np.uint8))


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def golden_inputs() -> dict:
    """The two inputs of g10_reference_compressed_ply_small.npz, regenerated from gsx.synth (pinned by SHA-256):
    'mixed' -- 12 000 SH-3 rows with edge rows spliced in; 'deg1' -- 3 000 rows whose f_rest_9..44 are zero."""
    from gsx import synth
    a = synth.structured(12_000, "mixed")
    rng = np.random.default_rng(10)
    a["x"][:600], a["y"][:600], a["z"][:600] = 1.25, -3.5, 2.0          # 600 coincident splats: a chunk of equal positions
    b = slice(1000, 1400)                                                # a blob tighter than one Morton cell: recursion
    a["x"][b], a["y"][b], a["z"][b] = (np.float32(v) + rng.normal(0, 1e-4, 400).astype(np.float32)
                                       for v in (4.0, 4.0, -4.0))
    quats = [(0, 0, 0, 0), (0.5, 0.5, 0.5, 0.5), (0.5, -0.5, 0.5, -0.5), (-0.9, 0.1, 0.2, 0.3), (0.1, -0.2, -0.95, 0.1),
             (0.0, 0.0, -0.0, -1.0), (3.0, 4.0, 0.0, 0.0), (1e-30, 0, 0, 0)]
    for k, q in enumerate(quats):
        for i in range(4):
            a[f"rot_{i}"][2000 + k] = q[i]
    for k, v in enumerate((25.0, -25.0, 20.0, -20.0, 19.99, -19.99, 1e6, -1e6)):
        a[f"scale_{k % 3}"][2100 + k] = v
    for k, v in enumerate((5.0, -5.0, 4.0, -4.0, 3.99, -4.01, 100.0, -100.0, 1e-7, -1e-7)):
        a[f"f_rest_{(7 * k) % 45}"][2200 + k] = v
    for k, v in enumerate((200.0, -200.0, 88.0, -88.0, 20.0, -20.0)):
        a["opacity"][2300 + k] = v
    d = synth.structured(3_000, "uniform")
    for i in range(9, 45):
        d[f"f_rest_{i}"] = 0.0
    return {"mixed": a, "deg1": d}

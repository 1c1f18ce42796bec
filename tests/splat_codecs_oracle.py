"""NumPy restatement of the .ksplat, .spz and .splat writers of 3dgsconverter (KSplatFormat.write,
formats/ksplat.py:319-544; SpzFormat.write / _pack_v3, spz.py:49-173; SplatFormat.write, splat.py:82-166), plus the
inputs and cases of tests/golden/g12_reference_splat_codecs_small.npz.

Float32 semantics of NumPy 2: Python float constants are weak scalars (rounded to float32 first).  The .splat order is
NumPy's stable argsort (equal metrics keep ascending index)."""
from __future__ import annotations

import hashlib
import struct

import numpy as np

SH_C0 = 0.28209479177387814
SQRT1_2 = 0.707106781186547524401


def _nonzero(a, f):
    return f in a.dtype.names and bool(np.any(a[f] != 0))


def _u8_color(dc):
    return np.clip((0.5 + SH_C0 * dc) * 255, 0, 255).astype(np.uint8)


def _u8_alpha(op):
    return np.clip((1 / (1 + np.exp(-op))) * 255, 0, 255).astype(np.uint8)


def ksplat_file(a: np.ndarray, compression_level=0, sh_level=None, bucket_size=256, block_size=5.0) -> bytes:
    """The bytes KSplatFormat.write writes for `a`."""
    level, n = int(compression_level), len(a)
    bucket_size = 256 if bucket_size is None else int(bucket_size)
    block_size = 5.0 if block_size is None else float(block_size)
    degree = 0
    if any(_nonzero(a, f"f_rest_{j}") for j in range(9)):
        degree = 2 if any(_nonzero(a, f"f_rest_{j}") for j in range(9, 24)) else 1
    if sh_level is not None and int(sh_level) < degree:
        degree = int(sh_level)
    sh_count = {1: 9, 2: 24}.get(degree, 0)
    head = bytearray(4096)
    head[1] = 1
    struct.pack_into("<IIIIH", head, 4, 1, 1, n, n, level)
    struct.pack_into("<ff", head, 36, -2.0, 2.0)
    sec = bytearray(1024)
    struct.pack_into("<II", sec, 0, n, n)
    full, partial = n // bucket_size, int(n % bucket_size != 0)
    if level >= 1:
        struct.pack_into("<IIfHxxI", sec, 8, bucket_size, full + partial, block_size, 12, 32767)
    item = 4 if level == 0 else 2 if level == 1 else 1
    per = (44 if level == 0 else 24) + item * sh_count
    struct.pack_into("<IIIH", sec, 28, partial * 4 + (12 * (full + partial) if level else 0) + n * per, full, partial,
                     degree)
    parts = [bytes(head), bytes(sec)] + ([struct.pack("<I", n % bucket_size)] if partial else [])
    xyz = [a[f] for f in ("x", "y", "z")]
    f_pos, f_lin = (np.float32, np.float32) if level == 0 else (np.uint16, np.float16)
    f_sh = np.float32 if level == 0 else np.float16 if level == 1 else np.uint8
    layout = [("pos", f_pos, 3), ("scale", f_lin, 3), ("rot", f_lin, 4), ("color", np.uint8, 4)]
    rec = np.zeros(n, dtype=[(k, t, (c,)) for k, t, c in layout + ([("sh", f_sh, sh_count)] if sh_count else [])])
    with np.errstate(all="ignore"):
        if level >= 1:
            starts = np.arange(0, n, bucket_size)
            centres = np.zeros((0, 3), np.float32)
            if n:
                centres = np.stack([(np.minimum.reduceat(v, starts) + np.maximum.reduceat(v, starts)) / 2.0
                                    for v in xyz], 1).astype(np.float32)
            parts.append(centres.tobytes())
            c = centres[np.arange(n) // bucket_size]
            sf = np.float32(32767 / (block_size / 2.0))
            rec["pos"] = np.stack([np.clip(np.round((v - c[:, k]) * sf) + 32767, 0, 65535).astype(np.uint16)
                                   for k, v in enumerate(xyz)], 1)
        else:
            rec["pos"] = np.stack(xyz, 1)
        rec["scale"] = np.stack([np.exp(a[f"scale_{k}"]) for k in range(3)], 1).astype(f_lin)
        rec["rot"] = np.stack([a[f"rot_{k}"] for k in range(4)], 1).astype(f_lin)
        rec["color"] = np.stack([_u8_color(a[f"f_dc_{k}"]) for k in range(3)] + [_u8_alpha(a["opacity"])], 1)
        if sh_count:
            sh = np.stack([a[f"f_rest_{j}"] for j in range(sh_count)], 1)
            if level == 2:
                sh = np.clip((sh - -2.0) / 4.0 * 255, 0, 255)
            rec["sh"] = sh.astype(f_sh)
    return b"".join(parts + [rec.tobytes()])


def spz_degree(a: np.ndarray) -> int:
    names = a.dtype.names
    if "f_rest_0" not in names:
        return 0
    top = 44 if "f_rest_44" in names else 23 if "f_rest_23" in names else 8 if "f_rest_8" in names else -1
    last = next((i for i in range(top, -1, -1) if _nonzero(a, f"f_rest_{i}")), -1)
    return 3 if last >= 24 else 2 if last >= 9 else 1 if last >= 0 else 0


def _smallest_three(w, x, y, z):
    n = len(w)
    norm = np.sqrt(w * w + x * x + y * y + z * z + 1e-9)
    R = np.stack([x / norm, y / norm, z / norm, w / norm], 1)
    big = np.argmax(np.abs(R), 1)
    flip = R[np.arange(n), big] < 0
    out = big.astype(np.uint32) << 30
    for j in range(4):
        sel = big != j
        v = R[sel, j]                          # the same subset the reference casts (its SIMD tail included)
        mag = np.clip(np.abs(v) * (511.0 / SQRT1_2) + 0.5, 0, 511).astype(np.uint32)
        sign = (np.not_equal(v < 0, flip[sel])).astype(np.uint32)
        shift = (2 - (j - (big[sel] < j))).astype(np.uint32) * 10
        out[sel] |= ((sign << 9) | mag) << shift
    return out


def spz_payload(a: np.ndarray) -> bytes:
    """The uncompressed bytes SpzFormat.write hands to gzip.compress (KeyError where the reference raises one)."""
    n, degree = len(a), spz_degree(a)
    dim = {0: 0, 1: 3, 2: 8, 3: 15}[degree]
    sh = [a[f"f_rest_{i + 15 * c}"] for i in range(dim) for c in range(3)]
    with np.errstate(all="ignore"):
        q = np.round(np.stack([a[f] * 4096 for f in ("x", "y", "z")], 1)).astype(np.int32)
        pos = q.astype("<i4").view(np.uint8).reshape(n, 3, 4)[:, :, :3]
        alpha = (1.0 / (1.0 + np.exp(-np.clip(a["opacity"], -20, 20))) * 255.0).astype(np.uint8)
        col = np.stack([np.clip((a[f"f_dc_{k}"] * 0.15 + 0.5) * 255.0, 0, 255).astype(np.uint8) for k in range(3)], 1)
        scl = np.stack([np.clip((a[f"scale_{k}"] + 10.0) * 16.0, 0, 255).astype(np.uint8) for k in range(3)], 1)
        rot = _smallest_three(*(a[f"rot_{k}"] for k in range(4)))
        parts = [struct.pack("<IIIBBBB", 0x5053474E, 3, n, degree, 12, 1, 0), pos.tobytes(), alpha.tobytes(),
                 col.tobytes(), scl.tobytes(), rot.astype("<u4").tobytes()]
        if dim:
            v = np.stack(sh, 1)
            out = np.zeros(v.shape, np.uint8)
            for cols, bs in ((slice(0, 9), 8), (slice(9, None), 16)):
                qi = np.round(v[:, cols] * 128.0 + 128.0).astype(np.int32)
                out[:, cols] = np.clip((qi + bs // 2) // bs * bs, 0, 255).astype(np.uint8)
            parts.append(out.tobytes())
    return b"".join(parts)


def splat_order(a: np.ndarray) -> np.ndarray:
    with np.errstate(all="ignore"):
        metric = np.exp(a["scale_0"] + a["scale_1"] + a["scale_2"]) * (1.0 / (1.0 + np.exp(-a["opacity"])))
    return np.argsort(-metric, kind="stable")


def splat_file(a: np.ndarray) -> bytes:
    """The bytes SplatFormat.write writes for `a`, equal metrics in ascending index."""
    s = a[splat_order(a)]
    rec = np.zeros(len(s), dtype=[("pos", "<f4", (3,)), ("scale", "<f4", (3,)), ("color", "u1", (4,)),
                                  ("rot", "u1", (4,))])
    with np.errstate(all="ignore"):
        rec["pos"] = np.stack([s[f] for f in ("x", "y", "z")], 1)
        rec["scale"] = np.exp(np.stack([s[f"scale_{k}"] for k in range(3)], 1))
        r = [s[f"rot_{k}"] for k in range(4)]
        norm = np.sqrt(r[0] ** 2 + r[1] ** 2 + r[2] ** 2 + r[3] ** 2)
        rec["rot"] = np.stack([np.clip(v / norm * 128 + 128, 0, 255) for v in r], 1).astype(np.uint8)
        rec["color"] = np.stack([_u8_color(s[f"f_dc_{k}"]) for k in range(3)] + [_u8_alpha(s["opacity"])], 1)
    return rec.tobytes()


def digest(a) -> str:
    return hashlib.sha256(a if isinstance(a, bytes) else np.ascontiguousarray(a).tobytes()).hexdigest()


# (compression_level, sh_level, bucket_size, block_size) of every ksplat case of the golden
KSPLAT_CASES = [(0, None, 256, 5.0), (1, None, 256, 5.0), (2, None, 256, 5.0), (5, None, 256, 5.0),
                (1, None, 7, 5.0), (2, None, 1, 5.0), (1, None, 256, 2.5), (1, 0, 256, 5.0), (2, 1, 7, 5.0)]


def ksplat_tag(case) -> str:
    lv, shl, bs, blk = case
    return f"ksplat_l{lv}_sh{shl}_b{bs}_k{blk}"


def golden_inputs() -> dict:
    """The inputs of g12_reference_splat_codecs_small.npz, regenerated from gsx.synth (pinned by SHA-256)."""
    from gsx import synth
    f32 = np.float32
    a = synth.structured(2002, "mixed")                          # 2002 = 7 * 286: whole 7-buckets, a partial 256
    nan, inf = f32(np.nan), f32(np.inf)
    for k, v in enumerate((nan, inf, -inf)):                      # positions (ksplat buckets, SPZ cast)
        a[("x", "y", "z")[k]][10 + k] = v
    for k, v in enumerate((3000.0, -3000.0, 2048.0, -2048.0, 2047.99, 1e6, -1e6, 524288.0, -524288.5, 5e5)):
        a[("x", "y", "z")[k % 3]][20 + k] = v                     # past 2^23 / 4096 and past int32 after * 4096
    for k, v in enumerate((nan, inf, -inf, 12.0, -12.0, 11.09, 11.1, -15.0, -17.0, -25.0, 89.0, -104.0, 0.0, -0.0)):
        a[f"scale_{k % 3}"][40 + k] = v                           # float16 overflow / subnormal / zero, exp limits
    for k, v in enumerate((nan, -nan, inf, -inf, 20.0, -20.0, 20.5, -20.5, 25.0, -25.0, 100.0, -100.0, 0.0, -0.0)):
        a["opacity"][60 + k] = v
    quats = [(0, 0, 0, 0), (nan, 0.1, 0.2, 0.3), (0.1, nan, 0.2, 0.3), (inf, 0, 0, 0), (0, 0, -inf, 1),
             (0.5, 0.5, 0.5, 0.5), (-0.5, 0.5, -0.5, 0.5), (0.0, -0.0, 0.0, -1.0), (3.0, 4.0, 0.0, 0.0),
             (1e-30, 0, 0, 0), (1e20, 1e20, 0, 0), (-0.6, 0.6, 0.3, -0.3)]
    for k, q in enumerate(quats):
        for i in range(4):
            a[f"rot_{i}"][80 + k] = q[i]
    for k, v in enumerate((nan, inf, -inf, 1e6, -1e6)):
        a[f"f_dc_{k % 3}"][100 + k] = v
    # SH on the rint and floor-division boundaries of the SPZ quantiser (v * 128 + 128 = m + 0.5, q + bs/2 = k * bs),
    # the ksplat uint8 mapping, float16 limits, NaN and +-inf
    sh_vals = [(m + 0.5 - 128) / 128 for m in (3, 4, 11, 12, 123, 124, 131, 132, 251, 252)]
    sh_vals += [(k * 8 - 4 - 128) / 128 for k in (1, 16, 31)] + [(k * 16 - 8 - 128) / 128 for k in (1, 8, 15)]
    sh_vals += [2.0, -2.0, 2.01, -2.01, 70000.0, -1e-7, 3e-8, 1e10, -1e10, 300.0, -1.5, nan, inf, -inf, -0.0]
    for k, v in enumerate(sh_vals):
        for c in (0, 15, 30, 8, 23, 44):
            a[f"f_rest_{(k + c) % 45}"][120 + k] = v
    a["x"][300:310] = 0.0                                         # mixed-sign zeros inside a bucket
    a["x"][300:310:2] = -0.0
    for r in (400, 401, 402, 1990, 1991):                         # exact .splat metric ties (and identical rows)
        a[r] = a[399]
    for f in ("scale_0", "scale_1", "scale_2", "opacity"):
        a[f][500:505] = a[f][505]
    out = {"mixed3": a}
    for deg in (0, 1, 2):
        c = synth.structured(1500, "uniform")
        for i in range((0, 9, 24)[deg], 45):
            c[f"f_rest_{i}"] = 0.0
        c["f_rest_44"][::7] = -0.0
        out[f"content{deg}"] = c
    out["fields0"] = synth.structured(700, "mixed", sh_degree=0)
    out["fields1"] = synth.structured(700, "mixed", sh_degree=1)      # the reference SPZ writer rejects it
    for n in (0, 1, 255, 256, 257):
        out[f"n{n}"] = synth.structured(n, "mixed")
    return out

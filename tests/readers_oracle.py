"""NumPy restatement of the reference's .splat, .ksplat, .spz and compressed PLY readers (formats/splat.py:9-80,
ksplat.py:29-317, spz.py:18-47 and 175-296, compressed_ply.py:14-123 and 342-378), statement for statement, from the
file's bytes; the reference for the device readers at sizes the golden fixture does not reach.  Each reader raises
ValueError where gsx's `decode` refuses (the reference raises there, or returns something the device does not
reproduce).  Returns (array, metadata)."""
import gzip
import struct

import numpy as np

from gsx.compressed_ply import CHUNK_DTYPE, FIXED_FIELDS, VERTEX_DTYPE
from gsx.readers import gaussian_dtype, parse_ply_header

SH_C0 = 0.28209479177387814


def _logit_u8(u8):
    v = u8.astype(np.float32) / 255.0
    v = np.clip(v, 1e-7, 1.0 - 1e-7)
    return np.log(v / (1.0 - v))


def splat(buf: bytes):
    n = len(buf) // 32
    raw = np.frombuffer(buf, np.dtype([("x", "f4"), ("y", "f4"), ("z", "f4"), ("scale_0", "f4"), ("scale_1", "f4"),
                                       ("scale_2", "f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1"),
                                       ("opacity", "u1"), ("rot_0", "u1"), ("rot_1", "u1"), ("rot_2", "u1"),
                                       ("rot_3", "u1")]), count=n)
    out = np.zeros(n, gaussian_dtype(has_rgb=True, sh_degree=0))
    for f in "xyz":
        out[f] = raw[f]
    for k in range(3):
        out[f"scale_{k}"] = np.log(np.maximum(raw[f"scale_{k}"], 1e-6))
    r = [(raw[f"rot_{k}"].astype(np.float32) - 128) / 128.0 for k in range(4)]
    norms = np.maximum(np.sqrt(r[0] ** 2 + r[1] ** 2 + r[2] ** 2 + r[3] ** 2), 1e-6)
    for k in range(4):
        out[f"rot_{k}"] = r[k] / norms
    la = np.clip(raw["opacity"].astype(np.float32) / 255.0, 1.0 / 255.0, 0.9999)
    out["opacity"] = -np.log((1.0 / la) - 1.0)
    for k, c in enumerate(("red", "green", "blue")):
        out[f"f_dc_{k}"] = (raw[c].astype(np.float32) / 255.0 - 0.5) / SH_C0
    return out, None


SECTION_KEYS = ("splatCount", "maxSplatCount", "bucketSize", "bucketCount", "bucketBlockSize", "bucketStorageSizeBytes",
                "compressionScaleRange", "storageSizeBytes", "fullBucketCount", "partiallyFilledBucketCount",
                "shDegree")


def ksplat(buf: bytes):
    if len(buf) < 4096 or (buf[0], buf[1]) != (0, 1):
        raise ValueError("header")
    msc, _, _, splat_count = struct.unpack_from("<IIII", buf, 4)
    level = struct.unpack_from("<H", buf, 20)[0]
    min_sh, max_sh = struct.unpack_from("<ff", buf, 36)
    payload = 4096 + 1024 * msc
    if payload > len(buf):
        raise ValueError("section headers")
    secs = []
    for i in range(msc):
        s = dict(zip(SECTION_KEYS, struct.unpack_from("<IIIIfHxxIIIIH", buf, 4096 + 1024 * i)))
        if s["compressionScaleRange"] == 0 and level >= 1:
            s["compressionScaleRange"] = 32767
        secs.append(s)
    meta = {"v_major": buf[0], "v_minor": buf[1], "splat_count": splat_count, "compression_level": level,
            "min_sh": min_sh, "max_sh": max_sh, "sections": secs}
    degree = max((s["shDegree"] for s in secs), default=3)
    if degree > 255:
        raise ValueError("degree")
    dtype = gaussian_dtype(sh_degree=degree)
    parts, off = [], payload
    for s in secs:
        n, npfb, nb = s["splatCount"], s["partiallyFilledBucketCount"], s["bucketCount"]
        lengths = np.frombuffer(buf, "<u4", npfb, off) if off + 4 * npfb <= len(buf) else None
        off += 4 * npfb
        centres = np.frombuffer(buf, "<f4", 3 * nb, off).reshape(-1, 3) if off + 12 * nb <= len(buf) else None
        off += 12 * nb
        sh_count = {1: 9, 2: 24}.get(s["shDegree"], 0)
        if level == 0:
            raw_dt = [("pos", "3f4"), ("scale", "3f4"), ("rot", "4f4"), ("color", "4u1")]
            per = 44 + 4 * sh_count
            if sh_count:
                raw_dt.append(("sh", f"{sh_count}f4"))
        else:
            raw_dt = [("pos", "3u2"), ("scale", "3u2"), ("rot", "4u2"), ("color", "4u1")]
            per = 24 + (2 if level == 1 else 1) * sh_count
            if sh_count:
                raw_dt.append(("sh", f"{sh_count}f2" if level == 1 else f"{sh_count}u1"))
        if off + n * per > len(buf):
            raise ValueError("section cut short")
        raw = np.frombuffer(buf, np.dtype(raw_dt), n, off)
        off += s["maxSplatCount"] * per
        part = np.zeros(n, dtype)
        if level == 0:
            pos, scales, rots = raw["pos"], raw["scale"], raw["rot"]
        else:
            if nb == 0:
                raise ValueError("no centres")
            full = s["fullBucketCount"] * s["bucketSize"]
            ends = np.cumsum(lengths, dtype=np.int64)
            if full + (int(ends[-1]) if npfb else 0) < n:
                raise ValueError("bucket lengths")
            i = np.arange(n, dtype=np.int64)
            b = np.where(i < full, i // max(s["bucketSize"], 1),
                         s["fullBucketCount"] + np.searchsorted(ends, i - full, side="right"))
            if n and b[-1] >= nb:
                raise ValueError("bucket past the centres")
            sr = s["compressionScaleRange"]
            sf = (s["bucketBlockSize"] / 2.0) / sr
            pos = (raw["pos"].astype(np.float32) - sr) * sf + centres[b]
            scales = raw["scale"].view(np.float16).astype(np.float32)
            rots = ((raw["rot"].astype(np.float32) - 32767.5) / 32767.5) * 1.41421356
        rgba = raw["color"].astype(np.float32) / 255.0
        f_dc = (rgba[:, :3] - 0.5) / 0.28209479177387814
        for k, f in enumerate("xyz"):
            part[f] = pos[:, k]
        for k in range(3):
            part[f"scale_{k}"] = scales[:, k]
            part[f"f_dc_{k}"] = f_dc[:, k]
        for k in range(4):
            part[f"rot_{k}"] = rots[:, k]
        part["opacity"] = _logit_u8(raw["color"][:, 3])
        if sh_count:
            sh = raw["sh"]
            sh = sh if level == 0 else sh.astype(np.float32) if level == 1 else (sh.astype(np.float32) - 128.0) / 128.0
            for k in range(sh_count):
                part[f"f_rest_{k}"] = sh[:, k]
        parts.append(part)
    if sum(len(p) for p in parts) >= 1 << 31:
        raise ValueError("size")
    return (np.concatenate(parts) if parts else np.zeros(0, dtype)), meta


def spz(buf: bytes):
    if len(buf) > 2 and buf[0] == 0x1F and buf[1] == 0x8B:
        buf = gzip.decompress(buf)
    if len(buf) < 16:
        raise ValueError("header")
    magic, version, N, deg, fb, _, _ = struct.unpack_from("<IIIBBBB", buf, 0)
    if magic != 0x5053474E or not 1 <= version <= 3 or fb > 127:
        raise ValueError("header")
    dim = {0: 0, 1: 3, 2: 8, 3: 15}.get(deg, 0)
    raw = buf[16:]
    if len(raw) < N * ((6 if version == 1 else 9) + 7 + (4 if version >= 3 else 3) + 3 * dim):
        raise ValueError("body cut short")
    out = np.zeros(N, gaussian_dtype(has_rgb=True, sh_degree=deg))
    ptr = 0
    if version == 1:
        p = np.frombuffer(raw, np.float16, N * 3, ptr).reshape(N, 3).astype(np.float32)
        ptr += N * 6
    else:
        b = np.frombuffer(raw, np.uint8, N * 9, ptr).reshape(N, 3, 3).astype(np.int32)
        ptr += N * 9
        i32 = b[:, :, 0] | (b[:, :, 1] << 8) | (b[:, :, 2] << 16)
        i32[(i32 & 0x800000) != 0] |= -16777216
        p = i32.astype(np.float32) / (1 << fb)
    out["x"], out["y"], out["z"] = p[:, 0], p[:, 1], p[:, 2]
    out["opacity"] = _logit_u8(np.frombuffer(raw, np.uint8, N, ptr))
    ptr += N
    col = np.frombuffer(raw, np.uint8, N * 3, ptr).reshape(N, 3)
    ptr += N * 3
    for k, c in enumerate(("red", "green", "blue")):
        dc = (col[:, k].astype(np.float32) / 255.0 - 0.5) / 0.15
        out[f"f_dc_{k}"] = dc
        out[c] = np.clip((0.5 + SH_C0 * dc) * 255.0, 0, 255).astype(np.uint8)
    sc = np.frombuffer(raw, np.uint8, N * 3, ptr).reshape(N, 3)
    ptr += N * 3
    for k in range(3):
        out[f"scale_{k}"] = sc[:, k] / 16.0 - 10.0
    if version >= 3:
        packed = np.frombuffer(raw, np.uint32, N, ptr)
        ptr += N * 4
        idx = (packed >> 30) & 0x3

        def unq(c):
            return ((c & 0x1FF).astype(np.float32) / 511.0) * 0.707106781186547524401 * (1.0 - 2.0 * ((c >> 9) & 0x1))

        v = [unq((packed >> 20) & 0x3FF), unq((packed >> 10) & 0x3FF), unq(packed & 0x3FF)]
        m = np.sqrt(np.maximum(0.0, 1.0 - (v[0] ** 2 + v[1] ** 2 + v[2] ** 2)))
        comps = [np.zeros(N, "f4") for _ in range(4)]   # x, y, z, w
        for i in range(4):
            sel = idx == i
            others = [j for j in range(4) if j != i]
            comps[i][sel] = m[sel]
            for k in range(3):
                comps[others[k]][sel] = v[k][sel]
        out["rot_0"], out["rot_1"], out["rot_2"], out["rot_3"] = comps[3], comps[0], comps[1], comps[2]
    else:
        xyz = np.frombuffer(raw, np.uint8, N * 3, ptr).reshape(N, 3).astype(np.float32) / 127.5 - 1.0
        ptr += N * 3
        out["rot_0"] = np.sqrt(np.maximum(0.0, 1.0 - np.sum(xyz ** 2, axis=1)))
        out["rot_1"], out["rot_2"], out["rot_3"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    if dim:
        sh = (np.frombuffer(raw, np.uint8, N * dim * 3, ptr).reshape(N, dim, 3).astype(np.float32) - 128.0) / 128.0
        for j in range(dim):
            for c in range(3):
                out[f"f_rest_{j + c * dim}"] = sh[:, j, c]
    return out, None


def compressed_ply(buf: bytes):
    els, end = parse_ply_header(buf)
    if "chunk" not in els or "vertex" not in els or end > len(buf):
        raise ValueError("elements")
    ch, vx, sh = els["chunk"], els["vertex"], els.get("sh")
    for el, names, t in ((ch, CHUNK_DTYPE.names, "<f4"), (vx, VERTEX_DTYPE.names, "<u4")):
        if any(f not in (el.dtype.names or ()) or el.dtype.fields[f][0] != np.dtype(t) for f in names):
            raise ValueError("fields")
    names = list(sh.dtype.names or ()) if sh is not None else []
    if any(sh.dtype.fields[f][0] != np.dtype("u1") for f in names) or (sh is not None and sh.count < vx.count) \
            or len(names) > 64 or set(names) & set(FIXED_FIELDS):
        raise ValueError("sh")
    chunks = np.frombuffer(buf, ch.dtype, ch.count, ch.offset)
    vertices = np.frombuffer(buf, vx.dtype, vx.count, vx.offset)
    sh_data = np.frombuffer(buf, sh.dtype, sh.count, sh.offset) if names else None
    n = len(vertices)
    degree = 3 if len(names) >= 45 else 2 if len(names) >= 24 else 1 if len(names) >= 9 else 0
    meta = {"count": n, "sh_degree": degree, "chunks": len(chunks)}
    data = np.zeros(n, np.dtype([(f, "f4") for f in FIXED_FIELDS + tuple(names)]))

    def denorm3(packed, mins, maxs):
        out = []
        for nv, lo, hi, t in (((packed >> 21) & 0x7FF, mins[0], maxs[0], 2047), ((packed >> 11) & 0x3FF, mins[1], maxs[1], 1023),
                              (packed & 0x7FF, mins[2], maxs[2], 2047)):
            out.append((nv / t) * (hi - lo) + lo)
        return out

    with np.errstate(all="ignore"):
        for i in range(len(chunks)):
            start, end = i * 256, min(i * 256 + 256, n)
            if start >= n:
                break
            c, v = chunks[i], vertices[start:end]
            for f, val in zip("xyz", denorm3(v["packed_position"], [c["min_x"], c["min_y"], c["min_z"]],
                                             [c["max_x"], c["max_y"], c["max_z"]])):
                data[f][start:end] = val
            pr = v["packed_rotation"]
            largest = pr >> 30
            dv = [(((pr >> s) & 0x3FF) / 1023.0 - 0.5) / 0.7071067811865476 for s in (20, 10, 0)]
            missing = np.sqrt(np.clip(1.0 - (dv[0] ** 2 + dv[1] ** 2 + dv[2] ** 2), 0, 1))
            q = np.zeros((len(pr), 4), np.float32)
            for j in range(4):
                m = largest == j
                others = [k for k in range(4) if k != j]
                q[m, j] = missing[m]
                for k in range(3):
                    q[m, others[k]] = dv[k][m]
            for k in range(4):
                data[f"rot_{k}"][start:end] = q[:, k]
            for k, val in enumerate(denorm3(v["packed_scale"], [c["min_scale_x"], c["min_scale_y"], c["min_scale_z"]],
                                            [c["max_scale_x"], c["max_scale_y"], c["max_scale_z"]])):
                data[f"scale_{k}"][start:end] = val
            pc = v["packed_color"]
            for k, (s, lo, hi) in enumerate(((24, "min_r", "max_r"), (16, "min_g", "max_g"), (8, "min_b", "max_b"))):
                col = (((pc >> s) & 0xFF) / 255.0) * (c[hi] - c[lo]) + c[lo]
                data[f"f_dc_{k}"][start:end] = (col - 0.5) / SH_C0
            a = np.clip((pc & 0xFF) / 255.0, 1e-6, 1.0 - 1e-6)
            data["opacity"][start:end] = np.log(a / (1.0 - a))
            for f in names:
                data[f][start:end] = (sh_data[start:end][f] / 256.0 - 0.5) * 8.0
    return data, meta


READERS = {"splat": splat, "ksplat": ksplat, "spz": spz, "cply": compressed_ply}

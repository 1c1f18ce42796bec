"""NumPy restatement of the SOG reader (SogFormat.read, formats/sog.py:23-247 of 3dgsconverter) working from the
bundle's bytes, with the palette double loop (sog.py:190-202) vectorised; the reader's centroid indexing is kept.

    read(blob)      -> the reference's array, or the exception the reference raises
    decode(blob)    -> read(blob), with every exception and every bundle gsx refuses (shN.bands outside 0 .. 3, a
                       count or bands that is not an int) as ValueError: the device reader's contract
    from_pixels(pixels, meta) -> the array from already-decoded RGBA pixels (member name -> flat uint8)
"""
from __future__ import annotations

import hashlib
import io
import json
import zipfile

import numpy as np

COEFFS = (0, 9, 24, 45)


def gaussian_dtype(sh_degree):
    n_rest = 3 * ((sh_degree + 1) ** 2 - 1)
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", *[f"f_rest_{i}" for i in range(n_rest)],
             "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    return np.dtype([(n, "<f4") for n in names])


def webp_pixels(zf, name):
    """(flat uint8 RGBA, pixel count) of a member, as read_webp_to_flat decodes it."""
    from PIL import Image
    with zf.open(name) as f:
        img = Image.open(f)
        w, h = img.size
        if img.mode != "RGBA":
            img = img.convert("RGBA")
        return np.array(img).flatten(), w * h


def from_pixels(get, meta):
    """SogFormat.read after the ZIP step; get(name, expected_count) -> the flat pixels read_webp_to_flat returns."""
    count = meta["count"]
    means_l = get(meta["means"]["files"][0], count).reshape(-1, 4)[:count]
    means_u = get(meta["means"]["files"][1], count).reshape(-1, 4)[:count]
    mins, maxs = meta["means"]["mins"], meta["means"]["maxs"]

    def pos(ch, i):
        q = means_l[:, ch].astype(np.uint16) | (means_u[:, ch].astype(np.uint16) << 8)
        log_val = (q / 65535.0) * (maxs[i] - mins[i]) + mins[i]
        return np.sign(log_val) * (np.exp(np.abs(log_val)) - 1.0)

    x, y, z = pos(0, 0), pos(1, 1), pos(2, 2)
    scales = get(meta["scales"]["files"][0], count).reshape(-1, 4)[:count]
    scb = np.array(meta["scales"]["codebook"], dtype=np.float32)
    scale = [scb[scales[:, k]] for k in range(3)]
    quats = get(meta["quats"]["files"][0], count).reshape(-1, 4)[:count]
    q_rest = (quats[:, :3].astype(np.float32) / 255.0 - 0.5) * 2.0
    mc = quats[:, 3] - 252
    q_missing = np.sqrt(np.maximum(1.0 - np.sum(q_rest ** 2, axis=1), 0.0))
    rot = np.zeros((4, count), np.float32)
    for k in range(4):
        m = mc == k
        others = [i for i in range(4) if i != k]
        rot[k][m] = q_missing[m]
        for c, i in enumerate(others):
            rot[i][m] = q_rest[m, c]
    sh0 = get(meta["sh0"]["files"][0], count).reshape(-1, 4)[:count]
    ccb = np.array(meta["sh0"]["codebook"], dtype=np.float32)
    f_dc = [ccb[sh0[:, k]] for k in range(3)]
    alpha = np.clip(sh0[:, 3].astype(np.float32) / 255.0, 1.0 / 255.0, 0.9999)
    opacity = -np.log((1.0 / alpha) - 1.0)
    sh = {}
    if "shN" in meta:
        bands, P = meta["shN"]["bands"], meta["shN"]["count"]
        coeffs = COEFFS[bands]
        C = coeffs // 3
        w_c = 64 * coeffs
        h_c = int(np.ceil(P / 64))
        raw = get(meta["shN"]["files"][0], w_c * h_c)
        ind = np.zeros((P, 3, C), dtype=np.uint8)
        i, j = np.arange(P)[:, None], np.arange(C)[None, :]
        flat = ((i // 64) * w_c + (i % 64) * C + j) * 4
        for c in range(3):
            ind[:, c, :] = raw[flat + c]
        palette = np.array(meta["shN"]["codebook"], dtype=np.float32)[ind].reshape(P, -1)
        lab = get(meta["shN"]["files"][1], count).reshape(-1, 4)[:count]
        labels = lab[:, 0].astype(np.uint16) | (lab[:, 1].astype(np.uint16) << 8)
        values = palette[labels]
        sh = {f"f_rest_{k}": values[:, k] for k in range(coeffs)}
    deg = meta["shN"]["bands"] if "shN" in meta and "bands" in meta["shN"] else 0
    out = np.zeros(count, dtype=gaussian_dtype(deg))
    out["x"], out["y"], out["z"] = x, y, z
    for k in range(3):
        out[f"scale_{k}"] = scale[k]
        out[f"f_dc_{k}"] = f_dc[k]
    for k in range(4):
        out[f"rot_{k}"] = rot[k]
    out["opacity"] = opacity
    for k, v in sh.items():
        if k in out.dtype.names:
            out[k] = v
    return out


def read(blob: bytes) -> np.ndarray:
    bio = io.BytesIO(blob)
    if not zipfile.is_zipfile(bio):
        raise ValueError("SOG Format: Only ZIP-bundled .sog files are supported.")
    with zipfile.ZipFile(bio) as zf:
        with zf.open("meta.json") as f:
            meta = json.load(f)

        def get(name, expected):
            data, pixels = webp_pixels(zf, name)
            if pixels < expected:
                raise ValueError(f"Image {name} too small: {pixels} < {expected}")
            return data[:expected * 4]

        with np.errstate(all="ignore"):
            return from_pixels(get, meta)


def refused_meta(meta) -> str | None:
    """Why gsx refuses a meta.json the reference may accept, or None."""
    def not_int(v):
        return isinstance(v, bool) or not isinstance(v, int)
    if isinstance(meta, dict) and "count" in meta and not_int(meta["count"]):
        return "count is not an int"
    shn = meta.get("shN") if isinstance(meta, dict) else None
    if isinstance(shn, dict) and "bands" in shn and (not_int(shn["bands"]) or not 0 <= shn["bands"] <= 3):
        return "shN.bands outside 0 .. 3"
    return None


def decode(blob: bytes) -> np.ndarray:
    try:
        with zipfile.ZipFile(io.BytesIO(blob)) as zf:
            why = refused_meta(json.loads(zf.read("meta.json")))
    except Exception:  # noqa: BLE001
        why = None
    if why:
        raise ValueError(why)
    try:
        return read(blob)
    except ValueError:
        raise
    except Exception as e:  # noqa: BLE001
        raise ValueError(f"{type(e).__name__}: {e}") from None


def digest(b: bytes) -> str:
    return hashlib.sha256(b).hexdigest()


def pixels_reader(pixels: dict):
    """get() of from_pixels over decoded pixels (member name -> flat uint8 RGBA)."""
    def get(name, expected):
        data = np.asarray(pixels[name]).reshape(-1)
        if len(data) // 4 < expected:
            raise ValueError(f"Image {name} too small: {len(data) // 4} < {expected}")
        return data[:expected * 4]
    return get


def zip_bundle(members: dict, meta, raw_meta: bytes | None = None) -> bytes:
    """A ZIP_STORED bundle of encoded members (name -> bytes) and meta.json."""
    bio = io.BytesIO()
    with zipfile.ZipFile(bio, "w", zipfile.ZIP_STORED) as zf:
        for name, b in members.items():
            zf.writestr(name, b)
        if meta is not None or raw_meta is not None:
            zf.writestr("meta.json", raw_meta if raw_meta is not None else json.dumps(meta))
    return bio.getvalue()


def webp(rgba: np.ndarray, mode="RGBA") -> bytes:
    """A lossless WebP of uint8 [h, w, 4] (mode 'RGB' drops alpha), with the reference writer's arguments."""
    from PIL import Image
    a = np.ascontiguousarray(rgba, dtype=np.uint8)
    img = Image.frombytes("RGBA", (a.shape[1], a.shape[0]), a.tobytes())
    if mode != "RGBA":
        img = img.convert(mode)
    bio = io.BytesIO()
    img.save(bio, format="WEBP", lossless=True, quality=100, method=1)
    return bio.getvalue()

"""The SOG reader on the device: formats/sog.py:23-247 (SogFormat.read) from the bundle's bytes.

    dec = gsx.sog_reader.decode("in.sog")    # readers.Decoded: dec.to_host() is what SogFormat.read returns
    r = dec.records()                         # DeviceRecords (zero-copy: every field is float32)

The ZIP, meta.json and (by default) the WebP members are handled on the host: the members are decoded with Pillow exactly as
read_webp_to_flat does (Image.open, convert('RGBA') unless already RGBA), concurrently on GSX_HOST_THREADS threads, and
the pixels every step reads go to the device in one copy.  The maps of one stored value -- the three position axes
(65 536 u16 codes each, float64 exp as NumPy computes it), the quaternion component and opacity bytes -- are tables
built with the reference's own NumPy expressions.  On the device: the shN palette (gsx_sog_decode_palette) with the
reader's own centroid indexing, which differs from the writer's layout for palette entries >= 64 and is reproduced
as it is, then one row per splat (gsx_sog_decode).

decode_textures(pixels, meta) is the device stage alone, from already-decoded RGBA pixels.  decode(..., webp="device")
uploads the members' compressed bytes instead and decodes the lossless ones on the device (gsx.webp_decode).

Anything the reference rejects, or that gsx does not reproduce (negative `bands`, which the reference accepts through
Python's negative indexing), raises ValueError; the drop-in reader then runs the reference's own read.
"""
from __future__ import annotations

import ctypes as C
import io
import json
import os
import zipfile
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass

import numpy as np
import torch

from . import readers
from ._abi import lib, check
from ._abi import _ptr, _stream

COEFFS = (0, 9, 24, 45)        # sog.py:170: f_rest values per splat for 0 .. 3 bands
ROLES = ("means_l", "means_u", "quats", "scales", "sh0", "labels", "centroids")
_ERRORS = {1: "a scales index past the scales codebook", 2: "an sh0 index past the sh0 codebook",
           4: "a shN centroid index past the shN codebook", 8: "an shN label >= shN.count"}


def _int(v, what) -> int:
    if isinstance(v, bool) or not isinstance(v, int):
        raise ValueError(f"SOG meta: {what} is {v!r}, not an integer")
    return v


def _files(section, k, what):
    files = section["files"]
    if not isinstance(files, list) or len(files) < k or not all(isinstance(f, str) for f in files[:k]):
        raise ValueError(f"SOG meta: {what}.files must list {k} member names")
    return files[:k]


def _codebook(section, what) -> np.ndarray:
    try:
        cb = np.array(section["codebook"], dtype=np.float32)
    except (TypeError, ValueError, OverflowError) as e:
        raise ValueError(f"SOG meta: {what}.codebook: {e}") from None
    if cb.ndim != 1:
        raise ValueError(f"SOG meta: {what}.codebook is not a flat list")
    return cb


def position_tables(mins, maxs) -> np.ndarray:
    """float32 [3, 65536]: sog.py:78-86 for every u16 code of each axis, in float64 as the reference computes it."""
    qv = np.arange(65536, dtype=np.uint16)
    out = np.empty((3, 65536), np.float32)
    with np.errstate(all="ignore"):
        for i in range(3):
            norm = qv / 65535.0
            try:
                log_val = norm * (maxs[i] - mins[i]) + mins[i]
                v = np.sign(log_val) * (np.exp(np.abs(log_val)) - 1.0)
            except (TypeError, OverflowError) as e:
                raise ValueError(f"SOG meta: means bounds {mins[i]!r} / {maxs[i]!r}: {e}") from None
            if v.dtype != np.float64:
                raise ValueError(f"SOG meta: means bounds {mins[i]!r} / {maxs[i]!r} do not give float64 positions")
            out[i] = v
    return out


def byte_tables():
    """sog.py:108 (quaternion component of a byte) and sog.py:156-158 (opacity logit of the alpha byte), float32."""
    u = np.arange(256, dtype=np.uint8)
    q = (u.astype(np.float32) / 255.0 - 0.5) * 2.0
    a = np.clip(u.astype(np.float32) / 255.0, 1.0 / 255.0, 0.9999)
    with np.errstate(all="ignore"):
        return q, -np.log((1.0 / a) - 1.0)


@dataclass
class SogLayout:
    """What meta.json says, checked: the splat count, member names per role, codebooks and the shN palette shape."""
    count: int
    files: dict                  # role -> member name (ROLES; labels / centroids only with shN)
    mins: list
    maxs: list
    scales_codebook: np.ndarray
    sh0_codebook: np.ndarray
    bands: int | None            # None without shN
    palette_size: int = 0
    sh_codebook: np.ndarray | None = None

    @property
    def coeffs(self) -> int:
        return COEFFS[self.bands] if self.bands else 0

    def pixels_needed(self) -> dict:
        """role -> pixels read_webp_to_flat keeps (count, or w_c * h_c for the centroids)."""
        need = {r: self.count for r in ROLES[:5]}
        if self.bands is not None:
            need["labels"] = self.count
            need["centroids"] = 64 * self.coeffs * -(-self.palette_size // 64)
        return need

    def members(self) -> dict:
        """member name -> pixels needed (the largest of the roles that read it)."""
        out = {}
        for role, k in self.pixels_needed().items():
            name = self.files[role]
            out[name] = max(out.get(name, 0), k)
        return out


def parse_meta(meta) -> SogLayout:
    """The checks of sog.py:37-211 that precede any per-splat work, as ValueError."""
    try:
        count = _int(meta["count"], "count")
        if count < 0:
            raise ValueError(f"SOG meta: count {count} < 0")
        if count >= 2 ** 31:
            raise ValueError("SOG on the device supports fewer than 2^31 splats")
        files = dict(zip(("means_l", "means_u"), _files(meta["means"], 2, "means")))
        mins, maxs = meta["means"]["mins"], meta["means"]["maxs"]
        if not isinstance(mins, list) or not isinstance(maxs, list) or len(mins) < 3 or len(maxs) < 3:
            raise ValueError("SOG meta: means.mins and means.maxs need 3 values each")
        for v in mins[:3] + maxs[:3]:
            if isinstance(v, bool) or not isinstance(v, (int, float)):
                raise ValueError(f"SOG meta: means bound {v!r} is not a number")
        files["scales"], = _files(meta["scales"], 1, "scales")
        files["quats"], = _files(meta["quats"], 1, "quats")
        files["sh0"], = _files(meta["sh0"], 1, "sh0")
        layout = SogLayout(count, files, mins[:3], maxs[:3], _codebook(meta["scales"], "scales"),
                           _codebook(meta["sh0"], "sh0"), None)
        if "shN" in meta:
            shn = meta["shN"]
            bands = _int(shn["bands"], "shN.bands")
            if not 0 <= bands <= 3:
                raise ValueError(f"SOG meta: shN.bands {bands} is not 0 .. 3")
            p = _int(shn["count"], "shN.count")
            if p <= 0:
                raise ValueError(f"SOG meta: shN.count {p} <= 0 (the reference's palette reshape fails)")
            files["centroids"], files["labels"] = _files(shn, 2, "shN")
            layout.bands, layout.palette_size, layout.sh_codebook = bands, p, _codebook(shn, "shN")
            if p * layout.coeffs >= 2 ** 31:
                raise ValueError(f"SOG meta: a palette of {p} x {layout.coeffs} values is not supported")
    except (KeyError, TypeError, IndexError) as e:
        raise ValueError(f"SOG meta.json not readable as the reference reads it: {type(e).__name__}: {e}") from None
    return layout


def host_threads(jobs: int) -> int:
    """GSX_HOST_THREADS (default: 16 on hosts with >= 32 cores, else half of them), at most one per job."""
    t = int(os.environ.get("GSX_HOST_THREADS", "0") or 0)
    if t <= 0:
        hw = os.cpu_count() or 1
        t = 16 if hw >= 32 else max(1, hw // 2)
    return max(1, min(t, jobs))


def decode_members(zf: zipfile.ZipFile, members: dict, threads: int | None = None) -> np.ndarray:
    """uint8: the first `need` RGBA pixels of each member (in `members` order), concatenated; each decoded with Pillow
    as read_webp_to_flat does (sog.py:43-57), concurrently."""
    try:
        from PIL import Image
    except ImportError:
        raise ValueError("Pillow is required to read .sog files") from None
    names = list(members)
    blobs = {}
    for name in names:
        try:
            blobs[name] = zf.read(name)
        except KeyError:
            raise ValueError(f"SOG: member {name!r} named in meta.json is missing") from None
        except (zipfile.BadZipFile, OSError, NotImplementedError, RuntimeError) as e:
            raise ValueError(f"SOG: member {name!r}: {e}") from None
    offs = np.concatenate([[0], np.cumsum([4 * members[n] for n in names])]).astype(np.int64)
    out = np.empty(int(offs[-1]), np.uint8)

    def one(k):
        name, need = names[k], members[names[k]]
        try:
            img = Image.open(io.BytesIO(blobs[name]))
            width, height = img.size
            if img.mode != "RGBA":
                img = img.convert("RGBA")
            data = np.asarray(img).reshape(-1)
        except Exception as e:  # noqa: BLE001  (Pillow's own errors for a member that is not an image)
            raise ValueError(f"SOG: member {name!r} does not decode: {type(e).__name__}: {e}") from None
        if width * height < need:
            raise ValueError(f"Image {name} too small: {width * height} < {need}")
        out[offs[k]:offs[k + 1]] = data[:4 * need]

    n = host_threads(len(names)) if threads is None else threads
    if n <= 1:
        for k in range(len(names)):
            one(k)
    else:
        with ThreadPoolExecutor(n) as pool:
            for f in [pool.submit(one, k) for k in range(len(names))]:
                f.result()
    return out


def open_bundle(data):
    """(ZipFile, meta) of a .sog bundle given as bytes or a path."""
    bio = io.BytesIO(readers.file_bytes(data))
    if not zipfile.is_zipfile(bio):
        raise ValueError("SOG Format: Only ZIP-bundled .sog files are supported.")
    try:
        zf = zipfile.ZipFile(bio)
        meta = json.loads(zf.read("meta.json"))
    except KeyError:
        raise ValueError("SOG: no meta.json in the bundle") from None
    except (zipfile.BadZipFile, OSError, ValueError, NotImplementedError, RuntimeError) as e:
        raise ValueError(f"SOG: bundle not readable: {type(e).__name__}: {e}") from None
    return zf, meta


def decode_members_device(zf: zipfile.ZipFile, members: dict, device, threads: int | None = None) -> dict:
    """member name -> uint8 CUDA tensor of its first `need` RGBA pixels.  Lossless members whose main image has one
    prefix-code group and no colour cache (every member gsx.webp writes) are decoded on the device by gsx.webp_decode,
    so only their compressed bytes are uploaded; the others (libwebp's multi-group or cached streams, lossy WebP,
    ALPH, animation) are decoded with Pillow, concurrently, as decode_members does."""
    from .webp_decode import container, decode_lossless
    out, blobs, host = {}, {}, {}
    for name, need in members.items():
        try:
            blobs[name] = blob = zf.read(name)
        except KeyError:
            raise ValueError(f"SOG: member {name!r} named in meta.json is missing") from None
        except (zipfile.BadZipFile, OSError, NotImplementedError, RuntimeError) as e:
            raise ValueError(f"SOG: member {name!r}: {e}") from None
        px = None
        if container(blob) is not None:
            try:
                px = decode_lossless(blob, device, parallel_only=True)
            except ValueError as e:
                raise ValueError(f"SOG: member {name!r} does not decode: {e}") from None
        if px is None:
            host[name] = need
            continue
        px = px.reshape(-1)
        if px.numel() < 4 * need:
            raise ValueError(f"Image {name} too small: {px.numel() // 4} < {need}")
        out[name] = px[:4 * need]
    if host:
        from .hostcopy import to_device
        flat = to_device(decode_members(_Members(blobs), host, threads), device)
        off = 0
        for name, need in host.items():
            out[name] = flat[off:off + 4 * need]
            off += 4 * need
    return out


class _Members:
    """The read() of a ZipFile whose members are already read, for decode_members."""

    def __init__(self, blobs):
        self.blobs = blobs

    def read(self, name):
        return self.blobs[name]


def decode(data, device="cuda", threads: int | None = None, webp: str = "host") -> readers.Decoded:
    """SogFormat.read on the device: `data` is the bundle's bytes or a path.  threads: Pillow decode threads
    (default GSX_HOST_THREADS).  webp: "host" decodes the WebP members with Pillow and uploads their pixels;
    "device" decodes the single-group, cache-free lossless members on the device from their uploaded bytes and the
    rest with Pillow (decode_members_device)."""
    if webp not in ("host", "device"):
        raise ValueError(f"webp must be 'host' or 'device', not {webp!r}")
    zf, meta = open_bundle(data)
    layout = parse_meta(meta)
    members = layout.members()
    if webp == "device":
        with zf:
            pixels = decode_members_device(zf, members, device, threads)
        return decode_textures(pixels, layout)
    with zf:
        flat = decode_members(zf, members, threads)
    from .hostcopy import to_device
    dev = to_device(flat, device)
    pixels, off = {}, 0
    for name, need in members.items():
        pixels[name] = dev[off:off + 4 * need]
        off += 4 * need
    return decode_textures(pixels, layout)


def decode_textures(pixels: dict, meta) -> readers.Decoded:
    """The device stage of SogFormat.read: `pixels` maps each member name of `meta` (a meta.json dict or a SogLayout)
    to its decoded RGBA pixels as a uint8 CUDA tensor (flat or [pixels, 4]; at least the pixels the reader keeps)."""
    layout = meta if isinstance(meta, SogLayout) else parse_meta(meta)
    members = layout.members()
    flat = {}
    for name, need in members.items():
        if name not in pixels:
            raise ValueError(f"SOG: no pixels for member {name!r}")
        t = pixels[name]
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8:
            raise ValueError(f"SOG: pixels of {name!r} must be a uint8 CUDA tensor")
        t = t.reshape(-1)
        if t.numel() < 4 * need:
            raise ValueError(f"Image {name} too small: {t.numel() // 4} < {need}")
        if t.data_ptr() % 4:
            t = t.clone()
        flat[name] = t
    dev = next(iter(flat.values())).device
    n, coeffs, bands = layout.count, layout.coeffs, layout.bands
    dtype = readers.gaussian_dtype(sh_degree=bands or 0)

    def pad(cb):
        out = np.zeros(256, np.float32)
        out[:min(len(cb), 256)] = cb[:256]
        return out

    q, op = byte_tables()
    tabs = np.concatenate([position_tables(layout.mins, layout.maxs).reshape(-1), q, op,
                           pad(layout.scales_codebook), pad(layout.sh0_codebook),
                           pad(layout.sh_codebook if bands is not None else np.zeros(0, np.float32))])
    from .hostcopy import to_device, to_host
    tabs = to_device(tabs, dev)
    pos, small, shcb = tabs[:3 * 65536], tabs[3 * 65536:3 * 65536 + 1024], tabs[3 * 65536 + 1024:]
    rows = torch.empty((n, dtype.itemsize), dtype=torch.uint8, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    P = layout.palette_size
    palette = torch.empty((P, coeffs), dtype=torch.float32, device=dev) if bands is not None else None
    with torch.cuda.device(dev):
        if bands is not None:
            check(lib.gsx_sog_decode_palette(_ptr(flat[layout.files["centroids"]]), P, coeffs, _ptr(shcb),
                                             min(len(layout.sh_codebook), 256), _ptr(palette), _ptr(err), _stream()),
                  "gsx_sog_decode_palette")
        tex = (C.c_void_p * 6)(*[flat[layout.files[r]].data_ptr() if r in layout.files else 0 for r in ROLES[:6]])
        check(lib.gsx_sog_decode(tex, n, _ptr(pos), _ptr(small), min(len(layout.scales_codebook), 256),
                                 min(len(layout.sh0_codebook), 256), _ptr(palette), P, coeffs, _ptr(rows), _ptr(err),
                                 _stream()), "gsx_sog_decode")
    bits = int(to_host(err)[0])
    if bits:
        raise ValueError("SOG: the reference raises IndexError here: " +
                         ", ".join(msg for b, msg in _ERRORS.items() if bits & b))
    return readers.Decoded(rows, dtype, None)

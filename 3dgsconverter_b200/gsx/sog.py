"""Device helpers for the SOG writer steps either side of K-Means (formats/sog.py:262-552, SURVEY §8(f) item 1).

    lexsort_zyx(xyz)                     == np.lexsort((z, y, x))                       sog.py:264
    quantize_to_codebook(vals, codebook) == the writer's sorted-codebook nearest lookup  sog.py:408-419
    codebook_1d(values, k, max_iter)     == gpu_ops.kmeans(values.reshape(-1,1), k, max_iter) + sorted(c.flatten())
                                            (sog.py:402-403, 443-444) on the 1-D Lloyd kernel

and the whole writer, SogFormat.write (sog.py:249-639), over device-resident records:

    tex = encode(records, compression_level=0)  # DeviceRecords -> SogTextures (device uint8 [pixels, 4] textures)
    write_sog("out.sog", tex.to_host(), tex.meta)   # members by Pillow (libwebp's bytes)
    write_sog("out.sog", tex, tex.meta)              # members by gsx.webp from HBM

encode() runs the lexsort, the position / quaternion / scale / colour textures, the two 1-D codebook fits and the
chunked SH palette on the GPU.  What stays on the host: the reference's NumPy RNG draws (consumed from the global RNG
in the reference's order, so np.random.seed reproduces a run), the fit of the 256-entry SH codebook on the palette
(scikit-learn's MiniBatchKMeans by default, at most 65 536 x 45 values), and ZIP in write_sog, with
the WebP members by Pillow or, given the SogTextures themselves, by gsx.webp on the device.

Parity with the reference writer: every texture byte and meta.json entry is exact.  The position logarithm and the
opacity exponential are NumPy's SIMD float32 log and exp, restated exactly on the device.  The one exception is the
sign of a zero meta.means min or max: NumPy's depends on where the zeros sit in the array, the value does not.
"""
from __future__ import annotations

import ctypes as C
import io
import json
import sys
import time
import zipfile
from contextlib import contextmanager
from dataclasses import dataclass

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream
from .sor import _check_xyz


def lexsort_zyx(xyz: torch.Tensor) -> torch.Tensor:
    """int32 [N]: indices that order the splats by x, then y, then z (stable), like np.lexsort((z, y, x))."""
    _check_xyz(xyz)
    n = xyz.shape[0]
    order = torch.empty(n, dtype=torch.int32, device=xyz.device)
    ws = torch.empty(lib.gsx_lexsort_workspace_bytes(n), dtype=torch.uint8, device=xyz.device)
    check(lib.gsx_lexsort_zyx(_ptr(xyz), n, _ptr(order), _ptr(ws), ws.numel(), _stream()), "gsx_lexsort_zyx")
    return order


def quantize_to_codebook(vals: torch.Tensor, codebook) -> torch.Tensor:
    """uint8 [N]: nearest entry of the ascending float32 codebook (reference semantics incl. the left-neighbour rule)."""
    if not vals.is_cuda or vals.dtype != torch.float32 or not vals.is_contiguous():
        raise ValueError("vals must be a contiguous float32 CUDA tensor")
    cb = np.ascontiguousarray(codebook, dtype=np.float32)
    n = vals.numel()
    out = torch.empty(n, dtype=torch.uint8, device=vals.device)
    ws = torch.empty(max(4 * len(cb), 256), dtype=torch.uint8, device=vals.device)
    check(lib.gsx_quantize_to_codebook(_ptr(vals), n, cb.ctypes.data_as(C.POINTER(C.c_float)), len(cb), _ptr(out),
                                       _ptr(ws), ws.numel(), _stream()), "gsx_quantize_to_codebook")
    return out


def codebook_1d(values: np.ndarray, k: int = 256, max_iter: int = 20) -> np.ndarray:
    """The scalar codebook of sog.py:392-403 / 435-444: subsample <= 50 000 values with the reference's
    np.random.choice draw, Lloyd K-Means (D=1) on the GPU, return the sorted centroids (float32[k])."""
    from gsconverter.processing import gpu_ops
    fit = values
    if len(values) > 50000:
        fit = values[np.random.choice(len(values), 50000, replace=False)]
    c, _ = gpu_ops.kmeans(fit.reshape(-1, 1), k, max_iter=max_iter)
    return np.array(sorted(c.flatten()), dtype=np.float32)


# ------------------------------------------------------------------------------------------------------------------
# SogFormat.write on the device

SOG_FIELDS = ("x", "y", "z", "rot_0", "rot_1", "rot_2", "rot_3", "scale_0", "scale_1", "scale_2",
              "f_dc_0", "f_dc_1", "f_dc_2", "opacity")
MAIN_FILES = ("means_l.webp", "means_u.webp", "quats.webp", "scales.webp", "sh0.webp")
SHN_FILES = ("shN_centroids.webp", "shN_labels.webp")
FIT_SAMPLE = 50000        # sog.py:398, 439: the 1-D codebooks are fitted on at most this many values
CODEBOOK_K = 256
_MINMAX_WS = 1024 * 6 * 4


def texture_size(n: int) -> tuple:
    """(width, height) of the per-splat textures (sog.py:259-260)."""
    width = int(np.ceil(np.sqrt(n) / 4) * 4)
    height = int(np.ceil(n / width / 4) * 4)
    return width, height


def _bands(last_nonzero: int) -> int:
    return 3 if last_nonzero >= 24 else 2 if last_nonzero >= 9 else 1 if last_nonzero >= 0 else 0


def declared_bands(names) -> int:
    """sog.py:466-475: SH bands by how many f_rest_i fields the records have (before the content check)."""
    if "f_rest_0" not in names:
        return 0
    count = sum(f"f_rest_{i}" in names for i in range(45))
    return 3 if count >= 45 else 2 if count >= 24 else 1 if count >= 9 else 0


def chunk_schedule(n: int, compression_level=0) -> tuple:
    """sog.py:507-542: (chunk_size, [(start, end, this_k)]) of the shN palette, including N < 1024, where log2 goes
    negative and official_standard_k is a float."""
    try:
        comp_level = int(compression_level)
    except Exception:  # noqa: BLE001  (sog.py:509)
        comp_level = 0
    official_standard_k = min(64, 2 ** int(np.floor(np.log2(n / 1024)))) * 1024
    if comp_level <= 3:
        target_k = min(65536, official_standard_k)
    elif comp_level <= 6:
        target_k = min(16384, official_standard_k)
    else:
        target_k = min(4096, official_standard_k)
    target_k = max(256, target_k)
    num_chunks = max(1, min(64, n // 1024))
    chunk_size = int(np.ceil(n / num_chunks))
    k_per_chunk = max(16, int(np.ceil(target_k / num_chunks)))
    plan = []
    for i in range(num_chunks):
        start, end = i * chunk_size, min((i + 1) * chunk_size, n)
        if start >= end:
            break
        plan.append((start, end, min(end - start, k_per_chunk)))
    return chunk_size, plan


def default_codebook_fit(values: np.ndarray) -> np.ndarray:
    """sog.py:561: MiniBatchKMeans(n_clusters=256, n_init='auto') on the flattened palette (global NumPy RNG)."""
    from sklearn.cluster import MiniBatchKMeans
    return MiniBatchKMeans(n_clusters=CODEBOOK_K, n_init="auto").fit(values).cluster_centers_


@dataclass
class SogTextures:
    textures: dict                  # file name -> device uint8 [pixels, 4]
    sizes: dict                     # file name -> (width, height)
    meta: dict                      # the meta.json of sog.py:612-635
    order: torch.Tensor             # int32 [N]: record index of the j-th splat of the file

    def to_host(self) -> dict:
        """file name -> uint8 [height, width, 4], the RGBA image write_sog stores."""
        from .hostcopy import to_host
        return {name: to_host(t).reshape(self.sizes[name][1], self.sizes[name][0], 4)
                for name, t in self.textures.items()}


class _Stages:
    """Optional stage timing for encode(profile=dict): CUDA events around device stages, wall time around host
    stages; results in milliseconds, summed per stage name."""

    def __init__(self, out):
        self.out, self.events = out, []

    @contextmanager
    def device(self, name):
        if self.out is None:
            yield
            return
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        yield
        b.record()
        self.events.append((name, a, b))

    @contextmanager
    def host(self, name):
        if self.out is None:
            yield
            return
        t0 = time.perf_counter()
        yield
        self.out[name] = self.out.get(name, 0.0) + (time.perf_counter() - t0) * 1e3

    def finish(self):
        if self.out is None:
            return
        torch.cuda.synchronize()
        for name, a, b in self.events:
            self.out[name] = self.out.get(name, 0.0) + a.elapsed_time(b)


def _i32s(vals):
    return (C.c_int32 * max(len(vals), 1))(*vals)


def _check_records(records):
    rows = records.rows
    if not rows.is_cuda or rows.dtype != torch.float32 or rows.dim() != 2 or not rows.is_contiguous():
        raise ValueError("SOG on the device needs packed float32 records (a contiguous float32 CUDA matrix)")
    missing = [f for f in SOG_FIELDS if f not in records.col]
    if missing:
        raise ValueError(f"SOG needs the fields {missing}")
    if len(records) == 0:
        raise ValueError("SOG of no splats: the reference writer divides by zero")
    if len(records) >= 2 ** 31:
        raise ValueError("SOG on the device supports fewer than 2^31 splats")


def _gather_values(records, order, cols, sel, m):
    out = torch.empty(m, dtype=torch.float32, device=records.rows.device)
    sel_t = None if sel is None else torch.from_numpy(np.ascontiguousarray(sel, dtype=np.int64)).to(out.device)
    check(lib.gsx_sog_gather_values(_ptr(records.rows), len(records), records.F, _ptr(order), _i32s(cols), len(cols),
                                    _ptr(sel_t), m, _ptr(out), _stream()), "gsx_sog_gather_values")
    return out


def _codebook(records, order, fields, stages):
    """sog.py:392-403 / 435-444: the sorted 1-D codebook of np.concatenate(fields) in file order: the host draws of
    the subsample and the K-Means init, the fit data gathered on the device, 20 Lloyd iterations (D = 1, K = 256) or
    the passthrough of gpu_ops.kmeans when K >= len(fit)."""
    from .kmeans import kmeans_lloyd
    cols = [records.col[f] for f in fields]
    total = len(fields) * len(records)
    sel = None
    with stages.host("rng"):
        if total > FIT_SAMPLE:
            sel = np.random.choice(total, FIT_SAMPLE, replace=False)
    m = FIT_SAMPLE if sel is not None else total
    with stages.device("codebook_fits"):
        fit = _gather_values(records, order, cols, sel, m)
    if CODEBOOK_K >= m:
        c = fit
    else:
        with stages.host("rng"):
            init = np.random.choice(m, CODEBOOK_K, replace=False)
        with stages.device("codebook_fits"):
            init_rows = _gather_values(records, order, cols, init if sel is None else sel[init], CODEBOOK_K)
            c, _, _ = kmeans_lloyd(fit.view(m, 1), CODEBOOK_K, 20, init_rows.view(CODEBOOK_K, 1))
    from .hostcopy import to_host
    return sorted(to_host(c).reshape(-1))


def _sh_block(records, order, stages):
    """sog.py:463-503: (bands, float32 [N, coeffs] f_rest block in file order or None).  The band downgrade uses the
    per-column non-zero mask that gsx_sog_sh_gather collects while it gathers the declared columns."""
    from .hostcopy import to_host
    declared = declared_bands(records.col)
    if declared == 0:
        return 0, None
    n, dev = len(records), records.rows.device
    scan = [i for i in range({3: 44, 2: 23, 1: 8}[declared] + 1) if f"f_rest_{i}" in records.col]
    nonzero = torch.empty(1, dtype=torch.int64, device=dev)

    def gather(idx):
        out = torch.empty((n, len(idx)), dtype=torch.float32, device=dev)
        with stages.device("sh_gather"):
            check(lib.gsx_sog_sh_gather(_ptr(records.rows), n, records.F, _ptr(order),
                                        _i32s([records.col[f"f_rest_{i}"] for i in idx]), len(idx), _ptr(out),
                                        _ptr(nonzero), _stream()), "gsx_sog_sh_gather")
        return out

    block = gather(scan)
    mask = int(to_host(nonzero).view(np.uint64)[0])
    bands = _bands(max((i for k, i in enumerate(scan) if mask >> k & 1), default=-1))
    if bands == 0:
        return 0, None
    need = list(range([0, 9, 24, 45][bands]))
    missing = [f"f_rest_{i}" for i in need if f"f_rest_{i}" not in records.col]
    if missing:
        raise ValueError(f"SOG with {bands} SH bands needs the fields {missing}")
    return bands, (block if need == scan else gather(need))


def _palette(sh, chunk_size, plan, stages):
    """sog.py:527-553 over the device SH block: one kmeans_lloyd_batched launch per run of consecutive chunks with
    the same K (as gpu_ops._run_batch groups them); a chunk with this_k >= len is a passthrough (its rows are its
    centroids, labels arange, no draw).  The init draws are made on the host first, in chunk order.
    Returns (palette float32 [P, coeffs], chunk-local labels int32 [N], offsets, passthrough flags)."""
    from .kmeans import kmeans_lloyd_batched
    n, coeffs = sh.shape
    inits = []
    with stages.host("rng"):
        for s, e, k in plan:
            inits.append(None if k >= e - s else np.random.choice(e - s, k, replace=False))
    labels = torch.empty(n, dtype=torch.int32, device=sh.device)
    parts = [None] * len(plan)
    runs = []
    for i, (s, e, k) in enumerate(plan):
        if inits[i] is None:
            parts[i] = sh[s:e]
        elif runs and runs[-1][-1] == i - 1 and plan[runs[-1][-1]][2] == k:
            runs[-1].append(i)
        else:
            runs.append([i])
    with stages.device("chunk_kmeans"):
        for run in runs:
            k = plan[run[0]][2]
            s0, e1 = plan[run[0]][0], plan[run[-1]][1]
            offs = [plan[i][0] - s0 for i in run] + [e1 - s0]
            idx = np.concatenate([plan[i][0] + inits[i] for i in run]).astype(np.int32)
            idx_t = torch.from_numpy(idx).to(sh.device)
            init = torch.empty((len(idx), coeffs), dtype=torch.float32, device=sh.device)
            check(lib.gsx_records_gather_rows(_ptr(sh), _ptr(idx_t), len(idx), coeffs, _ptr(init), _stream()),
                  "gsx_records_gather_rows")
            Cc, L, _ = kmeans_lloyd_batched(sh[s0:e1], offs, k, 10, init)
            labels[s0:e1].copy_(L)
            for j, i in enumerate(run):
                parts[i] = Cc[j]
        palette = torch.cat(parts).contiguous()
    ks = [k for _, _, k in plan]
    offsets = [int(v) for v in np.concatenate([[0], np.cumsum(ks)[:-1]])]
    return palette, labels, offsets, [int(x is None) for x in inits]


def encode(records, compression_level=0, codebook_fit=None, profile: dict | None = None) -> SogTextures:
    """SogFormat.write (formats/sog.py:249-639) over `records` (DeviceRecords), up to the WebP / ZIP step.
    Consumes the global NumPy RNG in the reference's order: the scale subsample and init, the colour subsample and
    init, one init per non-passthrough SH chunk in chunk order, then the codebook fit.
    codebook_fit(values float32 [P * coeffs, 1]) -> centres: the fit of the SH codebook (default_codebook_fit).
    profile: if a dict, filled with per-stage times in ms (device stages by CUDA events, host stages by wall time).
    Raises ValueError, before any RNG draw, for no splats, missing fields and records that are not packed float32."""
    _check_records(records)
    stages = _Stages(profile)
    fit = codebook_fit or default_codebook_fit
    n, F, dev = len(records), records.F, records.rows.device
    col = records.col
    width, height = texture_size(n)
    pixels = width * height
    rows = _ptr(records.rows)

    def tex(count=pixels):
        return torch.empty((count, 4), dtype=torch.uint8, device=dev)

    with stages.device("lexsort"):
        order = lexsort_zyx(records.xyz_opacity()[0])
    o = _ptr(order)
    out = {name: tex() for name in MAIN_FILES}
    xyz_cols = _i32s([col["x"], col["y"], col["z"]])
    minmax = torch.empty(6, dtype=torch.float32, device=dev)
    with stages.device("positions"):
        ws = torch.empty(_MINMAX_WS, dtype=torch.uint8, device=dev)
        check(lib.gsx_sog_means_minmax(rows, n, F, xyz_cols, _ptr(ws), ws.numel(), _ptr(minmax), _stream()),
              "gsx_sog_means_minmax")
        check(lib.gsx_sog_means(rows, n, F, o, xyz_cols, _ptr(minmax), pixels, _ptr(out["means_l.webp"]),
                                _ptr(out["means_u.webp"]), _stream()), "gsx_sog_means")
    with stages.device("quats"):
        check(lib.gsx_sog_quats(rows, n, F, o, _i32s([col[f"rot_{i}"] for i in range(4)]), pixels,
                                _ptr(out["quats.webp"]), _stream()), "gsx_sog_quats")
    # the SH block (and the band decision, which may refuse) comes before the first RNG draw
    bands, sh = _sh_block(records, order, stages)

    scale_codebook = _codebook(records, order, ("scale_0", "scale_1", "scale_2"), stages)
    color_codebook = _codebook(records, order, ("f_dc_0", "f_dc_1", "f_dc_2"), stages)
    with stages.device("sh0_scales"):
        scb = torch.from_numpy(np.array(scale_codebook, dtype=np.float32)).to(dev)
        ccb = torch.from_numpy(np.array(color_codebook, dtype=np.float32)).to(dev)
        c7 = _i32s([col[f] for f in ("scale_0", "scale_1", "scale_2", "f_dc_0", "f_dc_1", "f_dc_2", "opacity")])
        check(lib.gsx_sog_scales_sh0(rows, n, F, o, c7, _ptr(scb), len(scale_codebook), _ptr(ccb),
                                     len(color_codebook), pixels, _ptr(out["scales.webp"]), _ptr(out["sh0.webp"]),
                                     _stream()), "gsx_sog_scales_sh0")
    sizes = {name: (width, height) for name in MAIN_FILES}

    shn_meta = None
    if bands:
        coeffs = sh.shape[1]
        chunk_size, plan = chunk_schedule(n, compression_level)
        palette, labels, offsets, passthrough = _palette(sh, chunk_size, plan, stages)
        P = palette.shape[0]
        from .hostcopy import to_host
        with stages.device("palette_textures"):
            out["shN_labels.webp"] = tex()
            check(lib.gsx_sog_labels(_ptr(labels), n, chunk_size, len(plan), _i32s(offsets), _i32s(passthrough),
                                     pixels, _ptr(out["shN_labels.webp"]), _stream()), "gsx_sog_labels")
            pal_host = to_host(palette)
        with stages.host("codebook_fit"):
            codebook = sorted(np.asarray(fit(pal_host.reshape(-1, 1))).flatten())
        w_c, h_c = 64 * coeffs, int(np.ceil(P / 64))
        with stages.device("palette_textures"):
            cb = torch.from_numpy(np.array(codebook, dtype=np.float32)).to(dev)
            out["shN_centroids.webp"] = tex(w_c * h_c)
            check(lib.gsx_sog_centroids(_ptr(palette), P, coeffs, _ptr(cb), len(codebook), w_c * h_c,
                                        _ptr(out["shN_centroids.webp"]), _stream()), "gsx_sog_centroids")
        sizes["shN_centroids.webp"], sizes["shN_labels.webp"] = (w_c, h_c), (width, height)
        shn_meta = {"count": int(P), "bands": int(bands), "codebook": [float(c) for c in codebook],
                    "files": list(SHN_FILES)}

    from .hostcopy import to_host
    mm = to_host(minmax)
    meta = {
        "version": 2,
        "asset": {"generator": "gsconverter-sog"},
        "count": n,
        "means": {"mins": [float(m) for m in mm[:3]], "maxs": [float(m) for m in mm[3:]],
                  "files": ["means_l.webp", "means_u.webp"]},
        "scales": {"codebook": [float(c) for c in scale_codebook], "files": ["scales.webp"]},
        "quats": {"files": ["quats.webp"]},
        "sh0": {"codebook": [float(c) for c in color_codebook], "files": ["sh0.webp"]},
    }
    if shn_meta:
        meta["shN"] = shn_meta
    stages.finish()
    textures = {name: out[name] for name in MAIN_FILES + (SHN_FILES if bands else ())}
    return SogTextures(textures, {k: sizes[k] for k in textures}, meta, order)


def write_sog(path, textures, meta: dict) -> None:
    """The .sog bundle of sog.py:268-276, 637-638: every texture as a lossless WebP, in the reference's member order,
    then meta.json, in a ZIP_STORED archive.  `textures` picks the encoder:
      * a dict of uint8 [height, width, 4] (as SogTextures.to_host returns them): Pillow with the reference's
        arguments, so the members are libwebp's bytes;
      * a SogTextures: gsx.webp encodes each member from HBM and only the compressed bytes come back.  The members
        decode to the same pixels (RGB wherever alpha is not 0; neither encoder keeps RGB under alpha 0) but are
        not libwebp's bytes."""
    names = list(MAIN_FILES) + (list(SHN_FILES) if "shN" in meta else [])
    if isinstance(textures, SogTextures):
        from .webp import encode_lossless
        with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as zf:
            for name in names:
                w, h = textures.sizes[name]
                zf.writestr(name, encode_lossless(textures.textures[name], w, h))
            zf.writestr("meta.json", json.dumps(meta))
        return
    from PIL import Image
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as zf:
        for name in names:
            a = np.ascontiguousarray(textures[name], dtype=np.uint8)
            h, w = a.shape[:2]
            img = Image.frombytes("RGBA", (w, h), a.tobytes())
            bio = io.BytesIO()
            img.save(bio, format="WEBP", lossless=True, quality=100, method=1)
            zf.writestr(name, bio.getvalue())
        zf.writestr("meta.json", json.dumps(meta))


def _module_codebook_fit(cls):
    """The codebook fit of sog.py:561 with MiniBatchKMeans resolved from the writer's module at call time, so a
    patched class there (gsx.dropin.patch(codebook="gpu")) applies."""
    def fit(values):
        mbk = getattr(sys.modules.get(cls.__module__), "MiniBatchKMeans", None)
        if mbk is None:
            from sklearn.cluster import MiniBatchKMeans as mbk
        return mbk(n_clusters=CODEBOOK_K, n_init="auto").fit(values).cluster_centers_
    return fit


def prepare_write(self, data: np.ndarray, *args, **kwargs):
    """SogFormat.write(data, path, **kwargs) for gsx.dropin.install_writer: packed-float32 records encoded on the
    device; returns the step that bundles them with write_sog, its WebP members by Pillow (install option webp="host",
    libwebp's bytes) or by gsx.webp from HBM (webp="device")."""
    from .records import DeviceRecords, is_packed_f32
    if args:
        raise TypeError("SogFormat.write takes no positional arguments after path")
    if not is_packed_f32(data):
        raise ValueError("SOG on the device needs packed all-float32 records")
    import PIL.Image  # noqa: F401  (the reference refuses without Pillow)
    tex = encode(DeviceRecords.from_structured(data), kwargs.get("compression_level", 0),
                 codebook_fit=_module_codebook_fit(type(self)))
    textures = tex if self._gsx_options["write"]["webp"] == "device" else tex.to_host()
    return lambda path: write_sog(path, textures, tex.meta)

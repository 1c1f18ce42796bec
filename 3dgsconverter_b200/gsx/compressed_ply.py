"""PlayCanvas compressed PLY on the device.  decode: formats/compressed_ply.py:14-123 (CompressedPlyFormat.read): the
PLY header parsed on the host, every splat de-normalised on the GPU (gsx_cply_decode).  encode / export:
formats/compressed_ply.py:126-250 (CompressedPlyFormat.write) over DeviceRecords.  The Morton order (gsx_morton_order), the chunk bounds (gsx_chunk_minmax) and the per-splat packing
(gsx_cply_pack) run on the GPU; only the packed 16 B per splat plus the SH bytes come back to the host.

    enc = encode(records)                       # DeviceRecords -> CompressedPly (device tensors)
    chunk_data, vertex_data, sh_data = enc.to_host()
    write_ply("out.compressed.ply", chunk_data, vertex_data, sh_data)
    dec = decode("in.compressed.ply")           # -> readers.Decoded (rows, dtype, metadata)
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

CHUNK = 256
PACK_FIELDS = ("x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2",
               "rot_0", "rot_1", "rot_2", "rot_3")
CHUNK_DTYPE = np.dtype([(f, "<f4") for f in (
    "min_x", "min_y", "min_z", "max_x", "max_y", "max_z",
    "min_scale_x", "min_scale_y", "min_scale_z", "max_scale_x", "max_scale_y", "max_scale_z",
    "min_r", "min_g", "min_b", "max_r", "max_g", "max_b")])
VERTEX_DTYPE = np.dtype([(f, "<u4") for f in ("packed_position", "packed_rotation", "packed_scale", "packed_color")])


def sh_keep_limit(last_nonzero: int) -> int:
    """compressed_ply.py:158-167: how many leading f_rest_i the file keeps, from the last non-zero index."""
    return 45 if last_nonzero >= 24 else 24 if last_nonzero >= 9 else 9 if last_nonzero >= 0 else 0


@dataclass
class CompressedPly:
    chunk: torch.Tensor             # float32 [C, 18]
    vertex: torch.Tensor            # int32 [N, 4]: the four uint32 words of every splat
    sh: torch.Tensor | None         # uint8 [N, len(sh_names)]
    sh_names: tuple
    order: torch.Tensor             # int32 [N]: record index of the j-th splat of the file

    def to_host(self):
        """(chunk_data, vertex_data, sh_data): the structured arrays the reference passes to _write_ply_file."""
        from .hostcopy import to_host
        chunk_data = to_host(self.chunk).reshape(-1).view(CHUNK_DTYPE)
        vertex_data = to_host(self.vertex).reshape(-1).view(VERTEX_DTYPE)
        sh_data = None
        if self.sh is not None:
            sh_data = to_host(self.sh).reshape(-1).view(np.dtype([(n, "u1") for n in self.sh_names]))
        return chunk_data, vertex_data, sh_data


def encode(records, order: torch.Tensor | None = None) -> CompressedPly:
    """Pack `records` (DeviceRecords) the way CompressedPlyFormat.write does.  order: None = the recursive Morton order
    of the reference (gsx_morton_order, ties in ascending index); otherwise a permutation of range(N) (int32)."""
    from .morton import chunk_minmax, morton_order
    missing = [f for f in PACK_FIELDS if f not in records.col]
    if missing:
        raise ValueError(f"compressed PLY needs the fields {missing}")
    n, dev = len(records), records.rows.device
    if order is None:
        order = morton_order(records.xyz_opacity()[0])
    else:
        order = order.to(device=dev, dtype=torch.int32).contiguous()
        if order.shape != (n,):
            raise ValueError(f"order must have shape ({n},), got {tuple(order.shape)}")
        if n:
            lo, hi = torch.aminmax(order)
            if int(lo) < 0 or int(hi) >= n:
                raise ValueError("order holds indices outside [0, N)")
    rest = [(i, records.col[f"f_rest_{i}"]) for i in range(45) if f"f_rest_{i}" in records.col]
    cols = [records.col[f] for f in PACK_FIELDS]
    nchunk = (n + CHUNK - 1) // CHUNK
    lo6, hi6 = chunk_minmax(records.rows, cols[:6], order, CHUNK)
    lo3, hi3 = chunk_minmax(records.rows, cols[7:10], order, CHUNK, clip=(-20.0, 20.0))
    chunk = torch.empty((nchunk, 18), dtype=torch.float32, device=dev)
    vertex = torch.empty((n, 4), dtype=torch.int32, device=dev)
    sh = torch.empty((n, len(rest)), dtype=torch.uint8, device=dev)
    nonzero = torch.empty(1, dtype=torch.int64, device=dev)
    c14 = (C.c_int32 * 14)(*cols)
    crest = (C.c_int32 * max(len(rest), 1))(*[c for _, c in rest])
    check(lib.gsx_cply_pack(_ptr(records.rows), n, records.F, _ptr(order), c14, crest, len(rest), _ptr(lo6), _ptr(hi6),
                            _ptr(lo3), _ptr(hi3), _ptr(chunk), _ptr(vertex), _ptr(sh), _ptr(nonzero), _stream()),
          "gsx_cply_pack")
    mask = 0
    if n:
        from .hostcopy import to_host
        mask = int(to_host(nonzero).view(np.uint64)[0])
    last = max((i for k, (i, _) in enumerate(rest) if mask >> k & 1), default=-1)
    limit = sh_keep_limit(last)
    keep = sum(1 for i, _ in rest if i < limit)
    if keep == 0:
        sh = None
    elif keep < len(rest):
        narrow = torch.empty((n, keep), dtype=torch.uint8, device=dev)
        check(lib.gsx_cply_narrow_sh(_ptr(sh), n, len(rest), keep, _ptr(narrow), _stream()), "gsx_cply_narrow_sh")
        sh = narrow
    names = tuple(f"f_rest_{i}" for i, _ in rest[:keep])
    return CompressedPly(chunk, vertex, sh, names, order)


PLY_TYPE_NAMES = {("i", 1): "char", ("u", 1): "uchar", ("i", 2): "short", ("u", 2): "ushort", ("i", 4): "int",
                  ("u", 4): "uint", ("f", 4): "float", ("f", 8): "double"}


def ply_header(elements) -> tuple[bytes, list]:
    """(header, layouts) of a binary little-endian PLY with `elements` = [(name, count, dtype)]: the text plyfile's
    PlyData(elements, byte_order='<').write emits, restated here because plyfile is not a dependency of gsx
    (property type names char uchar short ushort int uint float double), and each element's packed little-endian row
    dtype.  Raises ValueError for a field type plyfile does not write (bool, 8-byte integers, sub-arrays, ...)."""
    lines = ["ply", "format binary_little_endian 1.0"]
    layouts = []
    for name, count, dtype in elements:
        lines.append(f"element {name} {count}")
        fields = []
        for f in dtype.names:
            dt = dtype.fields[f][0]
            if dt.shape or (dt.kind, dt.itemsize) not in PLY_TYPE_NAMES:
                raise ValueError(f"{name}.{f}: unsupported PLY property type {dt}")
            lines.append(f"property {PLY_TYPE_NAMES[(dt.kind, dt.itemsize)]} {f}")
            fields.append((f, f"<{dt.kind}{dt.itemsize}"))
        layouts.append(np.dtype(fields))
    lines.append("end_header")
    return ("\n".join(lines) + "\n").encode("ascii"), layouts


def write_ply(path, chunk_data: np.ndarray, vertex_data: np.ndarray, sh_data: np.ndarray | None = None) -> None:
    """Binary little-endian PLY with the elements chunk, vertex and (if given) sh -- what _write_ply_file writes through
    plyfile (compressed_ply.py:380-385), for users of gsx without plyfile."""
    elements = [("chunk", chunk_data), ("vertex", vertex_data)] + ([("sh", sh_data)] if sh_data is not None else [])
    header, layouts = ply_header([(name, len(a), a.dtype) for name, a in elements])
    with open(path, "wb") as fh:
        fh.write(header)
        for (_, a), layout in zip(elements, layouts):
            fh.write(np.ascontiguousarray(a.astype(layout)).tobytes())


def prepare_write(self, data: np.ndarray, *args, **kwargs):
    """CompressedPlyFormat.write(data, path, **kwargs) for gsx.dropin.install_writer: packed-float32 records encoded
    on the device; returns the step that writes them with the class's own _write_ply_file."""
    from .records import DeviceRecords, is_packed_f32
    if args:
        raise TypeError("CompressedPlyFormat.write takes no positional arguments after path")
    if not is_packed_f32(data):
        raise ValueError("compressed PLY on the device needs packed all-float32 records")
    chunk_data, vertex_data, sh_data = encode(DeviceRecords.from_structured(data)).to_host()
    return lambda path: self._write_ply_file(path, chunk_data, vertex_data, sh_data)


FIXED_FIELDS = ("x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1",
                "scale_2", "rot_0", "rot_1", "rot_2", "rot_3")


def read_tables():
    """The byte-indexed maps of compressed_ply.py:113-122 (opacity logit, SH), float64 as NumPy promotes them and
    rounded to float32 as the reader stores them."""
    b = np.arange(256, dtype=np.uint8)
    a = np.clip(b / 255.0, 1e-6, 1.0 - 1e-6)
    return np.log(a / (1.0 - a)).astype(np.float32), ((b / 256.0 - 0.5) * 8.0).astype(np.float32)


def _offsets(el, names, want):
    """Byte offsets of `names` in element `el`, each of NumPy type `want`."""
    out = []
    for f in names:
        if f not in (el.dtype.names or ()) or el.dtype.fields[f][0] != np.dtype(want):
            raise ValueError(f"compressed PLY: {el.name}.{f} missing or not {want}")
        out.append(el.dtype.fields[f][1])
    return out


DECODE_ROWS = 128                  # rows per CTA of gsx_cply_decode
DECODE_ROW_MAX = 1024              # the widest chunk, vertex or sh row it stages
DECODE_SMEM_MAX = 200 * 1024       # dynamic shared memory per CTA it accepts


def decode_smem_bytes(vertex_row: int, sh_row: int, nsh: int) -> int:
    """Dynamic shared memory per CTA of gsx_cply_decode (cply_decode in gsx_readers.cu): the staged vertex and sh rows,
    each rounded up to 16 bytes with 16 bytes of slack, then the output rows."""
    up16 = lambda x: (x + 15) & ~15  # noqa: E731
    return (up16(DECODE_ROWS * vertex_row + 16) + (up16(DECODE_ROWS * sh_row + 16) if nsh else 0) +
            DECODE_ROWS * 4 * (len(FIXED_FIELDS) + nsh) + 16)


def decode(data, device="cuda"):
    """CompressedPlyFormat.read on the device, `data` the file's bytes or its path.  Binary little-endian PLY with the
    elements chunk (float32 bounds), vertex (uint32 packed words) and optionally sh (uchar); property types may use
    either PLY name (float / float32, uint / uint32, uchar / uint8) and come in any order.  Refused (ValueError): no
    chunk element (the reference reads such a file as a plain 3DGS PLY), anything parse_ply_header refuses, a body cut
    short, an sh element shorter than vertex or with more than 64 properties, SH names that repeat a fixed field, a
    chunk, vertex or sh row wider than 1024 bytes, rows that need more than 200 KB of shared memory per CTA."""
    from . import readers
    buf = readers.file_bytes(data)
    els, end = readers.parse_ply_header(buf)
    if "chunk" not in els or "vertex" not in els:
        raise ValueError("compressed PLY: no chunk or vertex element")
    if end > len(buf):
        raise ValueError("compressed PLY: body cut short")
    ch, vx, sh = els["chunk"], els["vertex"], els.get("sh")
    coffs = _offsets(ch, CHUNK_DTYPE.names, "<f4")
    voffs = _offsets(vx, VERTEX_DTYPE.names, "<u4")
    names = list(sh.dtype.names or ()) if sh is not None else []
    soffs = _offsets(sh, names, "u1") if names else []
    n = vx.count
    if sh is not None and sh.count < n:
        raise ValueError("compressed PLY: sh element shorter than vertex")
    if len(names) > 64 or set(names) & set(FIXED_FIELDS):
        raise ValueError("compressed PLY: sh properties not read on the device")
    if n >= 1 << 31:
        raise ValueError("compressed PLY: 2^31 splats or more")
    # the kernel refuses these too, but as a GsxError after the upload; the caller is promised a ValueError
    srow = sh.dtype.itemsize if names else 0
    if max(ch.dtype.itemsize, vx.dtype.itemsize, srow) > DECODE_ROW_MAX:
        raise ValueError(f"compressed PLY: rows of {ch.dtype.itemsize} / {vx.dtype.itemsize} / {srow} bytes (chunk / "
                         f"vertex / sh); at most {DECODE_ROW_MAX} are read on the device")
    smem = decode_smem_bytes(vx.dtype.itemsize, srow, len(names))
    if smem > DECODE_SMEM_MAX:
        raise ValueError(f"compressed PLY: these rows need {smem} bytes of shared memory per CTA, more than "
                         f"{DECODE_SMEM_MAX}")
    degree = 3 if len(names) >= 45 else 2 if len(names) >= 24 else 1 if len(names) >= 9 else 0
    metadata = {"count": n, "sh_degree": degree, "chunks": ch.count}
    dtype = np.dtype([(f, "<f4") for f in FIXED_FIELDS + tuple(names)])
    raw = readers.upload(buf, device)
    dev, base = raw.device, raw.data_ptr()
    rows = torch.empty((n, dtype.itemsize), dtype=torch.uint8, device=dev)
    tabs = readers.tables_on(dev, *read_tables())
    i32 = lambda v: (C.c_int32 * max(len(v), 1))(*v)  # noqa: E731
    with torch.cuda.device(dev):
        check(lib.gsx_cply_decode(C.c_void_p(base + ch.offset), ch.count, max(ch.dtype.itemsize, 1), i32(coffs),
                                  C.c_void_p(base + vx.offset), n, vx.dtype.itemsize, i32(voffs),
                                  C.c_void_p(base + sh.offset) if names else None, sh.dtype.itemsize if names else 0,
                                  i32(soffs), len(names), _ptr(tabs), _ptr(rows), _stream()), "gsx_cply_decode")
    return readers.Decoded(rows, dtype, metadata)

"""The .spz reader and writer on the device.  decode: formats/spz.py:18-47, 175-296 (SpzFormat.read, _read_body): gunzip
on the GPU (gsx.deflate.gunzip), the 16-byte header on the host, the planar body on the GPU (gsx_spz_decode).  encode: formats/spz.py:49-173
(SpzFormat.write, _pack_v3) over DeviceRecords.  The SH degree
rule reads one non-zero mask of the f_rest columns (gsx_codec_sh_mask); the planar body is packed on the GPU
(gsx_spz_pack) behind the 16-byte header; the host runs gzip, or with where="device" gsx.deflate does, cutting its
blocks at the section boundaries.

    enc = encode(records)                           # DeviceRecords -> Spz (device payload: header + body)
    write_spz("out.spz", enc, compression_level=0)
    write_spz("out.spz", enc, 6, where="device")    # gzip on the GPU: only the compressed file crosses PCIe
    dec = decode("in.spz")                          # -> readers.Decoded: dec.to_host() is what SpzFormat.read returns
"""
from __future__ import annotations

import ctypes as C
import gzip
import struct
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from . import readers
from ._abi import lib, check
from .compressed_ply import PACK_FIELDS
from ._abi import _ptr, _stream

MAGIC, VERSION, FRACTIONAL_BITS, FLAG_ANTIALIASED = 0x5053474E, 3, 12, 1
SH_DIM = {0: 0, 1: 3, 2: 8, 3: 15}


@dataclass
class Spz:
    payload: torch.Tensor   # uint8 [16 + N * (20 + 3 * sh_dim)]: the uncompressed file, header included
    sh_degree: int

    def to_host(self) -> bytes:
        """The payload the reference hands to gzip.compress."""
        from .hostcopy import to_host
        return to_host(self.payload).tobytes()

    def sections(self) -> list:
        """Offsets where the payload's sections start: the 16-byte header, then positions 9n, alphas n, colours 3n,
        scales 3n, rotations 4n and SH 3 * dim * n."""
        n = (self.payload.numel() - 16) // (20 + 3 * SH_DIM[self.sh_degree])
        return list(np.cumsum([16, 9 * n, n, 3 * n, 3 * n, 4 * n]))

    def compress(self, compression_level: int, mtime: int | None = None) -> bytes:
        """The .spz file: the payload gzipped on the device (gsx.deflate) with its blocks cut at the sections."""
        from .deflate import gzip as device_gzip
        return device_gzip(self.payload, compression_level, mtime=mtime, breaks=self.sections())


def sh_degree(records) -> int:
    """spz.py:50-77: the degree the field names allow, lowered to that of the last f_rest column with a value != 0."""
    col = records.col
    degree = 0
    if "f_rest_0" in col:
        degree = 3 if "f_rest_44" in col else 2 if "f_rest_23" in col else 1 if "f_rest_8" in col else 0
    if degree == 0:
        return 0
    top = {3: 44, 2: 23, 1: 8}[degree]
    nz = records.nonzero_columns([f"f_rest_{i}" for i in range(top + 1)])
    last = max((i for i in range(top + 1) if f"f_rest_{i}" in nz), default=-1)
    return 3 if last >= 24 else 2 if last >= 9 else 1 if last >= 0 else 0


def encode(records) -> Spz:
    """Pack `records` (DeviceRecords) as SpzFormat.write does, up to the gzip step."""
    missing = [f for f in PACK_FIELDS if f not in records.col]
    if missing:
        raise ValueError(f".spz needs the fields {missing}")
    degree = sh_degree(records)
    dim = SH_DIM[degree]
    sh_names = [f"f_rest_{i + 15 * c}" for i in range(dim) for c in range(3)]
    absent = [f for f in sh_names if f not in records.col]
    if absent:   # the reference raises a KeyError here
        raise ValueError(f"SH degree {degree} of the SPZ layout needs the fields {absent}")
    n, dev = len(records), records.rows.device
    from .hostcopy import to_device
    head = struct.pack("<IIIBBBB", MAGIC, VERSION, n, degree, FRACTIONAL_BITS, FLAG_ANTIALIASED, 0)
    payload = torch.empty(16 + n * (20 + 3 * dim), dtype=torch.uint8, device=dev)
    payload[:16].copy_(to_device(np.frombuffer(head, np.uint8), dev))
    c14 = (C.c_int32 * 14)(*[records.col[f] for f in PACK_FIELDS])
    csh = (C.c_int32 * max(len(sh_names), 1))(*[records.col[f] for f in sh_names])
    check(lib.gsx_spz_pack(_ptr(records.rows), n, records.F, c14, csh, dim, _ptr(payload[16:]), _stream()),
          "gsx_spz_pack")
    return Spz(payload, degree)


def _where(where: str) -> str:
    if where not in ("host", "device"):
        raise ValueError(f"gzip must run on the 'host' or the 'device', not {where!r}")
    return where


def write_spz(path, enc: Spz, compression_level=0, where: str = "host") -> None:
    """gzip at `compression_level` (0 = stored): where="host" copies the payload back and runs gzip.compress, as
    spz.py:97-102; where="device" runs gsx.deflate (Spz.compress) and copies back only the file."""
    if _where(where) == "device":
        blob = enc.compress(compression_level)
    else:
        blob = gzip.compress(enc.to_host(), compresslevel=compression_level)
    with open(path, "wb") as fh:
        fh.write(blob)


def prepare_write(self, data: np.ndarray, *args, **kwargs):
    """SpzFormat.write(data, path, **kwargs) for gsx.dropin.install_writer: the payload packed on the device and
    gzipped where the install option gzip says ("host": gzip.compress, the reference's bytes; "device": gsx.deflate);
    returns the step that writes the file to path."""
    from .records import DeviceRecords
    if args:
        raise TypeError("SpzFormat.write takes no positional arguments after path")
    enc = encode(DeviceRecords.from_writer_input(data))
    level = kwargs.get("compression_level", 0)
    if self._gsx_options["write"]["gzip"] == "device":
        blob = enc.compress(level)
    else:
        blob = gzip.compress(enc.to_host(), compresslevel=level)
    return lambda path: Path(path).write_bytes(blob)


def read_tables():
    """The byte-indexed maps of spz.py:200-222, 243, 345-348 (opacity logit, DC, red/green/blue, scale, SH), with the
    reference's expressions and dtypes; the scale map is float64 (u8 / 16.0), stored as float32 as the reader stores
    it."""
    b = np.arange(256, dtype=np.uint8)
    v = np.clip(b.astype(np.float32) / 255.0, 1e-7, 1.0 - 1e-7)
    dc = (b.astype(np.float32) / 255.0 - 0.5) / 0.15
    rgb = np.clip((0.5 + readers.SH_C0 * dc) * 255.0, 0, 255).astype(np.uint8)
    return np.log(v / (1.0 - v)), dc, rgb, (b / 16.0 - 10.0).astype(np.float32), (b.astype(np.float32) - 128.0) / 128.0


def decode(data, device="cuda") -> readers.Decoded:
    """SpzFormat.read on the device, `data` the file's bytes or its path.  A file that starts with 1f 8b is gunzipped
    on the device (gsx.deflate.gunzip: gzip.decompress's bytes or exception class), so only the file crosses PCIe and
    only the 16-byte header comes back -- unless its first block is stored (level 0, the reference writer's default),
    where gzip.decompress on the host is faster.  Refused (ValueError) where the reference raises or does not read the file
    as written: a bad magic or version, a body shorter than the header's count needs, 1 << frac_bits beyond
    float32."""
    buf = readers.file_bytes(data)
    payload = None
    if len(buf) > 2 and buf[0] == 0x1F and buf[1] == 0x8B:
        from .deflate import first_block_stored, gunzip
        if first_block_stored(buf):      # level 0: zlib's copy on the host is faster than the device's chunk chain
            buf = memoryview(gzip.decompress(buf))
        else:
            from .hostcopy import to_host
            payload = gunzip(buf, device)
    if payload is not None:
        size, head = payload.numel(), to_host(payload[:16]).tobytes()
    else:
        size, head = len(buf), bytes(buf[:16])
    if size < 16:
        raise ValueError("spz: shorter than its header")
    magic, version, n, degree, frac_bits, _, _ = struct.unpack_from("<IIIBBBB", head, 0)
    if magic != MAGIC or not 1 <= version <= 3:
        raise ValueError(f"spz: magic {magic:#x} / version {version}")
    if frac_bits > 127:
        raise ValueError(f"spz: 1 << {frac_bits} is not a float32")
    if n >= 1 << 31:
        raise ValueError("spz: 2^31 splats or more")
    dim = SH_DIM.get(degree, 0)
    need = n * ((6 if version == 1 else 9) + 7 + (4 if version >= 3 else 3) + 3 * dim)
    if size - 16 < need:
        raise ValueError("spz: body cut short")
    dtype = readers.gaussian_dtype(has_rgb=True, sh_degree=degree)
    raw = payload[16:16 + need] if payload is not None else readers.upload(buf[16:16 + need], device)
    rows = torch.empty((n, dtype.itemsize), dtype=torch.uint8, device=raw.device)
    tabs = readers.tables_on(raw.device, *read_tables())
    with torch.cuda.device(raw.device):
        check(lib.gsx_spz_decode(_ptr(raw), n, version, dim, frac_bits, _ptr(tabs), dtype.itemsize, _ptr(rows),
                                 _stream()), "gsx_spz_decode")
    return readers.Decoded(rows, dtype, None)

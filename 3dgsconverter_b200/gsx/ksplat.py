"""The .ksplat reader and writer on the device.  decode: formats/ksplat.py:29-317 (KSplatFormat.read): the headers are
parsed on the host, every section's records decoded on the GPU (gsx_ksplat_decode_section).  encode:
formats/ksplat.py:319-544 (KSplatFormat.write) over DeviceRecords.  The SH degree
rule reads one non-zero mask of the f_rest columns (gsx_codec_sh_mask); the bucket bounds (gsx_chunk_minmax), their
centres and the interleaved records are computed on the GPU; the host builds the two headers.

    enc = encode(records, compression_level=1)     # DeviceRecords -> KSplat (device tensors)
    write_ksplat("out.ksplat", enc)                 # or enc.to_host(): the file's bytes
    dec = decode("in.ksplat")                       # -> readers.Decoded (rows, dtype, metadata)
"""
from __future__ import annotations

import ctypes as C
import struct
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from . import readers
from ._abi import lib, check
from .compressed_ply import PACK_FIELDS
from ._abi import _ptr, _stream

HEADER_SIZE, SECTION_HEADER_SIZE = 4096, 1024
MAGIC_MAJOR, MAGIC_MINOR = 0, 1
MIN_SH, MAX_SH = -2.0, 2.0
SCALE_RANGE = 32767


@dataclass
class KSplat:
    head: bytes                     # file header, section header and the partial-bucket length word (if any)
    centres: torch.Tensor | None    # float32 [B, 3]: bucket centres (levels >= 1)
    records: torch.Tensor           # uint8 [N, record bytes]: the interleaved splats
    sh_degree: int

    def to_host(self) -> bytes:
        """The whole .ksplat file."""
        from .hostcopy import to_host
        parts = [self.head] + ([to_host(self.centres).data] if self.centres is not None else [])
        return b"".join(parts + [to_host(self.records).data])


def _headers(n: int, level: int, sh_degree: int, sh_count: int, bucket_size: int, block_size: float) -> bytes:
    """ksplat.py:370-417, field for field."""
    header = bytearray(HEADER_SIZE)
    header[0], header[1] = MAGIC_MAJOR, MAGIC_MINOR
    struct.pack_into("<IIII", header, 4, 1, 1, n, n)
    struct.pack_into("<H", header, 20, level)
    struct.pack_into("<ff", header, 36, MIN_SH, MAX_SH)
    section = bytearray(SECTION_HEADER_SIZE)
    struct.pack_into("<II", section, 0, n, n)
    if level >= 1:
        struct.pack_into("<II", section, 8, bucket_size, (n + bucket_size - 1) // bucket_size)
        struct.pack_into("<f", section, 16, block_size)
        struct.pack_into("<H", section, 20, 12)
        struct.pack_into("<I", section, 24, SCALE_RANGE)
    per_splat = 44 + 4 * sh_count if level == 0 else 24 + (2 if level == 1 else 1) * sh_count
    full, partial = n // bucket_size, 1 if n % bucket_size else 0
    storage = partial * 4 + ((full + partial) * 12 if level >= 1 else 0) + n * per_splat
    struct.pack_into("<III", section, 28, storage, full, partial)
    struct.pack_into("<H", section, 40, sh_degree)
    return bytes(header) + bytes(section) + (struct.pack("<I", n % bucket_size) if partial else b"")


def encode(records, compression_level=0, sh_level=None, bucket_size=256, block_size=5.0) -> KSplat:
    """Pack `records` (DeviceRecords) as KSplatFormat.write(data, path, compression_level, sh_level=...,
    bucket_size=..., block_size=...) does.  None takes the reference's default for any argument but the level."""
    level = int(compression_level)
    sh_level = None if sh_level is None else int(sh_level)
    bucket_size = 256 if bucket_size is None else int(bucket_size)
    block_size = 5.0 if block_size is None else float(block_size)
    if not 0 <= level <= 65535 or bucket_size < 1:
        raise ValueError(f"compression_level {level} / bucket_size {bucket_size} out of range")
    missing = [f for f in PACK_FIELDS if f not in records.col]
    if missing:
        raise ValueError(f".ksplat needs the fields {missing}")
    nz = records.nonzero_columns([f"f_rest_{j}" for j in range(24)])
    degree = 0
    if any(f"f_rest_{j}" in nz for j in range(9)):
        degree = 2 if any(f"f_rest_{j}" in nz for j in range(9, 24)) else 1
    if sh_level is not None and sh_level < degree:
        degree = sh_level
    if degree < 0:
        raise ValueError(f"sh_level {sh_level} < 0")
    sh_count = {1: 9, 2: 24}.get(degree, 0)
    sh_names = [f"f_rest_{j}" for j in range(sh_count)]
    if any(f not in records.col for f in sh_names):
        raise ValueError(f"SH degree {degree} needs the fields f_rest_0 .. f_rest_{sh_count - 1}")
    n, dev = len(records), records.rows.device
    head = _headers(n, level, degree, sh_count, bucket_size, block_size)
    centres = None
    sf_inv = 0.0
    if level >= 1:
        from .morton import chunk_minmax
        nb = (n + bucket_size - 1) // bucket_size
        centres = torch.empty((nb, 3), dtype=torch.float32, device=dev)
        if n:
            lo, hi = chunk_minmax(records.rows, [records.col[f] for f in ("x", "y", "z")], None, bucket_size)
            check(lib.gsx_ksplat_centres(_ptr(lo), _ptr(hi), nb, _ptr(centres), _stream()), "gsx_ksplat_centres")
        sf_inv = float(np.float32(SCALE_RANGE / (block_size / 2.0)))
    rec = lib.gsx_ksplat_record_bytes(min(level, 3), sh_count)
    out = torch.empty((n, rec), dtype=torch.uint8, device=dev)
    c14 = (C.c_int32 * 14)(*[records.col[f] for f in PACK_FIELDS])
    csh = (C.c_int32 * max(sh_count, 1))(*[records.col[f] for f in sh_names])
    check(lib.gsx_ksplat_pack(_ptr(records.rows), n, records.F, c14, csh, sh_count, level, bucket_size, sf_inv,
                              _ptr(centres), _ptr(out), _stream()), "gsx_ksplat_pack")
    return KSplat(head, centres, out, degree)


def write_ksplat(path, enc: KSplat) -> None:
    with open(path, "wb") as fh:
        fh.write(enc.to_host())


def prepare_write(self, data: np.ndarray, *args, **kwargs):
    """KSplatFormat.write(data, path, compression_level=0, **kwargs) for gsx.dropin.install_writer: the file's bytes,
    packed on the device; returns the step that writes them to path."""
    from .records import DeviceRecords
    level = args[0] if args else kwargs.get("compression_level", 0)
    blob = encode(DeviceRecords.from_writer_input(data), level, kwargs.get("sh_level"), kwargs.get("bucket_size"),
                  kwargs.get("block_size")).to_host()
    return lambda path: Path(path).write_bytes(blob)


def read_tables():
    """The byte-indexed maps of ksplat.py:24-27, 229-234, 257-258 (DC, opacity logit, level-2 SH), with the reference's
    expressions and dtypes."""
    b = np.arange(256, dtype=np.uint8)
    dc = (b.astype(np.float32) / 255.0 - 0.5) / 0.28209479177387814
    alpha = np.clip(b.astype(np.float32) / 255.0, 1e-7, 1.0 - 1e-7)
    return dc, np.log(alpha / (1.0 - alpha)), (b.astype(np.float32) - 128.0) / 128.0


_SECTION_KEYS = ("splatCount", "maxSplatCount", "bucketSize", "bucketCount", "bucketBlockSize", "bucketStorageSizeBytes",
                 "compressionScaleRange", "storageSizeBytes", "fullBucketCount", "partiallyFilledBucketCount",
                 "shDegree")


def decode(data, device="cuda") -> readers.Decoded:
    """KSplatFormat.read on the device, `data` the file's bytes or its path.  Refused (ValueError) where the reference
    raises or does not read the file as written: a version other than 0.1, headers or sections cut short, levels >= 1
    without bucket centres or with partial-bucket lengths that leave splats without a bucket or reach a bucket past the
    centres, SH degrees above 255."""
    buf = readers.file_bytes(data)
    if len(buf) < HEADER_SIZE:
        raise ValueError("ksplat: file shorter than its header")
    if (buf[0], buf[1]) != (MAGIC_MAJOR, MAGIC_MINOR):
        raise ValueError(f"ksplat: version {buf[0]}.{buf[1]}, not {MAGIC_MAJOR}.{MAGIC_MINOR}")
    max_sections, _, _, splat_count = struct.unpack_from("<IIII", buf, 4)
    level = struct.unpack_from("<H", buf, 20)[0]
    min_sh, max_sh = struct.unpack_from("<ff", buf, 36)
    payload = HEADER_SIZE + max_sections * SECTION_HEADER_SIZE
    if payload > len(buf):
        raise ValueError("ksplat: section headers cut short")
    sections = []
    for i in range(max_sections):
        vals = struct.unpack_from("<IIIIfHxxIIIIH", buf, HEADER_SIZE + i * SECTION_HEADER_SIZE)
        sec = dict(zip(_SECTION_KEYS, vals))
        if sec["compressionScaleRange"] == 0 and level >= 1:
            sec["compressionScaleRange"] = 32767
        sections.append(sec)
    metadata = {"v_major": buf[0], "v_minor": buf[1], "splat_count": splat_count, "compression_level": level,
                "min_sh": min_sh, "max_sh": max_sh, "sections": sections}
    degree = max((s["shDegree"] for s in sections), default=3)
    if degree > 255:
        raise ValueError(f"ksplat: SH degree {degree}")
    dtype = readers.gaussian_dtype(sh_degree=degree)
    lv = min(level, 2)
    plan, off, total = [], payload, 0
    for sec in sections:   # ksplat.py:109-145: where each section's arrays lie, checked before any upload
        n, npart, nb = sec["splatCount"], sec["partiallyFilledBucketCount"], sec["bucketCount"]
        sh_count = {1: 9, 2: 24}.get(sec["shDegree"], 0)
        per = 44 + 4 * sh_count if lv == 0 else 24 + (2 if lv == 1 else 1) * sh_count
        lengths_at, centres_at, rec_at = off, off + 4 * npart, off + 4 * npart + 12 * nb
        if rec_at + n * per > len(buf):
            raise ValueError("ksplat: section cut short")
        ends = None
        if lv >= 1:
            if nb == 0:
                raise ValueError("ksplat: no bucket centres")
            full = sec["fullBucketCount"] * sec["bucketSize"]
            ends = np.cumsum(np.frombuffer(buf, "<u4", npart, lengths_at), dtype=np.int64)
            if full + (int(ends[-1]) if npart else 0) < n:
                raise ValueError("ksplat: the bucket lengths leave splats without a bucket")
            if n:
                last = (n - 1) // sec["bucketSize"] if n <= full else \
                    sec["fullBucketCount"] + int(np.searchsorted(ends, n - 1 - full, side="right"))
                if last >= nb:
                    raise ValueError("ksplat: a splat's bucket has no centre")
        plan.append((sec, n, sh_count, centres_at, rec_at, ends))
        off += 4 * npart + 12 * nb + sec["maxSplatCount"] * per
        total += n
    if total >= 1 << 31:
        raise ValueError("ksplat: 2^31 splats or more")
    raw = readers.upload(buf, device)
    dev = raw.device
    rows = torch.empty((total, dtype.itemsize), dtype=torch.uint8, device=dev)
    tabs = readers.tables_on(dev, *read_tables())
    base, row = raw.data_ptr(), 0
    with torch.cuda.device(dev):
        for sec, n, sh_count, centres_at, rec_at, ends in plan:
            if n == 0:
                continue
            sr = sec["compressionScaleRange"]
            sf = (sec["bucketBlockSize"] / 2.0) / sr if lv >= 1 else 0.0
            ends_dev = None
            if ends is not None and len(ends):
                from .hostcopy import to_device
                ends_dev = to_device(ends, dev)
            check(lib.gsx_ksplat_decode_section(
                C.c_void_p(base + rec_at), n, lv, sh_count, float(np.float32(sr)), float(np.float32(sf)),
                C.c_void_p(base + centres_at), sec["bucketCount"], sec["fullBucketCount"], sec["bucketSize"],
                _ptr(ends_dev), 0 if ends is None else len(ends), _ptr(tabs), dtype.itemsize,
                _ptr(rows[row:row + n]), _stream()), "gsx_ksplat_decode_section")
            row += n
    return readers.Decoded(rows, dtype, metadata)

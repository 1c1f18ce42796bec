"""The .splat reader and writer on the device.  decode: formats/splat.py:9-80 (SplatFormat.read) from the file's bytes
(gsx_splat_decode).  encode: formats/splat.py:82-166 (SplatFormat.write) over DeviceRecords.  The sort metric
and its keys (gsx_splat_sort_keys), the stable radix sort (gsx_sort_pairs) and the 32-byte records (gsx_splat_pack)
run on the GPU.  Equal metrics keep ascending index (NumPy's stable argsort; the reference's default argsort leaves
their order unspecified).

    enc = encode(records)                           # DeviceRecords -> Splat (device tensors)
    write_splat("out.splat", enc)
    dec = decode("in.splat")                        # -> readers.Decoded: dec.to_host() is what SplatFormat.read returns
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from . import readers
from ._abi import lib, check
from .compressed_ply import PACK_FIELDS
from ._abi import _ptr, _stream
from .sor import sort_pairs


@dataclass
class Splat:
    data: torch.Tensor      # uint8 [N, 32]: the file
    order: torch.Tensor     # int32 [N]: record index of the j-th splat of the file

    def to_host(self) -> bytes:
        from .hostcopy import to_host
        return to_host(self.data).tobytes()


def encode(records) -> Splat:
    """Sort and pack `records` (DeviceRecords) as SplatFormat.write does."""
    missing = [f for f in PACK_FIELDS if f not in records.col]
    if missing:
        raise ValueError(f".splat needs the fields {missing}")
    n, dev = len(records), records.rows.device
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    order = torch.empty(n, dtype=torch.int32, device=dev)
    c4 = (C.c_int32 * 4)(*[records.col[f] for f in ("scale_0", "scale_1", "scale_2", "opacity")])
    check(lib.gsx_splat_sort_keys(_ptr(records.rows), n, records.F, c4, _ptr(keys), _ptr(order), _stream()),
          "gsx_splat_sort_keys")
    if n:
        sort_pairs(keys, order, 0, 32)
    out = torch.empty((n, 32), dtype=torch.uint8, device=dev)
    c14 = (C.c_int32 * 14)(*[records.col[f] for f in PACK_FIELDS])
    check(lib.gsx_splat_pack(_ptr(records.rows), n, records.F, _ptr(order), c14, _ptr(out), _stream()), "gsx_splat_pack")
    return Splat(out, order)


def write_splat(path, enc: Splat) -> None:
    with open(path, "wb") as fh:
        fh.write(enc.to_host())


def prepare_write(self, data: np.ndarray, *args, **kwargs):
    """SplatFormat.write(data, path, **kwargs) for gsx.dropin.install_writer: the file's bytes, sorted and packed on
    the device; returns the step that writes them to path."""
    from .records import DeviceRecords
    if args:
        raise TypeError("SplatFormat.write takes no positional arguments after path")
    blob = encode(DeviceRecords.from_writer_input(data)).to_host()
    return lambda path: Path(path).write_bytes(blob)


def read_tables():
    """The byte-indexed maps of splat.py:67-77 (DC, opacity logit), with the reference's expressions and dtypes."""
    b = np.arange(256, dtype=np.uint8)
    dc = (b.astype(np.float32) / 255.0 - 0.5) / readers.SH_C0
    linear_alpha = np.clip(b.astype(np.float32) / 255.0, 1.0 / 255.0, 0.9999)
    return dc, -np.log((1.0 / linear_alpha) - 1.0)


def decode(data, device="cuda") -> readers.Decoded:
    """SplatFormat.read on the device: every whole 32-byte record of `data` (bytes or a path), trailing bytes ignored
    as np.fromfile ignores them."""
    buf = readers.file_bytes(data)
    n = len(buf) // 32
    dtype = readers.gaussian_dtype(has_rgb=True, sh_degree=0)
    raw = readers.upload(buf[:n * 32], device)
    rows = torch.empty((n, dtype.itemsize), dtype=torch.uint8, device=raw.device)
    tabs = readers.tables_on(raw.device, *read_tables())
    with torch.cuda.device(raw.device):
        check(lib.gsx_splat_decode(_ptr(raw), n, _ptr(tabs), _ptr(rows), _stream()), "gsx_splat_decode")
    return readers.Decoded(rows, dtype, None)

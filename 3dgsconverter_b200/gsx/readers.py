"""What the device readers share (gsx.splat / gsx.ksplat / gsx.spz / gsx.compressed_ply `decode`): the file's bytes,
uploaded once; the reference's output dtype (structures.py:23-59); the result object; and the binary little-endian PLY
header parser of the compressed PLY reader.

    dec = gsx.ksplat.decode("in.ksplat")     # Decoded: rows (uint8 [n, itemsize] on the device), dtype, metadata
    a = dec.to_host()                        # what KSplatFormat.read returns, byte for byte
    r = dec.records()                        # DeviceRecords for FilterChain and the device writers, no host copy

Anything `decode` does not reproduce raises ValueError; the drop-in then runs the reference's own read.
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch

SH_C0 = 0.28209479177387814


def gaussian_dtype(has_rgb: bool = False, sh_degree: int = 3) -> np.dtype:
    """GaussianStruct.define_dtype(has_scal=False, has_rgb, sh_degree=...)[0] as a NumPy dtype (structures.py:23-59)."""
    n_rest = 3 * ((sh_degree + 1) ** 2 - 1)
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", *[f"f_rest_{i}" for i in range(n_rest)],
             "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    fields = [(n, "<f4") for n in names]
    if has_rgb:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    return np.dtype(fields)


def file_bytes(data) -> memoryview:
    """`data` as bytes: a bytes-like object as it is, a path read whole."""
    if isinstance(data, (str, os.PathLike)):
        with open(data, "rb") as fh:
            data = fh.read()
    return memoryview(data).cast("B")


def upload(buf, device) -> torch.Tensor:
    """The bytes of `buf` in one uint8 device tensor (one staged H2D)."""
    from .hostcopy import to_device
    return to_device(np.frombuffer(buf, np.uint8), device)


def tables_on(device, *tables) -> torch.Tensor:
    """float32 [len(tables), 256] on the device: the byte-indexed maps a kernel reads."""
    from .hostcopy import to_device
    return to_device(np.stack([np.asarray(t, np.float32) for t in tables]), device)


@dataclass
class Decoded:
    rows: torch.Tensor          # uint8 [n, dtype.itemsize]: the reference reader's array, row by row
    dtype: np.dtype
    metadata: dict | None       # what the reference sets on self.metadata (ksplat, compressed PLY), else None

    def __len__(self):
        return self.rows.shape[0]

    def to_host(self) -> np.ndarray:
        """The structured array the reference reader returns (one D2H)."""
        from .hostcopy import to_host
        return to_host(self.rows).reshape(-1).view(self.dtype)

    def records(self):
        """DeviceRecords of the float32 fields: a zero-copy view when every field is float32, else gathered on the
        device (gsx_records_from_bytes; the u1 red/green/blue are dropped, as DeviceRecords.from_writer_input does)."""
        from .records import DeviceRecords, is_packed_f32
        if is_packed_f32(np.zeros(0, self.dtype)):
            rows = self.rows.view(torch.float32).view(len(self), len(self.dtype.names))
            return DeviceRecords(rows, self.dtype.names, self.dtype)
        return DeviceRecords.from_device_bytes(self.rows, self.dtype)


# ---------------------------------------------------------------------------------------------- binary PLY header
PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "<i2", "int16": "<i2",
             "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4",
             "float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8"}


@dataclass
class PlyElement:
    name: str
    count: int
    dtype: np.dtype       # one row: its properties in file order, packed
    offset: int           # byte offset of the element's first row in the file


def parse_ply_header(buf):
    """({name: PlyElement}, end of the last element's data) of a binary little-endian PLY whose properties all have a
    fixed size.  Raises ValueError for anything else (ASCII or big-endian bodies, list properties, repeated names)."""
    buf = bytes(buf[:65536]) if len(buf) > 65536 else bytes(buf)
    end = buf.find(b"end_header\n")
    if not buf.startswith(b"ply\n") or end < 0:
        raise ValueError("not a PLY file with a complete header")
    lines = buf[4:end].decode("ascii").split("\n")
    if not lines or lines[0].split() != ["format", "binary_little_endian", "1.0"]:
        raise ValueError("only binary_little_endian 1.0 PLY bodies are read on the device")
    elements, cur = [], None
    for line in lines[1:]:
        w = line.split()
        if not w or w[0] in ("comment", "obj_info"):
            continue
        if w[0] == "element" and len(w) == 3:
            if any(e[0] == w[1] for e in elements):
                raise ValueError(f"element {w[1]!r} repeated")
            cur = [w[1], int(w[2]), []]
            if cur[1] < 0:
                raise ValueError(f"element {w[1]!r} has a negative count")
            elements.append(cur)
        elif w[0] == "property" and len(w) == 3 and cur is not None and w[1] in PLY_TYPES:
            if any(p[0] == w[2] for p in cur[2]):
                raise ValueError(f"property {w[2]!r} repeated in element {cur[0]!r}")
            cur[2].append((w[2], PLY_TYPES[w[1]]))
        else:
            raise ValueError(f"PLY header line {line!r} is not read on the device")
    out, off = {}, end + len(b"end_header\n")
    for name, count, props in elements:
        dt = np.dtype(props) if props else np.dtype([])
        out[name] = PlyElement(name, count, dt, off)
        off += count * dt.itemsize
    return out, off

"""Plain binary PLY on the device, both flavours the reference reads and writes: "3dgs" (formats/ply_3dgs.py,
Ply3DGSFormat: the Inria 3DGS layout, optionally with `scalar_`, `scal_` or `scalar_scal_` prefixes) and "cc"
(formats/ply_cc.py, PlyCCFormat: CloudCompare's `scalar_`-prefixed properties).  The header and the field mapping are
worked out on the host, statement for statement as the reference's read / write; the rows are transcoded on the GPU
in one launch (gsx_ply_transcode: each output field copied from one input field, with a cast, or left zero).

    dec = decode("in.ply")                      # readers.Decoded: rows on the device, dtype
    a = dec.to_host()                           # what Ply3DGSFormat.read returns, byte for byte
    r = dec.records()                           # DeviceRecords (a zero-copy view when every field is float32)
    enc = encode(r, "cc", crop_sh=True)         # Encoded: the rows PlyCCFormat.write hands to PlyElement.describe
    write_ply("out.ply", enc)                   # header + body, as PlyData([el], byte_order='<').write

plyfile is not needed: the header text is a restatement of what plyfile writes (compressed_ply.ply_header).  Anything
decode or encode does not reproduce raises ValueError; the drop-in then runs the reference's own read or write.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

FLAVORS = ("3dgs", "cc")
ROW_MAX = 1024          # widest input or output row gsx_ply_transcode takes, bytes
# PLY property types as gsx_ply_transcode numbers them (char uchar short ushort int uint float double)
TYPE_CODES = {("i", 1): 0, ("u", 1): 1, ("i", 2): 2, ("u", 2): 3, ("i", 4): 4, ("u", 4): 5, ("f", 4): 6, ("f", 8): 7}
_F4, _F8, _U1 = 6, 7, 1
SPATIAL = {"x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"}   # ply_cc.py:86: written without `scalar_`


def standard_order(has_rgb: bool) -> list:
    """GaussianStruct.get_standard_order (structures.py:6-20)."""
    order = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", *[f"f_rest_{i}" for i in range(45)],
             "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    return order + (["red", "green", "blue"] if has_rgb else [])


def _check_flavor(flavor):
    if flavor not in FLAVORS:
        raise ValueError(f"flavor must be one of {FLAVORS}, not {flavor!r}")


def type_code(dt: np.dtype, what: str) -> int:
    """gsx_ply_transcode's number of a field type plyfile writes as listed, in native (little-endian) byte order."""
    if dt.shape or (dt.kind, dt.itemsize) not in TYPE_CODES or dt.byteorder not in "=<|":
        raise ValueError(f"{what}: field type {dt.str} is not read or written on the device")
    return TYPE_CODES[(dt.kind, dt.itemsize)]


def cast_supported(s: int, d: int) -> bool:
    """The casts gsx_ply_transcode reproduces: identity, integer or double -> float, anything -> uchar."""
    return s == d or (d == _F4 and (s <= 5 or s == _F8)) or d == _U1


# ------------------------------------------------------------------------------------------------ host-side layouts
def read_layout(src: np.dtype, flavor: str):
    """(dtype, [(target, source)]): the array Ply3DGSFormat.read (ply_3dgs.py:21-58) or PlyCCFormat.read
    (ply_cc.py:21-60) builds from vertex rows of dtype `src`, and the source field of each target field it fills."""
    _check_flavor(flavor)
    names = src.names or ()
    prefix = ""
    if flavor == "3dgs":   # ply_3dgs.py:22-28
        if "scalar_f_dc_0" in names:
            prefix = "scalar_scal_" if "scalar_scal_f_dc_0" in names else "scalar_"
        elif "scal_f_dc_0" in names:
            prefix = "scal_"
        std = standard_order(True)
    else:                  # ply_cc.py:22-30
        if "scalar_f_dc_0" in names:
            prefix = "scalar_"
        elif "scalar_scal_f_dc_0" in names:
            prefix = "scalar_scal_"
        std = standard_order(True) + ["nx", "ny", "nz"]
    std_source = {prefix + s for s in std} | set(std)
    extras = []
    for name in names:
        if name not in std_source:   # kept with their file type; CC strips `scalar_`
            internal = name[7:] if flavor == "cc" and name.startswith("scalar_") else name
            extras.append((internal, src.fields[name][0].str))
    from .readers import gaussian_dtype
    fields = gaussian_dtype(has_rgb="red" in names).descr
    for name, t in extras:   # define_dtype's duplicate skip (structures.py:53-57)
        if not any(f[0] == name for f in fields):
            fields.append((name, t))
    if any(f[0] == "" for f in fields):
        raise ValueError("PLY: an extra property whose internal name is empty")
    dtype = np.dtype(fields)
    pairs = []
    for target in dtype.names:
        if target in names:
            pairs.append((target, target))
        elif prefix + target in names:
            pairs.append((target, prefix + target))
        elif flavor == "cc" and f"scalar_{target}" in names:
            pairs.append((target, f"scalar_{target}"))
    return dtype, pairs


def write_layout(src: np.dtype, flavor: str, last_rest: int | None = None):
    """(dtype, [(field, out_name)]): the output_data Ply3DGSFormat.write (ply_3dgs.py:65-109) or PlyCCFormat.write
    (ply_cc.py:67-116) builds from records of dtype `src`, and the output field each input field is copied into.
    last_rest: None without crop_sh, else the last f_rest index holding a non-zero value (-1 for none)."""
    _check_flavor(flavor)
    names = src.names or ()
    std = standard_order("red" in names)
    crop = last_rest is not None
    if crop:
        std = [s for s in std if not (s.startswith("f_rest_") and int(s.split("_")[-1]) > last_rest)]
    out_name = (lambda s: s) if flavor == "3dgs" else (lambda s: s if s in SPATIAL else f"scalar_{s}")
    fields, mapping = [], []
    for s in std:
        if s in names:
            fields.append((out_name(s), src.fields[s][0].str))
            mapping.append((s, out_name(s)))
        elif s.startswith("f_rest_"):
            if not crop:
                fields.append((out_name(s), "f4"))
        elif s in ("nx", "ny", "nz"):
            fields.append((s, "f4"))
    full_std = set(standard_order(True))
    for s in names:
        if s not in std and s not in full_std:
            o = s if flavor == "3dgs" else f"scalar_{s}"
            fields.append((o, src.fields[s][0].str))
            mapping.append((s, o))
    return np.dtype(fields), mapping


def field_table(src: np.dtype, dst: np.dtype, pairs, what: str) -> list:
    """gsx_ply_transcode's field table for `pairs` [(source field, destination field)]; ValueError for a cast it does
    not reproduce."""
    table = []
    for s, d in pairs:
        sc, dc = type_code(src.fields[s][0], f"{what}: {s}"), type_code(dst.fields[d][0], f"{what}: {d}")
        if not cast_supported(sc, dc):
            raise ValueError(f"{what}: no device cast from {src.fields[s][0].str} ({s}) to {dst.fields[d][0].str} ({d})")
        table += [src.fields[s][1], sc, dst.fields[d][1], dc]
    return table


def transcode(src_rows: torch.Tensor, src_offset: int, n: int, src_row: int, dst_row: int, table) -> torch.Tensor:
    """uint8 [n, dst_row] on src_rows' device: gsx_ply_transcode of the n rows starting at byte src_offset."""
    if max(src_row, dst_row) > ROW_MAX or min(src_row, dst_row) < 1:
        raise ValueError(f"PLY rows of {src_row} / {dst_row} bytes (in / out); 1 .. {ROW_MAX} are transcoded on the "
                         "device")
    dev = src_rows.device
    out = torch.empty((n, dst_row), dtype=torch.uint8, device=dev)
    nf = len(table) // 4
    with torch.cuda.device(dev):
        check(lib.gsx_ply_transcode(C.c_void_p(src_rows.data_ptr() + src_offset), n, src_row, _ptr(out), dst_row,
                                    (C.c_int32 * max(len(table), 1))(*table), nf, _stream()), "gsx_ply_transcode")
    return out


# ---------------------------------------------------------------------------------------------------------- reading
def read_plan(buf, flavor: str = "3dgs"):
    """(vertex element, output dtype, gsx_ply_transcode field table) of decode, on the host: every refusal of decode
    happens here, before anything is uploaded."""
    from . import readers
    _check_flavor(flavor)
    els, end = readers.parse_ply_header(buf)
    if list(els) != ["vertex"]:
        raise ValueError(f"PLY: elements {list(els)}; only a lone vertex element is read on the device")
    if end > len(buf):
        raise ValueError("PLY: body cut short")
    vx = els["vertex"]
    if vx.count >= 1 << 31:
        raise ValueError("PLY: 2^31 rows or more")
    if not vx.dtype.names:
        raise ValueError("PLY: a vertex element without properties")
    dtype, pairs = read_layout(vx.dtype, flavor)
    if max(vx.dtype.itemsize, dtype.itemsize) > ROW_MAX:
        raise ValueError(f"PLY: rows of {vx.dtype.itemsize} / {dtype.itemsize} bytes (file / array); at most "
                         f"{ROW_MAX} are read on the device")
    return vx, dtype, field_table(vx.dtype, dtype, [(s, t) for t, s in pairs], "PLY read")


def decode(data, flavor: str = "3dgs", device="cuda"):
    """Ply3DGSFormat.read ("3dgs") or PlyCCFormat.read ("cc") on the device, `data` the file's bytes or its path.
    Binary little-endian PLY whose only element is `vertex`, with scalar properties.  Refused (ValueError): anything
    parse_ply_header refuses (ASCII or big-endian bodies, list properties), any other element (the reference keeps
    those in extra_elements), a body cut short, 2^31 rows or more, input or output rows wider than 1024 bytes, a vertex
    element without properties, and a cast gsx_ply_transcode does not reproduce."""
    from . import readers
    buf = readers.file_bytes(data)
    vx, dtype, table = read_plan(buf, flavor)
    raw = readers.upload(buf, device)
    rows = transcode(raw, vx.offset, vx.count, vx.dtype.itemsize, dtype.itemsize, table)
    return readers.Decoded(rows, dtype, None)


# ---------------------------------------------------------------------------------------------------------- writing
@dataclass
class Encoded:
    rows: torch.Tensor       # uint8 [n, dtype.itemsize] on the device
    dtype: np.dtype          # the writer's output dtype (packed, the PLY vertex properties in file order)

    def __len__(self):
        return self.rows.shape[0]

    def to_host(self) -> np.ndarray:
        """The output_data the reference writer hands to PlyElement.describe (one D2H)."""
        from .hostcopy import to_host
        return to_host(self.rows).reshape(-1).view(self.dtype)


def _device_rows(src, device):
    """(uint8 [n, itemsize] device rows, their dtype, DeviceRecords or None) of the three inputs encode takes."""
    from .readers import Decoded
    from .records import DeviceRecords
    if isinstance(src, DeviceRecords):
        dt = np.dtype([(f, "<f4") for f in src.names])
        return src.rows.contiguous().view(torch.uint8).view(len(src), dt.itemsize), dt, src
    if isinstance(src, Decoded):
        return src.rows, src.dtype, None
    if isinstance(src, np.ndarray) and src.dtype.names and src.ndim == 1:
        from .hostcopy import to_device
        a = np.ascontiguousarray(src)
        return to_device(a.view(np.uint8).reshape(len(a), a.dtype.itemsize), device), a.dtype, None
    raise ValueError("encode takes DeviceRecords, readers.Decoded or a 1-D structured NumPy array")


def last_nonzero_rest(rows: torch.Tensor, dt: np.dtype, records=None) -> int:
    """The writers' crop_sh scan (ply_3dgs.py:70-76, ply_cc.py:70-76): the largest i <= 44 whose f_rest_i holds a
    value != 0 (NaN included), -1 if none.  DeviceRecords: DeviceRecords.nonzero_columns; raw rows: the f_rest columns
    gathered with gsx_records_from_bytes, then the same gsx_codec_sh_mask."""
    from .records import DeviceRecords
    rest = [f"f_rest_{i}" for i in range(45) if f"f_rest_{i}" in (dt.names or ())]
    if not rest or rows.shape[0] == 0:
        return -1
    if records is None:
        sub = np.dtype({"names": rest, "formats": ["<f4"] * len(rest), "offsets": [dt.fields[f][1] for f in rest],
                        "itemsize": dt.itemsize})
        records = DeviceRecords.from_device_bytes(rows.reshape(-1), sub)
    hit = records.nonzero_columns(rest)
    return max((int(f.split("_")[-1]) for f in hit), default=-1)


def encode(src, flavor: str = "3dgs", crop_sh: bool = False, device="cuda") -> Encoded:
    """Ply3DGSFormat.write ("3dgs") or PlyCCFormat.write ("cc") up to PlyElement.describe, on the device.  src:
    DeviceRecords (its float32 rows), readers.Decoded (raw device rows and their dtype) or a 1-D structured NumPy array
    (its raw bytes, uploaded once).  Refused (ValueError): output field types plyfile does not write as listed (bool,
    8-byte integers, ...) or in non-native byte order, f_rest fields that are not float32, and rows wider than 1024
    bytes."""
    _check_flavor(flavor)
    rows, dt, records = _device_rows(src, device)
    check_write_input(dt)
    last = last_nonzero_rest(rows, dt, records) if crop_sh else None
    out, table = write_plan(dt, flavor, last)
    return Encoded(transcode(rows, 0, rows.shape[0], dt.itemsize, out.itemsize, table), out)


def check_write_input(dt: np.dtype) -> None:
    """encode's refusal of f_rest fields that are not float32 (the crop_sh scan reads them as float32)."""
    for f in dt.names:
        if f.startswith("f_rest_") and f in standard_order(False) and dt.fields[f][0] != np.dtype("<f4"):
            raise ValueError(f"PLY write: {f} is {dt.fields[f][0].str}, not float32")


def write_plan(dt: np.dtype, flavor: str, last_rest: int | None = None):
    """(output dtype, gsx_ply_transcode field table) of encode, on the host; ValueError for output fields of a type
    plyfile does not write as listed.  Every output field not in the table is a float32 zero column."""
    out, mapping = write_layout(dt, flavor, last_rest)
    if max(dt.itemsize, out.itemsize) > ROW_MAX:
        raise ValueError(f"PLY write: rows of {dt.itemsize} / {out.itemsize} bytes (records / file); at most "
                         f"{ROW_MAX} are written on the device")
    return out, field_table(dt, out, mapping, "PLY write")


def write_ply(path, enc: Encoded) -> None:
    """The file PlyData([PlyElement.describe(output_data, 'vertex')], byte_order='<').write(path) writes."""
    from .compressed_ply import ply_header
    from .hostcopy import to_host
    header, _ = ply_header([("vertex", len(enc), enc.dtype)])
    body = to_host(enc.rows)
    with open(path, "wb") as fh:
        fh.write(header)
        fh.write(memoryview(body).cast("B"))


def prepare_write(self, data, *args, **kwargs):
    """Ply3DGSFormat.write / PlyCCFormat.write (data, path, **kwargs) for gsx.dropin.install_writer, in the install
    option flavor: encode(data, crop_sh=...); returns the step that writes the file with write_ply.  Positional
    arguments and a non-empty extra_elements are refused, so the reference's write handles them."""
    if args:
        raise TypeError("PLY write on the device takes no positional arguments after path")
    if kwargs.get("extra_elements"):
        raise ValueError("PLY write on the device writes no extra_elements")
    enc = encode(data, self._gsx_options["write"]["flavor"], crop_sh=kwargs.get("crop_sh", False))
    return lambda path: write_ply(path, enc)

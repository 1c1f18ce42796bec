"""Device-resident splat records (SURVEY 8(f) items 2 and 4): the reference's structured array (structures.py:23-59,
all-float32 fields) as one row-major float32 matrix in HBM.  Upload once, extract the filter columns on the device,
gather the survivors on the device, one D2H at the end; plus the writers' elementwise attribute transforms."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

SH_C0 = 0.28209479177387814


def is_packed_f32(a: np.ndarray) -> bool:
    """True iff `a` is a structured array of float32 fields only, packed without padding (what DeviceRecords holds)."""
    dt = a.dtype
    if dt.names is None or dt.itemsize != 4 * len(dt.names):
        return False
    return all(dt.fields[n][0] == np.float32 and dt.fields[n][1] == 4 * i for i, n in enumerate(dt.names))


class DeviceRecords:
    def __init__(self, rows: torch.Tensor, names, dtype):
        self.rows, self.names, self.dtype = rows, tuple(names), dtype
        self.col = {n: i for i, n in enumerate(self.names)}

    @classmethod
    def from_structured(cls, a: np.ndarray, device="cuda"):
        if not is_packed_f32(a):
            raise ValueError("DeviceRecords needs a packed all-float32 structured array")
        flat = np.ascontiguousarray(a).view(np.float32).reshape(len(a), len(a.dtype.names))
        from .hostcopy import to_device
        return cls(to_device(flat, device), a.dtype.names, a.dtype)

    @classmethod
    def from_writer_input(cls, a: np.ndarray, device="cuda"):
        """Every float32 field of a writer's input `a`, whatever other fields it also carries (the converter adds
        red/green/blue u1 before the .splat / .ksplat / SOG writers, converter.py:244-253); the other fields are
        dropped.  Packed float32 records go up as from_structured does; any other layout is uploaded as raw rows once
        and its float32 fields gathered on the device (gsx_records_from_bytes)."""
        if is_packed_f32(a):
            return cls.from_structured(a, device)
        dt = a.dtype
        names = [n for n in (dt.names or ()) if dt.fields[n][0] == np.dtype("<f4")]
        if a.ndim != 1 or not names:
            raise ValueError("DeviceRecords needs a 1-D structured array with float32 fields")
        from .hostcopy import to_device
        a = np.ascontiguousarray(a)
        return cls.from_device_bytes(to_device(a.view(np.uint8).reshape(-1), device), dt)

    @classmethod
    def from_device_bytes(cls, raw: torch.Tensor, dt: np.dtype):
        """The float32 fields of structured rows of dtype `dt` already on the device (`raw`: their bytes, contiguous),
        gathered on the device (gsx_records_from_bytes); the other fields are dropped."""
        names = [n for n in (dt.names or ()) if dt.fields[n][0] == np.dtype("<f4")]
        if not names:
            raise ValueError("DeviceRecords needs a structured dtype with float32 fields")
        n = raw.numel() // dt.itemsize
        rows = torch.empty((n, len(names)), dtype=torch.float32, device=raw.device)
        offs = (C.c_int32 * len(names))(*[dt.fields[f][1] for f in names])
        with torch.cuda.device(raw.device):
            check(lib.gsx_records_from_bytes(_ptr(raw), n, dt.itemsize, offs, len(names), _ptr(rows), _stream()),
                  "gsx_records_from_bytes")
        return cls(rows, names, np.dtype([(f, "<f4") for f in names]))

    def __len__(self):
        return self.rows.shape[0]

    @property
    def F(self):
        return self.rows.shape[1]

    def xyz_opacity(self):
        """np.column_stack((x, y, z)) and v['opacity'] (None if the field is absent), on the device."""
        n = len(self)
        xyz = torch.empty((n, 3), dtype=torch.float32, device=self.rows.device)
        has_op = "opacity" in self.col
        op = torch.empty(n, dtype=torch.float32, device=self.rows.device) if has_op else None
        check(lib.gsx_records_extract_xyz_opacity(_ptr(self.rows), n, self.F, self.col["x"], self.col["y"], self.col["z"],
                                                  self.col.get("opacity", 0), _ptr(xyz), _ptr(op), _stream()),
              "gsx_records_extract_xyz_opacity")
        return xyz, op

    def gather(self, idx: torch.Tensor) -> "DeviceRecords":
        """rows[idx] (idx: device int32, the surviving row indices in ascending order)."""
        idx = idx.to(device=self.rows.device, dtype=torch.int32).contiguous()
        out = torch.empty((idx.numel(), self.F), dtype=torch.float32, device=self.rows.device)
        check(lib.gsx_records_gather_rows(_ptr(self.rows), _ptr(idx), idx.numel(), self.F, _ptr(out), _stream()),
              "gsx_records_gather_rows")
        return DeviceRecords(out, self.names, self.dtype)

    def to_host(self) -> np.ndarray:
        """The structured array the writers consume (one D2H)."""
        from .hostcopy import to_host
        flat = to_host(self.rows)
        return flat.reshape(-1).view(self.dtype)

    # ---- elementwise attribute transforms of the writers
    def color_rgba8(self, scale: float = SH_C0) -> torch.Tensor:
        """uint8 [n,4]: clip((0.5 + scale*f_dc_i)*255).astype(u8), clip(sigmoid(opacity)*255).astype(u8)
        (formats/splat.py:131-144, ksplat.py:464-468; scale=0.15 is spz.py:131's colour scale)."""
        n = len(self)
        out = torch.empty((n, 4), dtype=torch.uint8, device=self.rows.device)
        check(lib.gsx_records_color_rgba8(_ptr(self.rows), n, self.F, self.col["f_dc_0"], self.col["f_dc_1"],
                                          self.col["f_dc_2"], self.col["opacity"], float(np.float32(scale)), _ptr(out),
                                          _stream()), "gsx_records_color_rgba8")
        return out

    def scale_exp(self) -> torch.Tensor:
        """float32 [n,3] = exp(scale_0..2) (formats/splat.py:108, ksplat.py:447)."""
        n = len(self)
        out = torch.empty((n, 3), dtype=torch.float32, device=self.rows.device)
        check(lib.gsx_records_scale_exp(_ptr(self.rows), n, self.F, self.col["scale_0"], self.col["scale_1"],
                                        self.col["scale_2"], _ptr(out), _stream()), "gsx_records_scale_exp")
        return out

    def nonzero_columns(self, names) -> set:
        """The fields among `names` (at most 45) that hold a value != 0, NaN included: np.any(a[f] != 0) for each, in
        one pass over the rows (the input of the writers' SH-degree rules)."""
        names = [f for f in names if f in self.col]
        if not names or len(self) == 0:
            return set()
        from .hostcopy import to_host
        mask = torch.empty(1, dtype=torch.int64, device=self.rows.device)
        cols = (C.c_int32 * len(names))(*[self.col[f] for f in names])
        check(lib.gsx_codec_sh_mask(_ptr(self.rows), len(self), self.F, cols, len(names), _ptr(mask), _stream()),
              "gsx_codec_sh_mask")
        m = int(to_host(mask).view(np.uint64)[0])
        return {f for k, f in enumerate(names) if m >> k & 1}

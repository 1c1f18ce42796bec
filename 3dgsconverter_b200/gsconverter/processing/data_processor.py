"""Drop-in for ``gsconverter/processing/data_processor.py``: the filter API on a NumPy structured
array, with every keep-mask computed by libgsx.so on the GPU.

Public surface and behaviour follow the reference (data_processor.py:7-354): each filter rebinds
``self.data`` to the compacted array and returns it; slider formulas (:17-28, :125-134), early-outs
and console messages are preserved.  Host-only helpers (RGB from SH, SH capping, auto-bbox report)
are plain NumPy and stay on the host (SURVEY §2.1 "OUT").

Working set: the columns the filters read (xyz, opacity) are uploaded once and stay in HBM across the
chain (gsx.pipeline.FilterChain); the 248-byte records are gathered on the host with the surviving row
indices.  With ``DataProcessor.defer_compaction = True`` (what ``gsx.dropin.patch(defer=True)`` sets
for converter.py, which ignores the filters' return values and reads ``processor.data`` once,
converter.py:259) that host gather happens ONCE, when ``.data`` is read, and the filters return None.

Constraint of the cached working set: the xyz / opacity columns are uploaded when the first filter runs and stay
in HBM; in-place edits of ``dp.data['x']`` (etc.) BETWEEN two filters are not seen by the later filter -- assign
``dp.data = new_array`` (the setter drops the device copy) or call ``dp.invalidate()`` after such an edit.  The
reference re-reads ``self.data`` in every filter; converter.py never edits coordinates between filters.

No CPU fallback: if the CUDA backend is unavailable the filters raise instead of silently running
the reference's SciPy path (whose mask the reference computes and then discards -- SURVEY F5).
"""
from __future__ import annotations

import os

import numpy as np

from ..utils.utility_functions import debug_print, status_print

_SH_C0 = 0.28209479177387814


def _require_backend():
    from .gpu_ops import HAS_TAICHI
    if not HAS_TAICHI:
        raise RuntimeError("gsx: no CUDA device available and CPU fallback is disabled by design")


class DataProcessor:
    defer_compaction = os.environ.get("GSX_DEFER_COMPACTION", "0") == "1"
    # SURVEY 8(f)2: keep the WHOLE records (all 62 float32 fields) in HBM: one upload, survivors gathered on the
    # device, one D2H when `.data` is read -- instead of fancy-indexing 248 bytes per splat on one CPU thread.
    device_records = os.environ.get("GSX_DEVICE_RECORDS", "0") == "1"

    def __init__(self, data):
        self._data = data
        self._chain = None      # device-resident working set (gsx.pipeline.FilterChain)
        self._pending = False   # host records not yet gathered with the chain's surviving indices
        self._records = None    # gsx.records.DeviceRecords (device_records mode)

    # ------------------------------------------------------------------ host records, lazily compacted
    @property
    def data(self):
        if self._pending:
            if self._records is not None:
                if self._chain.idx is not None:
                    self._records = self._records.gather(self._chain.idx)
                self._data = self._records.to_host()
            else:
                from gsx import hostrows
                self._data = hostrows.take_rows(self._data, self._chain.indices())   # vertices[mask], threaded
            self._chain.rebase()
            self._pending = False
        return self._data

    @data.setter
    def data(self, value):
        self._data = value
        self._chain = None
        self._records = None
        self._pending = False

    def invalidate(self):
        """Drop the device-resident columns (call after editing coordinates / opacity of ``.data`` in place)."""
        _ = self.data          # gathers pending survivors first
        self._chain = None
        self._records = None

    def _working_set(self):
        _require_backend()
        if self._chain is None:
            from gsx.pipeline import FilterChain
            v = self._data
            if self.device_records:
                from gsx import records
                if records.is_packed_f32(v):
                    self._records = records.DeviceRecords.from_structured(v)
                    xyz, op = self._records.xyz_opacity()
                    self._chain = FilterChain(xyz, op)
                    return self._chain
            from gsx import hostrows
            xyz, op = hostrows.xyz_opacity(v)        # np.column_stack((x, y, z)), v["opacity"] -- threaded
            self._chain = FilterChain(xyz, op)
        return self._chain

    def _count(self):
        return self._chain.count if self._chain is not None else len(self._data)

    def _done(self):
        self._pending = True
        return None if self.defer_compaction else self.data

    # ------------------------------------------------------------------ density (:11-117)
    def apply_density_filter(self, voxel_size=1.0, threshold_percentage=0.32, sensitivity=None,
                             keep_multicluster=False):
        debug_print("[DEBUG] Executing 'apply_density_filter' function...")
        if not isinstance(self._data, np.ndarray):
            raise TypeError("self.data must be a numpy structured array.")
        _require_backend()   # imports .gpu_ops first: that module puts GSX_HOME on sys.path (file-copy integration)
        from gsx import density
        if sensitivity is not None:
            voxel_size, threshold_percentage = density.slider(sensitivity)
        debug_print(f"Density Filter Params: Voxel={voxel_size:.4f}, Thresh={threshold_percentage:.4f}%, "
                    f"MultiCluster={keep_multicluster}")
        before = self._count()
        if before == 0:
            status_print("Warning: Density filter removed all points.")
            return self.data
        chain = self._working_set()
        kept, info = chain.density(voxel_size, threshold_percentage, None, keep_multicluster)
        debug_print(f"[DEBUG] Found {info['voxels']} unique voxels.")
        if info["dense"] == 0 or info["clusters"] == 0:
            status_print("Warning: Density filter removed all points.")
            return self._done()
        status_print(f"Density Filter: Kept {info['clusters']} clusters (largest: {info['max_len']} voxels).")
        status_print(f"After density filter, retained {kept} out of {before} vertices.")
        return self._done()

    # ------------------------------------------------------------------ SOR (:119-182)
    def remove_flyers(self, k=25, threshold_factor=10.5, chunk_size=50000, intensity=None):
        debug_print("[DEBUG] Executing 'remove_flyers' function...")
        if not isinstance(self._data, np.ndarray):
            raise TypeError("self.data must be a numpy structured array.")
        if intensity is not None:  # :125-134
            k = int(10 + (intensity - 1) * (40 / 9))
            threshold_factor = 20.0 - (intensity - 1) * (17.0 / 9)
        debug_print(f"SOR Filter (Remove Flyers) Params: K={k}, Sigma={threshold_factor:.2f}")
        num_points = self._count()
        _require_backend()
        status_print("[SOR] Determining outliers on GPU (gsx / sm_90a)...")
        if num_points == 0:
            return self.data
        chain = self._working_set()
        kept = chain.sor(int(k), float(threshold_factor), hash_mode=os.environ.get("GSX_SOR_HASH", "i32wrap"),
                         semantics=os.environ.get("GSX_SOR_SEMANTICS", "taichi"))
        status_print(f"After removing flyers (GPU), retained {kept} out of {num_points} vertices.")
        return self._done()

    # ------------------------------------------------------------------ alpha (:184-213)
    def apply_alpha_filter(self, min_opacity_u8):
        debug_print(f"[DEBUG] Executing 'apply_alpha_filter' with min={min_opacity_u8}")
        if "opacity" not in self._data.dtype.names:
            status_print("Warning: No opacity channel found. Alpha filter skipped.")
            return
        limit = min_opacity_u8
        if limit <= 0:
            return
        if limit >= 255:
            self.data = self.data[:0]
            return
        original_len = self._count()
        if original_len:
            self._working_set().alpha(limit)
        status_print(f"Alpha Filter (min {limit}): Retained {self._count()} out of {original_len} splats.")
        return self._done()

    # ------------------------------------------------------------------ bbox (:215-231)
    def crop_by_bbox(self, min_x, min_y, min_z, max_x, max_y, max_z):
        if self._count():
            self._working_set().crop_by_bbox(min_x, min_y, min_z, max_x, max_y, max_z)
        debug_print(f"[DEBUG] Number of vertices after cropping: {self._count()}")
        status_print(f"After cropping, retained {self._count()} vertices.")
        return self._done()

    # ------------------------------------------------------------------ host-only helpers (:233-354)
    @staticmethod
    def _dc_triplet(vertices):
        for prefix in ("", "scalar_", "scalar_scalar_"):
            names = [f"{prefix}f_dc_{i}" for i in range(3)]
            if names[0] in vertices.dtype.names:
                return np.column_stack([vertices[nm] for nm in names])
        return None

    @staticmethod
    def _compute_rgb_from_sh(vertices):
        """sRGB u8 from the SH DC term: clip(0.5 + C0*dc, 0, 1) ** (1/2.2) * 255."""
        dc = DataProcessor._dc_triplet(vertices)
        if dc is None:
            return None
        lin = np.clip(0.5 + dc * _SH_C0, 0.0, 1.0)
        return (np.power(lin, 1.0 / 2.2) * 255).astype(np.uint8)

    def add_rgb_from_sh(self):
        debug_print("[DEBUG] Executing 'add_rgb_from_sh' function...")
        cur = self.data
        names = cur.dtype.names
        if "red" in names:
            return
        if "f_dc_0" not in names and "scalar_f_dc_0" not in names:
            debug_print("[DEBUG] No SH DC components found, cannot compute RGB.")
            return
        rgb = self._compute_rgb_from_sh(cur)
        if rgb is None:
            return
        out = np.empty(len(cur), dtype=cur.dtype.descr + [("red", "u1"), ("green", "u1"), ("blue", "u1")])
        for nm in names:
            out[nm] = cur[nm]
        out["red"], out["green"], out["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
        chain = self._chain            # same rows: the device working set stays valid
        self.data = out
        self._chain = chain

    def cap_sh_degree(self, degree):
        """Zero the f_rest_* coefficients above `degree` (0 -> all 45, 1 -> from 9, 2 -> from 24)."""
        if degree is None or degree >= 3:
            return self.data
        cur = self.data
        first = {0: 0, 1: 9, 2: 24}.get(degree, 45)
        for i in range(first, 45):
            nm = f"f_rest_{i}"
            if nm in cur.dtype.names:
                cur[nm] = 0.0
        return cur

    def apply_auto_bbox(self):
        """Report the tight bounding box of what is left (no change to the data)."""
        cur = self.data
        if len(cur) == 0:
            status_print("Auto-BBox: No points remaining. Bounding box is undefined.")
            return
        lo = [np.min(cur[a]) for a in "xyz"]
        hi = [np.max(cur[a]) for a in "xyz"]
        status_print(f"Auto-BBox Applied: [{lo[0]:.4f}, {lo[1]:.4f}, {lo[2]:.4f}] to "
                     f"[{hi[0]:.4f}, {hi[1]:.4f}, {hi[2]:.4f}]")

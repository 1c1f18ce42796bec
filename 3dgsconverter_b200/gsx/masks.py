"""bbox / alpha keep-masks on device buffers (data_processor.py:184-231)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ._abi import lib, check, f32x
from ._abi import _ptr, _stream
from .sor import _check_xyz


def bbox_mask(xyz: torch.Tensor, min_x, min_y, min_z, max_x, max_y, max_z) -> torch.Tensor:
    """keep <=> f32(lo) <= v <= f32(hi) on every axis (NumPy-2 weak-scalar semantics, SURVEY A.4)."""
    _check_xyz(xyz)
    n = xyz.shape[0]
    mask = torch.empty(n, dtype=torch.uint8, device=xyz.device)
    lohi = f32x(*[np.float32(v) for v in (min_x, min_y, min_z, max_x, max_y, max_z)])
    check(lib.gsx_bbox_mask(_ptr(xyz), n, lohi, _ptr(mask), _stream()), "gsx_bbox_mask")
    return mask.view(torch.bool)


def alpha_logit_threshold(min_opacity_u8) -> float:
    """data_processor.py:203-205, evaluated by NumPy itself: np.log's float64 SIMD loop may differ from
    libm by an ulp, and the reference's threshold is whatever NumPy returns on this host.
    (gsx_alpha_logit_threshold is the libm version for non-Python FFI clients.)"""
    a = np.clip(min_opacity_u8 / 255.0, 1e-6, 1.0 - 1e-6)
    return float(np.log(a / (1.0 - a)))


def alpha_mask(opacity: torch.Tensor, min_opacity_u8) -> torch.Tensor:
    """keep <=> (double)opacity >= logit(clip(min/255)) (data_processor.py:199-208); the early-outs
    (<=0 keep all, >=255 keep none) are the caller's, as in the reference."""
    if not opacity.is_cuda or opacity.dtype != torch.float32 or not opacity.is_contiguous():
        raise ValueError("opacity must be a contiguous float32 CUDA tensor")
    n = opacity.numel()
    mask = torch.empty(n, dtype=torch.uint8, device=opacity.device)
    check(lib.gsx_alpha_mask(_ptr(opacity), n, alpha_logit_threshold(min_opacity_u8), _ptr(mask), _stream()),
          "gsx_alpha_mask")
    return mask.view(torch.bool)

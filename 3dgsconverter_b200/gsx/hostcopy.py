"""NumPy array <-> CUDA tensor through libgsx's staged copies (gsx_copy_h2d / gsx_copy_d2h, csrc/gsx_hostcopy.cu):
pageable host buffers are moved by several host threads through pinned chunks, so the PCIe link stays busy
(torch's `.to(device)` / `.cpu()` of a pageable array run on one thread)."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

_NP2T = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64, np.dtype(np.int32): torch.int32,
         np.dtype(np.int64): torch.int64, np.dtype(np.uint8): torch.uint8, np.dtype(np.bool_): torch.bool}
_T2NP = {v: k for k, v in _NP2T.items()}


def to_device(a: np.ndarray, device="cuda") -> torch.Tensor:
    """Contiguous copy of `a` on `device` (made current for the duration of the copy: libgsx's copy streams and
    pinned chunks belong to the current device)."""
    a = np.ascontiguousarray(a)
    t = torch.empty(a.shape, dtype=_NP2T[a.dtype], device=device)
    if a.nbytes:
        with torch.cuda.device(t.device):
            check(lib.gsx_copy_h2d(_ptr(t), a.ctypes.data, a.nbytes, _stream()), "gsx_copy_h2d")
    return t


def to_host(t: torch.Tensor) -> np.ndarray:
    """NumPy copy of a CUDA tensor (blocks until the data is there)."""
    t = t.contiguous()
    out = np.empty(tuple(t.shape), dtype=_T2NP[t.dtype])
    if out.nbytes:
        with torch.cuda.device(t.device):
            check(lib.gsx_copy_d2h(out.ctypes.data, _ptr(t), out.nbytes, _stream()), "gsx_copy_d2h")
    return out


# a new bytes object of n uninitialised bytes, and the address of its contents: the C API's way to fill a bytes object
# before anyone else holds it, so that a device buffer lands in the returned bytes without a second host copy
_new_bytes = ctypes.pythonapi.PyBytes_FromStringAndSize
_new_bytes.restype, _new_bytes.argtypes = ctypes.py_object, [ctypes.c_void_p, ctypes.c_ssize_t]
_bytes_at = ctypes.pythonapi.PyBytes_AsString
_bytes_at.restype, _bytes_at.argtypes = ctypes.c_void_p, [ctypes.py_object]


def to_bytes(t: torch.Tensor) -> bytes:
    """The bytes of a uint8 CUDA tensor, copied once, straight into the returned object (blocks until they are
    there)."""
    t = t.contiguous()
    if t.dtype != torch.uint8:
        raise ValueError(f"to_bytes needs a uint8 tensor, not {t.dtype}")
    out = _new_bytes(None, t.numel())
    if t.numel():
        with torch.cuda.device(t.device):
            check(lib.gsx_copy_d2h(_bytes_at(out), _ptr(t), t.numel(), _stream()), "gsx_copy_d2h")
    return out

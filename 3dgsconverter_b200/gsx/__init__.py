"""gsx -- host side of the H100-native filtering / clustering backend.

Python here is plumbing only: torch tensors are the device-buffer container and the
stream source; all compute is in libgsx.so (hand-written sm_90a CUDA behind a C ABI).
"""
from . import _abi  # noqa: F401  (raises ImportError if libgsx.so has not been built)
from ._abi import GsxError  # noqa: F401

__all__ = ["GsxError", "backend_available"]


def backend_available() -> bool:
    """True iff a CUDA device is usable (libgsx.so itself is mandatory at import)."""
    try:
        import torch
        return bool(torch.cuda.is_available())
    except Exception:
        return False

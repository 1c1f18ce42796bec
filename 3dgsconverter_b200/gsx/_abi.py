"""ctypes binding of libgsx.so, derived from include/gsx.h.  No torch types cross this boundary.

The library is built in-tree by ``__graft_entry__.build()`` (3dgsconverter_b200/lib/libgsx.so).
There is NO CPU fallback: if the shared object or the header is missing this module raises at import.
Every ``gsx_*`` prototype of the header becomes one ctypes signature: pointers are ``c_void_p`` (a
``const char*`` return is ``c_char_p``), scalars map through ``_SCALARS``; any other type is an ImportError.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent.parent
LIB_PATH = Path(os.environ.get("GSX_LIB", _PKG / "lib" / "libgsx.so"))


class GsxError(RuntimeError):
    """A libgsx entry point returned a non-zero status."""


if not LIB_PATH.exists():
    raise ImportError(
        f"libgsx.so not found at {LIB_PATH}: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(nvcc, sm_90a).  gsx has no CPU fallback.")

lib = C.CDLL(str(LIB_PATH))

_HEADER = _PKG.parent / "include" / "gsx.h"
_SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "int64_t": C.c_int64, "long long": C.c_int64,
            "uint64_t": C.c_uint64, "float": C.c_float, "double": C.c_double, "void": None}


def _ctype(decl: str, proto: str, ret: bool = False):
    """ctypes type of a return type, or of a parameter declaration (type and name)."""
    if "*" in decl:
        return C.c_char_p if ret and decl.split() == ["const", "char*"] else C.c_void_p
    words = [w for w in decl.split() if w != "const"]
    t = " ".join(words if ret else words[:-1])
    if t not in _SCALARS:
        raise ImportError(f"include/gsx.h: no ctypes type for '{decl.strip()}' in {proto}")
    return _SCALARS[t]


def _signatures(header: Path) -> dict:
    """{name: (restype, argtypes)} of every gsx_* prototype of include/gsx.h."""
    if not header.exists():
        raise ImportError(f"{header} not found: gsx binds libgsx.so from its header")
    src = re.sub(r"/\*.*?\*/", " ", header.read_text(), flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    sigs = {}
    for ret, name, args in re.findall(r"([A-Za-z_][\w\s]*?\**)\s*\b(gsx_\w+)\s*\(([^)]*)\)\s*;", src):
        params = [a for a in args.split(",") if a.strip() and a.strip() != "void"]
        sigs[name] = (_ctype(ret, name, ret=True), [_ctype(a, name) for a in params])
    return sigs


_SIGS = _signatures(_HEADER)

for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)  # AttributeError here == a symbol declared in gsx.h is missing
    _fn.restype = _res
    _fn.argtypes = _args

HASH_MODES = {"i32wrap": 0, "i64": 1}
KM_ASSIGN = {"auto": 0, "strict": 1, "tensor": 3}


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib.gsx_last_error().decode("utf-8", "replace")
        raise GsxError(f"{what or 'gsx'} failed (status {rc}): {msg}")


def f32x(*vals):
    return (C.c_float * len(vals))(*[float(v) for v in vals])


def _stream():
    """The current torch CUDA stream, as the ``void* stream`` of an entry point."""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    """A tensor's data pointer (NULL for None)."""
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)

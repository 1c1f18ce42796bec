"""CPU: libgsx.so loads without a GPU and exports every function include/gsx.h declares."""
import ctypes as C
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def declared_functions():
    src = (ROOT / "include" / "gsx.h").read_text()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gsx_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(gsx_lib):
    names = declared_functions()
    assert len(names) >= 20
    for name in names:
        assert hasattr(gsx_lib, name), f"{name} declared in include/gsx.h but not exported by libgsx.so"


def test_binding_covers_header(gsx_lib):
    """The ctypes signatures are parsed from include/gsx.h: one per declared function, each from the known types."""
    from gsx import _abi
    assert set(declared_functions()) == set(_abi._SIGS), "gsx/_abi.py and include/gsx.h disagree"
    known = set(_abi._SCALARS.values()) | {C.c_void_p, C.c_char_p}
    for name, (res, args) in _abi._SIGS.items():
        fn = getattr(gsx_lib, name)
        assert fn.restype is res and fn.argtypes == args, name
        assert res in known and all(a in known - {None, C.c_char_p} for a in args), name
    sig = _abi._SIGS
    assert sig["gsx_last_error"] == (C.c_char_p, [])
    assert sig["gsx_sor_cell_size"] == (C.c_float, [C.c_void_p, C.c_int64])
    assert sig["gsx_alpha_logit_threshold"] == (C.c_double, [C.c_double])
    assert sig["gsx_density_voxel_range"][0] is None
    assert sig["gsx_webp_emit"][1][4] is C.c_uint64
    assert len(sig["gsx_sog_decode"][1]) == 12


def test_void_pointer_takes_every_argument_form():
    """Where the old hand-typed table had POINTER(...) parameters, c_void_p accepts what the product passes there."""
    import numpy as np
    a = np.arange(3, dtype=np.float32)
    for arg in ((C.c_int32 * 4)(1, 2, 3, 4), (C.c_float * 3)(1, 2, 3), (C.c_void_p * 6)(), C.byref(C.c_int64()),
                a.ctypes.data_as(C.POINTER(C.c_float)), a.ctypes.data_as(C.c_void_p), None):
        C.c_void_p.from_param(arg)
    assert C.c_void_p.from_param(None) is None


def test_no_torch_types_in_abi():
    src = (ROOT / "include" / "gsx.h").read_text()
    assert "torch" not in src and "at::" not in src and "std::" not in src


def test_host_helpers_run_without_gpu(gsx_lib):
    assert gsx_lib.gsx_version() >= 100
    assert isinstance(gsx_lib.gsx_last_error(), bytes)
    assert gsx_lib.gsx_mean_std_workspace_bytes(10_000_000) > 0


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under 3dgsconverter_b200/ may reference it."""
    for p in (ROOT / "3dgsconverter_b200").rglob("*"):
        if p.suffix in (".py", ".cu", ".cuh", ".h") and p.is_file():
            txt = p.read_text()
            assert "import oracle" not in txt and "from oracle" not in txt and "liborc" not in txt, p

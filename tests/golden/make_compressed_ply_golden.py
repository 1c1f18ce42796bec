"""Generate tests/golden/g10_reference_compressed_ply_small.npz: the reference's own CompressedPlyFormat.write
(formats/compressed_ply.py:126-250) run on the two inputs of compressed_ply_oracle.golden_inputs().

    python tests/golden/make_compressed_ply_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

`plyfile` is stubbed and `_write_ply_file` is intercepted, so no file is written: the script stores the Morton order
and the three arrays the writer hands to `_write_ply_file`.  `numpy.argsort` is forced to kind="stable" for the call:
the reference's default argsort leaves the order of equal Morton codes unspecified, and gsx orders them by ascending
index.  The script asserts that the oracle reproduces the reference's arrays bit for bit before it writes the file.
"""
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import compressed_ply_oracle as cpo  # noqa: E402


def import_reference_writer(ref_root):
    """gsconverter.formats.compressed_ply loaded by file path, without the package's other imports."""
    ref = Path(ref_root) / "gsconverter"
    for name, path in (("gsconverter", ref), ("gsconverter.formats", ref / "formats"), ("gsconverter.utils", ref / "utils")):
        m = types.ModuleType(name)
        m.__path__ = [str(path)]
        sys.modules[name] = m
    uf = types.ModuleType("gsconverter.utils.utility_functions")
    uf.debug_print = lambda *a, **k: None
    sys.modules[uf.__name__] = uf
    ply = types.ModuleType("plyfile")
    ply.PlyData = ply.PlyElement = object
    sys.modules["plyfile"] = ply
    spec = importlib.util.spec_from_file_location("gsconverter.formats.compressed_ply", ref / "formats" / "compressed_ply.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod.CompressedPlyFormat


def run_reference(cls, a):
    got = {}

    class Capture(cls):
        def _sort_morton_order(self, data, indices):
            super()._sort_morton_order(data, indices)
            got["order"] = indices.astype(np.int32)

        def _write_ply_file(self, path, chunk_data, vertex_data, sh_data):
            got["arrays"] = (chunk_data, vertex_data, sh_data)

    argsort = np.argsort
    np.argsort = lambda x, *args, **kw: argsort(x, kind="stable")
    try:
        Capture().write(a, "unused.ply")
    finally:
        np.argsort = argsort
    return got["order"], got["arrays"]


def main(ref_root):
    cls = import_reference_writer(ref_root)
    out = {}
    for tag, a in cpo.golden_inputs().items():
        order, (chunk, vertex, sh) = run_reference(cls, a)
        cpo.assert_packed_equal(cpo.encode(a, order), (chunk, vertex, sh))
        assert np.array_equal(cpo.encode(a, order)[1], vertex)     # the oracle's alpha bytes are NumPy's own
        out[f"{tag}_input_sha256"] = np.array(cpo.digest(a))
        out[f"{tag}_order"] = order
        out[f"{tag}_chunk"] = chunk
        out[f"{tag}_vertex"] = vertex
        out[f"{tag}_sh_names"] = np.array(sh.dtype.names if sh is not None else (), dtype="U16")
        if sh is not None:
            out[f"{tag}_sh"] = sh
    np.savez_compressed(HERE / "g10_reference_compressed_ply_small.npz", **out)


if __name__ == "__main__":
    main(sys.argv[1])

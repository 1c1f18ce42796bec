"""Generate tests/golden/g12_reference_splat_codecs_small.npz: the reference's own SplatFormat.write,
KSplatFormat.write and SpzFormat.write (formats/splat.py, ksplat.py, spz.py) run on the inputs of
splat_codecs_oracle.golden_inputs().

    python tests/golden/make_splat_codecs_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

The three writer modules are loaded by file path with `debug_print` / `status_print` stubbed and write into a temporary
directory.  `numpy.argsort` is forced to kind="stable" for the .splat call (the reference's default argsort leaves the
order of equal metrics unspecified; gsx keeps ascending index).  The SPZ file is stored gunzipped, because the gzip
header carries the mtime.  Every file is stored as its SHA-256 and length (plus the bytes themselves for the small
inputs); the script asserts that the oracle reproduces each one byte for byte before it writes the fixture.
An input the reference refuses is recorded with the exception's type name instead.
"""
import gzip
import importlib.util
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import splat_codecs_oracle as sco  # noqa: E402

KEEP_BYTES = 4 << 10   # files up to this size are stored whole


def import_reference_writers(ref_root):
    ref = Path(ref_root) / "gsconverter"
    for name, path in (("gsconverter", ref), ("gsconverter.formats", ref / "formats"), ("gsconverter.utils", ref / "utils")):
        m = types.ModuleType(name)
        m.__path__ = [str(path)]
        sys.modules[name] = m
    uf = types.ModuleType("gsconverter.utils.utility_functions")
    uf.debug_print = uf.status_print = lambda *a, **k: None
    sys.modules[uf.__name__] = uf
    out = {}
    for mod, cls in (("structures", None), ("formats.base", None), ("formats.splat", "SplatFormat"),
                     ("formats.ksplat", "KSplatFormat"), ("formats.spz", "SpzFormat")):
        spec = importlib.util.spec_from_file_location(f"gsconverter.{mod}", ref / (mod.replace(".", "/") + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = m
        spec.loader.exec_module(m)
        if cls:
            out[cls] = getattr(m, cls)
    return out


def run(write, path):
    """The file `write(path)` produces, or the name of the exception it raises."""
    try:
        write(path)
    except Exception as e:  # noqa: BLE001
        return type(e).__name__
    return Path(path).read_bytes()


def main(ref_root):
    cls = import_reference_writers(ref_root)
    out = {}
    argsort = np.argsort
    with tempfile.TemporaryDirectory() as tmp:
        f = Path(tmp) / "out"
        for tag, a in sco.golden_inputs().items():
            out[f"{tag}_input_sha256"] = np.array(sco.digest(a))
            files = {}
            for case in sco.KSPLAT_CASES:
                lv, shl, bs, blk = case
                files[sco.ksplat_tag(case)] = (
                    run(lambda p: cls["KSplatFormat"]().write(a, p, lv, sh_level=shl, bucket_size=bs, block_size=blk), f),
                    lambda case=case: sco.ksplat_file(a, *case))
            got = run(lambda p: cls["SpzFormat"]().write(a, p, compression_level=1), f)
            files["spz"] = (gzip.decompress(got) if isinstance(got, bytes) else got, lambda a=a: sco.spz_payload(a))
            np.argsort = lambda x, *args, **kw: argsort(x, kind="stable")
            try:
                got = run(lambda p: cls["SplatFormat"]().write(a, p), f)
            finally:
                np.argsort = argsort
            files["splat"] = (got, lambda a=a: sco.splat_file(a))
            for name, (want, oracle) in files.items():
                key = f"{tag}_{name}"
                if isinstance(want, str):
                    try:
                        oracle()
                    except Exception as e:  # noqa: BLE001
                        assert type(e).__name__ == want, (key, e)
                    else:
                        raise AssertionError(f"{key}: the reference raises {want}, the oracle does not")
                    out[f"{key}_raises"] = np.array(want)
                    continue
                assert oracle() == want, f"{key}: the oracle differs from the reference"
                out[f"{key}_sha256"] = np.array(sco.digest(want))
                out[f"{key}_len"] = np.array(len(want))
                if len(want) <= KEEP_BYTES:
                    out[f"{key}_bytes"] = np.frombuffer(want, np.uint8)
                print(key, len(want), "OK")
    np.savez_compressed(HERE / "g12_reference_splat_codecs_small.npz", **out)


if __name__ == "__main__":
    main(sys.argv[1])

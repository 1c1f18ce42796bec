"""Generate tests/golden/g16_reference_parquet_small.npz: the reference's own ParquetFormat.write
(formats/parquet.py:59-112, pandas' to_parquet with pyarrow) run on the inputs of parquet_oracle.golden_inputs().

    python tests/golden/make_parquet_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

formats/parquet.py is loaded by file path with `debug_print` / `status_print` stubbed (and plyfile stubbed for the
package's structures module) and writes into a temporary directory.  Each case stores its input (bytes and dtype
description) and the reference's file whole, or the exception's type name; the large case stores its row-group and
column-chunk facts and the digests of its table instead of the file.  tests/test_parquet_cpu.py checks the oracle's
file of every case against it.
"""
import importlib.util
import io
import json
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import parquet_oracle as po  # noqa: E402

OUT = HERE / "g16_reference_parquet_small.npz"


def import_reference_writer(ref_root):
    ref = Path(ref_root) / "gsconverter"
    for name, path in (("gsconverter", ref), ("gsconverter.formats", ref / "formats"), ("gsconverter.utils", ref / "utils")):
        m = types.ModuleType(name)
        m.__path__ = [str(path)]
        sys.modules[name] = m
    uf = types.ModuleType("gsconverter.utils.utility_functions")
    uf.debug_print = uf.status_print = lambda *a, **k: None
    sys.modules[uf.__name__] = uf
    sys.modules.setdefault("plyfile", types.ModuleType("plyfile"))
    for mod in ("structures", "formats.base", "formats.parquet"):
        full = f"gsconverter.{mod}"
        spec = importlib.util.spec_from_file_location(full, ref / (mod.replace(".", "/") + ".py"))
        m = importlib.util.module_from_spec(spec)
        sys.modules[full] = m
        spec.loader.exec_module(m)
    return sys.modules["gsconverter.formats.parquet"].ParquetFormat


def main(ref_root):
    import pyarrow.parquet as pq
    Fmt = import_reference_writer(ref_root)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, a in po.golden_inputs().items():
            out[f"{name}/dtype"] = np.frombuffer(json.dumps(a.dtype.descr).encode(), np.uint8)
            if name != po.LARGE:
                out[f"{name}/input"] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
            path = Path(tmp) / f"{name}.parquet"
            try:
                Fmt().write(a, str(path))
            except Exception as e:  # noqa: BLE001
                out[f"{name}/error"] = np.frombuffer(type(e).__name__.encode(), np.uint8)
                print(f"{name}: reference raises {type(e).__name__}")
                continue
            blob = path.read_bytes()
            if name == po.LARGE:
                t = pq.read_table(io.BytesIO(blob))
                facts = {"digest": po.table_digest(t), "chunks": po.chunk_facts(pq.read_metadata(io.BytesIO(blob))),
                         "size": len(blob)}
                out[f"{name}/facts"] = np.frombuffer(json.dumps(facts).encode(), np.uint8)
            else:
                out[f"{name}/file"] = np.frombuffer(blob, np.uint8)
            print(f"{name}: {len(a)} rows, {len(blob)} bytes")
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main(sys.argv[1])

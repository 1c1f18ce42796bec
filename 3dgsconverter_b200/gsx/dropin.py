"""Put the gsx backend behind an already-installed 3dgsconverter without touching its files.

    import gsx.dropin; gsx.dropin.patch()      # before running gsconverter.main / Converter

Replaces, in the *installed* ``gsconverter.processing`` package (converter.py:10,150 and
formats/sog.py:11 import from there):
  * ``gpu_ops.kmeans``, ``gpu_ops.filter_sor_gpu``, ``gpu_ops.HAS_TAICHI``
  * the ``DataProcessor`` class (same public surface; the filters run on libgsx and keep their
    working set in HBM; ``defer=True`` gathers the host records once, when ``.data`` is read)
and, when ``gsconverter.formats.compressed_ply`` imports, ``CompressedPlyFormat.write`` (Morton order, chunk bounds
and packing on the device, the file still written by the class's own ``_write_ply_file``; records gsx refuses go to
the original ``write``).  With ``patch(sog="device")`` also ``SogFormat.write`` (gsx.sog.encode: every texture,
codebook and the chunked SH palette built on the device; opt-in because its position bytes can differ from NumPy's
log by one count on a small fraction of the splats); ``patch(sog="device", sog_webp="device")`` also encodes its
WebP members on the device (gsx.webp: lossless VP8L that decodes to the same pixels, in gsx's bytes, not libwebp's).
With ``patch(codecs="device")`` also ``SplatFormat.write``,
``KSplatFormat.write`` and ``SpzFormat.write`` (gsx.splat / gsx.ksplat / gsx.spz: sort, bucket bounds and packing on the
device, gzip and the file on the host; records gsx refuses go to the original ``write``);
``patch(codecs="device", spz_gzip="device")`` also gzips the .spz payload on the device (gsx.deflate: a file that
decompresses to the same payload, in gsx's bytes, not zlib's).  With
``patch(readers="device")`` also the ``read`` of ``SplatFormat``, ``KSplatFormat``, ``SpzFormat`` and
``CompressedPlyFormat`` (gsx.splat / gsx.ksplat / gsx.spz / gsx.compressed_ply ``decode``: headers and gunzip on the
host, every splat decoded on the device, byte for byte as the reference readers; files gsx refuses go to the original
``read``).  With ``patch(sog_reader="device")`` also ``SogFormat.read`` (gsx.sog_reader.decode: ZIP, meta.json and
WebP on the host, the shN palette and every splat decoded on the device, byte for byte as the reference reader, its
palette indexing included; bundles gsx refuses go to the original ``read``); ``patch(sog_reader="device",
sog_reader_webp="device")`` also decodes the lossless WebP members on the device (gsx.webp_decode), so only their
compressed bytes cross PCIe.  With ``patch(ply="device")`` also the
``read`` and ``write`` of ``Ply3DGSFormat`` and ``PlyCCFormat`` (gsx.ply: header and field mapping on the host, the rows
transcoded on the device, byte for byte as the reference; files and records gsx refuses, and writes with
``extra_elements``, go to the original method).  With ``patch(parquet="device")`` also ``ParquetFormat.write``
(gsx.parquet: columns, statistics, dictionaries, pages and Snappy built on the device; a file that pyarrow and pandas
read as the same table, in gsx's bytes, not pyarrow's; records gsx refuses go to the original ``write``).  The parquet
reader stays on the host.
Host-only helpers and everything else of the reference stay as they are.
"""
from __future__ import annotations

import importlib
import importlib.util
import sys
from pathlib import Path

_HERE = Path(__file__).resolve().parent.parent


def _load_ours(modname: str, relpath: str):
    spec = importlib.util.spec_from_file_location(modname, _HERE / relpath,
                                                  submodule_search_locations=None)
    mod = importlib.util.module_from_spec(spec)
    return spec, mod


class _GsxCodebookKMeans:
    """Opt-in stand-in for the scikit-learn MiniBatchKMeans that formats/sog.py:561 runs on the flattened shN
    centroids (~737 k scalars -> 256): exact Lloyd on the GPU (gsx 1-D kernel), init = the same kind of draw
    gpu_ops.kmeans makes.  A different algorithm than MiniBatchKMeans (which is itself unseeded), so it is not the
    default; `patch(codebook="gpu")` installs it."""

    def __init__(self, n_clusters=8, n_init="auto", max_iter=20, **_):
        self.n_clusters, self.max_iter = int(n_clusters), int(max_iter)

    def fit(self, X):
        import numpy as np
        from gsx import kmeans as _km
        x = np.ascontiguousarray(X, dtype=np.float32).reshape(len(X), -1)
        k = min(self.n_clusters, len(x))
        init = x[np.random.choice(len(x), k, replace=False)]
        C, L = _km.kmeans_host(x, k, self.max_iter, init)
        self.cluster_centers_, self.labels_ = C, L
        return self


def patch(verbose: bool = False, defer: bool = True, codebook: str = "sklearn", require_cuda: bool = True,
          sog: str = "host", codecs: str = "host", readers: str = "host", sog_reader: str = "host", ply: str = "host",
          sog_webp: str = "host", spz_gzip: str = "host", sog_reader_webp: str = "host", parquet: str = "host"):
    """require_cuda: refuse (return False, leave the reference untouched) when no CUDA device is usable, so that a
    CPU-only host keeps the reference's own SciPy / scikit-learn paths (there is no CPU fallback inside gsx).
    sog: "host" keeps the reference's SogFormat.write (with the patched gpu_ops.kmeans and its batch-ahead);
    "device" replaces it with gsx.sog's device encoder (records gsx refuses go to the original write).
    sog_webp: with sog="device" only.  "host" writes the bundle's WebP members with Pillow, as the reference does;
    "device" encodes them from HBM with gsx.webp.  The files then hold gsx's lossless bytes rather than libwebp's
    (same pixels, a different size), so this chooses the output, not only the speed.
    codecs: "host" keeps the reference's .splat / .ksplat / .spz writers; "device" installs gsx's device writers on
    them (records gsx refuses go to the original write).
    spz_gzip: with codecs="device" only.  "host" gzips the .spz payload with gzip.compress, as the reference does;
    "device" compresses it in HBM with gsx.deflate and copies back only the file.  The file then holds gsx's DEFLATE
    bytes rather than zlib's (the same payload inside), so this chooses the output, not only the speed.
    readers: "host" keeps the reference's .splat / .ksplat / .spz / compressed PLY readers; "device" installs gsx's
    device readers on them (files gsx refuses go to the original read).
    sog_reader: "host" keeps the reference's SogFormat.read; "device" installs gsx.sog_reader's device reader on it
    (bundles gsx refuses go to the original read).
    sog_reader_webp: with sog_reader="device" only.  "host" decodes the bundle's WebP members with Pillow, as the
    reference does; "device" uploads their bytes and decodes the lossless ones on the device (gsx.webp_decode, pixel
    for pixel as Pillow; a member it refuses sends the bundle to the original read).
    ply: "host" keeps the reference's plain 3DGS and CloudCompare PLY read and write; "device" installs gsx.ply's device
    reader and writer on Ply3DGSFormat and PlyCCFormat (files and records gsx refuses go to the original method).
    parquet: "host" keeps the reference's ParquetFormat.write (pandas and pyarrow); "device" installs gsx.parquet's
    device writer on it (records gsx refuses go to the original write).  The file then holds gsx's bytes, the same
    table pyarrow writes, so this chooses the output, not only the speed."""
    if sog not in ("host", "device"):
        raise ValueError(f"sog must be 'host' or 'device', not {sog!r}")
    if sog_webp not in ("host", "device"):
        raise ValueError(f"sog_webp must be 'host' or 'device', not {sog_webp!r}")
    if sog_webp == "device" and sog != "device":
        raise ValueError("sog_webp='device' needs sog='device': the reference writer has no device textures to encode")
    if codecs not in ("host", "device"):
        raise ValueError(f"codecs must be 'host' or 'device', not {codecs!r}")
    if spz_gzip not in ("host", "device"):
        raise ValueError(f"spz_gzip must be 'host' or 'device', not {spz_gzip!r}")
    if spz_gzip == "device" and codecs != "device":
        raise ValueError("spz_gzip='device' needs codecs='device': the reference writer has no device payload to gzip")
    if readers not in ("host", "device"):
        raise ValueError(f"readers must be 'host' or 'device', not {readers!r}")
    if sog_reader not in ("host", "device"):
        raise ValueError(f"sog_reader must be 'host' or 'device', not {sog_reader!r}")
    if sog_reader_webp not in ("host", "device"):
        raise ValueError(f"sog_reader_webp must be 'host' or 'device', not {sog_reader_webp!r}")
    if sog_reader_webp == "device" and sog_reader != "device":
        raise ValueError("sog_reader_webp='device' needs sog_reader='device': the reference reader decodes on the host")
    if ply not in ("host", "device"):
        raise ValueError(f"ply must be 'host' or 'device', not {ply!r}")
    if parquet not in ("host", "device"):
        raise ValueError(f"parquet must be 'host' or 'device', not {parquet!r}")
    if require_cuda:
        from . import backend_available
        if not backend_available():
            if verbose:
                print("[gsx] no CUDA device: gsconverter.processing left unpatched")
            return False
    ref_gpu_ops = importlib.import_module("gsconverter.processing.gpu_ops")
    ref_dp = importlib.import_module("gsconverter.processing.data_processor")
    if getattr(ref_gpu_ops, "_GSX_PATCHED", False):
        return True
    # load our two modules under private names but with the reference's package as parent, so their
    # relative imports (..utils.utility_functions) resolve to the installed reference
    ours = {}
    for name, rel in (("gpu_ops", "gsconverter/processing/gpu_ops.py"),
                      ("data_processor", "gsconverter/processing/data_processor.py")):
        full = f"gsconverter.processing._gsx_{name}"
        spec = importlib.util.spec_from_file_location(full, _HERE / rel)
        mod = importlib.util.module_from_spec(spec)
        mod.__package__ = "gsconverter.processing"
        sys.modules[full] = mod
        ours[name] = (spec, mod)
    ours["gpu_ops"][0].loader.exec_module(ours["gpu_ops"][1])
    g = ours["gpu_ops"][1]
    ref_gpu_ops.kmeans = g.kmeans
    ref_gpu_ops.filter_sor_gpu = g.filter_sor_gpu
    ref_gpu_ops.HAS_TAICHI = g.HAS_TAICHI
    ref_gpu_ops._GSX_PATCHED = True
    # our data_processor does `from .gpu_ops import ...`: that now resolves to the patched reference module
    ours["data_processor"][0].loader.exec_module(ours["data_processor"][1])
    Ours = ours["data_processor"][1].DataProcessor
    # the whole class is replaced: the device-resident working set needs the `data` property
    Ours.defer_compaction = bool(defer)   # converter.py ignores the filters' return values (converter.py:194-259)
    ref_dp.DataProcessor = Ours
    proc_pkg = importlib.import_module("gsconverter.processing")
    proc_pkg.DataProcessor = Ours
    conv = sys.modules.get("gsconverter.converter")
    if conv is not None and hasattr(conv, "DataProcessor"):
        conv.DataProcessor = Ours
    ref_gpu_ops._gsx_module = g     # batch-ahead statistics: gpu_ops._gsx_module.batch_stats
    sog_mod = sys.modules.get("gsconverter.formats.sog")
    if sog_mod is None:
        try:
            sog_mod = importlib.import_module("gsconverter.formats.sog")
        except Exception:  # noqa: BLE001  (optional dependency of the writer missing: nothing to patch there)
            sog_mod = None
    if sog_mod is not None and codebook == "gpu" and hasattr(sog_mod, "MiniBatchKMeans"):
        sog_mod.MiniBatchKMeans = _GsxCodebookKMeans  # sog.py:561 -> exact 1-D Lloyd on the GPU
    if sog_mod is not None and sog == "device" and hasattr(sog_mod, "SogFormat"):
        from .sog import install as install_sog
        install_sog(sog_mod.SogFormat, webp=sog_webp)  # sog.py:249-639 -> textures and palette on the GPU
    if sog_mod is not None and sog_reader == "device" and hasattr(sog_mod, "SogFormat"):
        from .sog_reader import install_reader as install_sog_reader
        install_sog_reader(sog_mod.SogFormat, webp=sog_reader_webp)   # sog.py:23-247 -> palette and rows on the GPU
    cply = sys.modules.get("gsconverter.formats.compressed_ply")
    if cply is None:
        try:
            cply = importlib.import_module("gsconverter.formats.compressed_ply")
        except Exception:  # noqa: BLE001  (writer not importable: nothing to patch there)
            cply = None
    if cply is not None and hasattr(cply, "CompressedPlyFormat"):
        from .compressed_ply import install
        install(cply.CompressedPlyFormat)             # compressed_ply.py:126-250 -> packing on the GPU
    if codecs == "device":
        from . import ksplat, splat, spz
        for modname, clsname, ours in (("splat", "SplatFormat", splat), ("ksplat", "KSplatFormat", ksplat),
                                       ("spz", "SpzFormat", spz)):
            fmt = sys.modules.get(f"gsconverter.formats.{modname}")
            if fmt is None:
                try:
                    fmt = importlib.import_module(f"gsconverter.formats.{modname}")
                except Exception:  # noqa: BLE001  (writer not importable: nothing to patch there)
                    continue
            if hasattr(fmt, clsname):                 # splat.py:82-166, ksplat.py:319-544, spz.py:49-173
                if ours is spz:
                    ours.install(getattr(fmt, clsname), where=spz_gzip)
                else:
                    ours.install(getattr(fmt, clsname))
    if readers == "device":
        from . import compressed_ply, ksplat, splat, spz
        for modname, clsname, ours in (("splat", "SplatFormat", splat), ("ksplat", "KSplatFormat", ksplat),
                                       ("spz", "SpzFormat", spz), ("compressed_ply", "CompressedPlyFormat",
                                                                   compressed_ply)):
            fmt = sys.modules.get(f"gsconverter.formats.{modname}")
            if fmt is None:
                try:
                    fmt = importlib.import_module(f"gsconverter.formats.{modname}")
                except Exception:  # noqa: BLE001  (reader not importable: nothing to patch there)
                    continue
            if hasattr(fmt, clsname):
                ours.install_reader(getattr(fmt, clsname))   # splat.py:9-80, ksplat.py:29-317, spz.py:18-296,
                #                                               compressed_ply.py:14-123
    if ply == "device":
        from . import ply as gply
        for modname, clsname, flavor in (("ply_3dgs", "Ply3DGSFormat", "3dgs"), ("ply_cc", "PlyCCFormat", "cc")):
            fmt = sys.modules.get(f"gsconverter.formats.{modname}")
            if fmt is None:
                try:
                    fmt = importlib.import_module(f"gsconverter.formats.{modname}")
                except Exception:  # noqa: BLE001  (plyfile missing: nothing to patch there)
                    continue
            if hasattr(fmt, clsname):
                gply.install_reader(getattr(fmt, clsname), flavor)   # ply_3dgs.py:8-60, ply_cc.py:8-62
                gply.install(getattr(fmt, clsname), flavor)          # ply_3dgs.py:62-121, ply_cc.py:64-132
    if parquet == "device":
        fmt = sys.modules.get("gsconverter.formats.parquet")
        if fmt is None:
            try:
                fmt = importlib.import_module("gsconverter.formats.parquet")
            except Exception:  # noqa: BLE001  (pandas missing: nothing to patch there)
                fmt = None
        if fmt is not None and hasattr(fmt, "ParquetFormat"):
            from . import parquet as gpq
            gpq.install(fmt.ParquetFormat)                           # parquet.py:59-112
    if verbose:
        print("[gsx] gsconverter.processing patched: SOR / density / bbox / alpha / K-Means / compressed PLY packing "
              "run on libgsx.so")
    return True

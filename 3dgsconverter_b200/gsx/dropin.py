"""Put the gsx backend behind an already-installed 3dgsconverter without touching its files.

    import gsx.dropin; gsx.dropin.patch()      # before running gsconverter.main / Converter

Replaces, in the *installed* ``gsconverter.processing`` package (converter.py:10,150 and
formats/sog.py:11 import from there):
  * ``gpu_ops.kmeans``, ``gpu_ops.filter_sor_gpu``, ``gpu_ops.HAS_TAICHI``
  * the ``DataProcessor`` class (same public surface; the filters run on libgsx and keep their
    working set in HBM; ``defer=True`` gathers the host records once, when ``.data`` is read)
and installs gsx's device readers and writers on the reference's format classes:

  =======================  =====================  ==========================================================
  class                    read / write keyword   gsx
  =======================  =====================  ==========================================================
  ``SplatFormat``          readers / codecs       gsx.splat ``decode`` / ``prepare_write``
  ``KSplatFormat``         readers / codecs       gsx.ksplat
  ``SpzFormat``            readers / codecs       gsx.spz (``spz_gzip="device"``: gzip with gsx.deflate)
  ``CompressedPlyFormat``  readers / always       gsx.compressed_ply
  ``SogFormat``            sog_reader / sog       gsx.sog_reader / gsx.sog (``sog_reader_webp`` / ``sog_webp``)
  ``Ply3DGSFormat``        ply / ply              gsx.ply, flavour "3dgs"
  ``PlyCCFormat``          ply / ply              gsx.ply, flavour "cc"
  ``ParquetFormat``        -- / parquet           gsx.parquet (the reader stays on the host)
  =======================  =====================  ==========================================================

Each installed method (install_reader / install_writer) keeps the original as ``_gsx_reference_read`` /
``_gsx_reference_write``.  It runs gsx's device path, and anything gsx refuses or fails on goes to the original method
with the original arguments and the global NumPy RNG as it was on entry.  The compressed PLY writer is installed
whatever the keywords; every other class only with its keyword set to "device".
Host-only helpers and everything else of the reference stay as they are.
"""
from __future__ import annotations

import importlib
import importlib.util
import sys
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent.parent


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


def _install(cls, method: str, wrapper, options: dict) -> None:
    """cls.<method> = wrapper, the original kept once as cls._gsx_reference_<method>; options always replaced."""
    ref = f"_gsx_reference_{method}"
    if ref not in cls.__dict__:
        setattr(cls, ref, getattr(cls, method))
        setattr(cls, method, wrapper)
    cls._gsx_options = {**cls.__dict__.get("_gsx_options", {}), method: options}


def install_writer(cls, prepare, **options) -> None:
    """Make cls.write the device writer `prepare`, keeping the original as cls._gsx_reference_write; installing again
    changes only the options.  prepare(self, data, *args, **kwargs) does all the device work and all the refusing, and
    returns finish(path), which writes the file.  Anything prepare raises sends the call to the original write with the
    original arguments and the global NumPy RNG as it was on entry; an error writing the file propagates.  prepare
    reads `options` at call time as self._gsx_options["write"]."""
    def write(self, data, path, *args, **kwargs):
        state = np.random.get_state()
        try:
            finish = prepare(self, data, *args, **kwargs)
        except Exception:  # noqa: BLE001  (the reference's convention: exception => CPU path)
            np.random.set_state(state)
            return self._gsx_reference_write(data, path, *args, **kwargs)
        finish(path)

    _install(cls, "write", write, options)


def install_reader(cls, decode, after=None, **options) -> None:
    """Make cls.read the device reader `decode`, keeping the original as cls._gsx_reference_read; installing again
    changes only the options.  read(path) returns decode(path, **options).to_host(), with options read at call time,
    sets self.metadata when the decode has metadata, then runs after(self) if given.  Anything the decode raises sends
    the call to the original read with the original arguments and the global NumPy RNG as it was on entry."""
    def read(self, path, *args, **kwargs):
        state = np.random.get_state()
        try:
            dec = decode(path, **self._gsx_options["read"])
            out = dec.to_host()
        except Exception:  # noqa: BLE001  (the reference's convention: exception => CPU path)
            np.random.set_state(state)
            return self._gsx_reference_read(path, *args, **kwargs)
        if dec.metadata is not None:
            self.metadata = dec.metadata
        if after is not None:
            after(self)
        return out

    _install(cls, "read", read, options)


def _vertex_only(self) -> None:
    """What BaseFormat.__init__ leaves in extra_elements after reading a vertex-only PLY."""
    self.extra_elements = []


def _formats(kw: dict):
    """One row per reference class: (gsconverter.formats module, class, reader, writer).  Reader and writer are each
    None (left to the reference) or (the patch keyword that turns it on, None for always; the gsx function; the
    install options), the options taken from the patch keywords in `kw`."""
    from . import compressed_ply, ksplat, parquet, ply, sog, sog_reader, splat, spz
    return (
        ("splat", "SplatFormat", ("readers", splat.decode, {}), ("codecs", splat.prepare_write, {})),
        ("ksplat", "KSplatFormat", ("readers", ksplat.decode, {}), ("codecs", ksplat.prepare_write, {})),
        ("spz", "SpzFormat", ("readers", spz.decode, {}), ("codecs", spz.prepare_write, {"gzip": kw["spz_gzip"]})),
        ("compressed_ply", "CompressedPlyFormat", ("readers", compressed_ply.decode, {}),
         (None, compressed_ply.prepare_write, {})),
        ("sog", "SogFormat", ("sog_reader", sog_reader.decode, {"webp": kw["sog_reader_webp"]}),
         ("sog", sog.prepare_write, {"webp": kw["sog_webp"]})),
        ("ply_3dgs", "Ply3DGSFormat", ("ply", ply.decode, {"flavor": "3dgs", "after": _vertex_only}),
         ("ply", ply.prepare_write, {"flavor": "3dgs"})),
        ("ply_cc", "PlyCCFormat", ("ply", ply.decode, {"flavor": "cc", "after": _vertex_only}),
         ("ply", ply.prepare_write, {"flavor": "cc"})),
        ("parquet", "ParquetFormat", None, ("parquet", parquet.prepare_write, {})),
    )


# "X='device' needs Y='device'": the reference's own method has nothing on the device for X to work on
_NEEDS = (("sog_webp", "sog", "the reference writer has no device textures to encode"),
          ("spz_gzip", "codecs", "the reference writer has no device payload to gzip"),
          ("sog_reader_webp", "sog_reader", "the reference reader decodes on the host"))


def _format_class(module: str, name: str):
    """gsconverter.formats.<module>.<name>, or None when the module does not import (its optional dependency, such as
    plyfile, pandas or Pillow, is missing) or has no such class."""
    try:
        mod = importlib.import_module(f"gsconverter.formats.{module}")
    except Exception:  # noqa: BLE001  (nothing to patch there)
        return None
    return getattr(mod, name, None)


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
    kw = dict(sog=sog, codecs=codecs, readers=readers, sog_reader=sog_reader, ply=ply, sog_webp=sog_webp,
              spz_gzip=spz_gzip, sog_reader_webp=sog_reader_webp, parquet=parquet)
    for name, value in kw.items():
        if value not in ("host", "device"):
            raise ValueError(f"{name} must be 'host' or 'device', not {value!r}")
    for name, needs, why in _NEEDS:
        if kw[name] == "device" and kw[needs] != "device":
            raise ValueError(f"{name}='device' needs {needs}='device': {why}")
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
    if codebook == "gpu" and _format_class("sog", "MiniBatchKMeans") is not None:
        sys.modules["gsconverter.formats.sog"].MiniBatchKMeans = _GsxCodebookKMeans  # sog.py:561 -> 1-D Lloyd on the GPU
    for module, name, *sides in _formats(kw):
        for install, side in zip((install_reader, install_writer), sides):
            if side is None or (side[0] is not None and kw[side[0]] != "device"):
                continue
            cls = _format_class(module, name)
            if cls is not None:
                install(cls, side[1], **side[2])
    if verbose:
        print("[gsx] gsconverter.processing patched: SOR / density / bbox / alpha / K-Means / compressed PLY packing "
              "run on libgsx.so")
    return True

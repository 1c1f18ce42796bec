"""Generate tests/golden/g11_reference_sog_small.npz: the reference's own SogFormat.write (formats/sog.py:249-639) run
on the inputs of sog_oracle.golden_inputs().

    python tests/golden/make_sog_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

The writer is loaded by file path with its package imports stubbed.  Three things are replaced:
  * Image: frombytes/save write the raw RGBA bytes into the ZIP, so every member is read back without WebP;
  * gpu_ops.kmeans: the oracle's Lloyd (oracle.kmeans_lloyd) with the reference's own init draw (gpu_ops.py:182) --
    the K-Means pinned to the reference's kernel source by g4 / g6;
  * MiniBatchKMeans: the real scikit-learn class, recording its input, its output and the RNG state around the fit
    (its fit is deterministic given the global NumPy RNG, which np.random.seed sets before every write).
The script stores the inputs' SHA-256, every texture (the two large 'mixed' palettes as SHA-256 and shape; members
identical to an earlier case's as a reference to it), meta.json, the codebook fit (for replay) and the RNG states,
and asserts that sog_oracle reproduces the textures, meta and final RNG state bit for bit before it writes the file.
"""
import importlib.util
import json
import sys
import tempfile
import types
import zipfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE.parent), str(HERE.parent.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import sog_oracle as so  # noqa: E402

SIZES = []


class _Img:
    def __init__(self, data, size):
        self.data, self.size = data, size

    def save(self, bio, **kwargs):
        assert kwargs == {"format": "WEBP", "lossless": True, "quality": 100, "method": 1}, kwargs
        bio.write(self.data)


class RawImage:
    @staticmethod
    def frombytes(mode, size, data):
        assert mode == "RGBA"
        SIZES.append(size)
        return _Img(data, size)


def import_reference_writer(ref_root):
    ref = Path(ref_root) / "gsconverter"
    for name, path in (("gsconverter", ref), ("gsconverter.formats", ref / "formats"),
                       ("gsconverter.utils", ref / "utils"), ("gsconverter.processing", ref / "processing")):
        m = types.ModuleType(name)
        m.__path__ = [str(path)]
        sys.modules[name] = m
    uf = types.ModuleType("gsconverter.utils.utility_functions")
    uf.debug_print = uf.status_print = lambda *a, **k: None
    base = types.ModuleType("gsconverter.formats.base")
    base.BaseFormat = object
    st = types.ModuleType("gsconverter.structures")
    st.GaussianStruct = None
    go = types.ModuleType("gsconverter.processing.gpu_ops")
    go.HAS_TAICHI = True
    go.kmeans = lambda data, k, max_iter=10, **kw: so.oracle_kmeans(data, k, max_iter)
    for m in (uf, base, st, go):
        sys.modules[m.__name__] = m
    sys.modules["gsconverter.processing"].gpu_ops = go
    spec = importlib.util.spec_from_file_location("gsconverter.formats.sog", ref / "formats" / "sog.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    mod.Image = RawImage
    return mod


def run_reference(mod, a, level, seed):
    rec = {}

    class Recording(mod.MiniBatchKMeans):
        def fit(self, X, y=None, sample_weight=None):
            rec["input_sha256"] = so.digest(np.ascontiguousarray(X, np.float32))
            rec["before"] = np.random.get_state()
            super().fit(X, y, sample_weight)
            rec["after"] = np.random.get_state()
            rec["centres"] = self.cluster_centers_.copy()
            return self

    mod.MiniBatchKMeans = Recording
    SIZES.clear()
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp) / "out.sog"
        np.random.seed(seed)
        mod.SogFormat().write(a, str(path), compression_level=level)
        end = np.random.get_state()
        with zipfile.ZipFile(path) as zf:
            members = zf.namelist()
            assert members[-1] == "meta.json" and all(i.compress_type == zipfile.ZIP_STORED for i in zf.infolist())
            tex = {}
            for name, (w, h) in zip(members[:-1], SIZES):
                tex[name] = np.frombuffer(zf.read(name), np.uint8).reshape(h, w, 4)
            meta_json = zf.read("meta.json").decode()
    return tex, meta_json, rec, end


def main(ref_root):
    mod = import_reference_writer(ref_root)
    out, written = {}, {}
    for case, (a, level, seed) in so.golden_inputs().items():
        tex, meta_json, rec, end = run_reference(mod, a, level, seed)
        written[case] = tex
        out[f"{case}_input_sha256"] = np.array(so.digest(a))
        out[f"{case}_members"] = np.array(list(tex), dtype="U24")
        so.store_case(out, case, tex)
        out[f"{case}_meta"] = np.array(meta_json)
        out[f"{case}_rng_end"] = so.rng_pack(end)
        if rec:
            out[f"{case}_fit_input_sha256"] = np.array(rec["input_sha256"])
            out[f"{case}_fit_centres"] = rec["centres"]
            out[f"{case}_rng_before_fit"] = so.rng_pack(rec["before"])
            out[f"{case}_rng_after_fit"] = so.rng_pack(rec["after"])
        # the oracle, fed the recorded codebook fit, reproduces every byte, meta.json and the final RNG state
        z = {k[len(case) + 1:]: v for k, v in out.items() if k.startswith(case + "_")}
        z = {f"{case}_{k}": v for k, v in z.items()}
        np.random.seed(seed)
        got, meta, _ = so.encode(a, level, codebook_fit=so.replay_fit(z, case) if rec else None)
        assert so.rng_equal(np.random.get_state(), end), case
        assert list(got) == list(tex) and all(np.array_equal(got[k], tex[k]) for k in tex), case
        assert json.dumps(meta) == meta_json, case
        print(case, {k: v.shape for k, v in tex.items()})
    np.savez_compressed(HERE / "g11_reference_sog_small.npz", **out)
    z = np.load(HERE / "g11_reference_sog_small.npz")            # the stored form reads back as what was written
    for case, tex in written.items():
        back, _ = so.golden_case(z, case)
        assert list(back) == list(tex), case
        for name, t in tex.items():
            if isinstance(back[name], so.Hashed):
                so.check_hashed(t, back[name], name)
            else:
                assert np.array_equal(back[name], t), (case, name)


if __name__ == "__main__":
    main(sys.argv[1])

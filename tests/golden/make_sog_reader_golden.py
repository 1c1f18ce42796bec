"""Generate tests/golden/g14_reference_sog_reader_small.npz: the reference's own SogFormat.read (formats/sog.py:23-247)
on small .sog bundles.

    python tests/golden/make_sog_reader_golden.py REFERENCE_ROOT     (a checkout of francescofugazzi/3dgsconverter)

sog.py and structures.py are loaded by file path, their package imports stubbed as make_sog_golden.py stubs them,
with the real Pillow Image and the real GaussianStruct.  Inputs: bundles of the reference writer itself (its K-Means
calls on the oracle's Lloyd, real Pillow) at SH degrees 0-3, levels 0 and 7 and 1 to 3 000 splats (a palette of 2 048 entries); hand-built
bundles (every u16 position code, degenerate and non-finite bounds, every quaternion and opacity byte, short
codebooks, palettes of 1, 64, 65 and 200 entries at every band count, members wider or narrower than the writer's
textures, RGB-mode members, custom member names, no splats); and malformed bundles.  Each case stores the bundle's
bytes, then the reader's result (length, SHA-256 and dtype of the array's bytes) or the name of the exception it
raises, and `expect`: "ok" where gsx decodes the bundle, "refuse" where it raises ValueError.  The script asserts that
sog_reader_oracle.py reproduces every case before it writes the fixture.
"""
import importlib.util
import io
import json
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE), str(HERE.parent), str(HERE.parent.parent), str(HERE.parent.parent / "3dgsconverter_b200")]
import sog_reader_oracle as sro  # noqa: E402
from make_sog_golden import import_reference_writer  # noqa: E402

OUT = HERE / "g14_reference_sog_reader_small.npz"


def import_reference_sog(ref_root):
    """SogFormat with the real Pillow Image and the real GaussianStruct (structures.py by file path)."""
    from PIL import Image
    mod = import_reference_writer(ref_root)
    spec = importlib.util.spec_from_file_location("gsconverter.structures",
                                                  Path(ref_root) / "gsconverter" / "structures.py")
    st = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = st
    spec.loader.exec_module(st)
    mod.GaussianStruct = st.GaussianStruct
    mod.Image = Image
    return mod


# ---------------------------------------------------------------------------------------------------- hand-built
def rgba(pixels, width=None, fill=255):
    """uint8 [h, w, 4] holding `pixels` ([k, 4]) row-major, padded with `fill`; width defaults to sqrt-ish."""
    pixels = np.asarray(pixels, np.uint8).reshape(-1, 4)
    k = max(len(pixels), 1)
    w = width or int(np.ceil(np.sqrt(k)))
    h = -(-k // w)
    out = np.full((h * w, 4), fill, np.uint8)
    out[:len(pixels)] = pixels
    return out.reshape(h, w, 4)


def base_meta(n, mins=(-2.0, -1.0, 0.5), maxs=(3.0, 2.5, 4.0), scb=None, ccb=None, names=None):
    rng = np.random.default_rng(n + 1)
    names = names or {}
    scb = sorted(np.round(rng.normal(-4, 1, 256), 1).tolist()) if scb is None else scb
    ccb = sorted(np.round(rng.normal(0, 1, 256), 1).tolist()) if ccb is None else ccb
    return {"version": 2, "asset": {"generator": "gsconverter-sog"}, "count": n,
            "means": {"mins": list(mins), "maxs": list(maxs),
                      "files": [names.get("means_l", "means_l.webp"), names.get("means_u", "means_u.webp")]},
            "scales": {"codebook": scb, "files": [names.get("scales", "scales.webp")]},
            "quats": {"files": [names.get("quats", "quats.webp")]},
            "sh0": {"codebook": ccb, "files": [names.get("sh0", "sh0.webp")]}}


def random_textures(n, seed, alpha_quats=True):
    """Per-splat RGBA pixels [n, 4] of every main member, random bytes (quaternion alpha in 252 .. 255)."""
    rng = np.random.default_rng(seed)
    t = {k: rng.integers(0, 256, (n, 4), dtype=np.uint8) for k in ("means_l", "means_u", "quats", "scales", "sh0")}
    if alpha_quats:
        t["quats"][:, 3] = rng.integers(252, 256, n)
    return t


def plain_textures(n):
    """Per-splat RGBA pixels [n, 4] of every main member, the same pixel for every splat."""
    px = {"means_l": (0, 0, 0, 255), "means_u": (0, 0, 0, 255), "quats": (128, 128, 128, 252),
          "scales": (1, 2, 3, 255), "sh0": (4, 5, 6, 200)}
    return {k: np.tile(np.array(v, np.uint8), (n, 1)) for k, v in px.items()}


def add_shn(meta, tex, n, bands, P, seed, cb_len=256, names=None):
    rng = np.random.default_rng(seed)
    coeffs = sro.COEFFS[bands]
    w_c, h_c = 64 * coeffs, -(-P // 64)
    names = names or ("shN_centroids.webp", "shN_labels.webp")
    meta["shN"] = {"count": P, "bands": bands, "codebook": sorted(np.round(rng.normal(0, 0.3, cb_len), 3).tolist()),
                   "files": list(names)}
    # the writer's layout: P * C pixels of indices, then padding (255, or the last entry of a short codebook)
    cent = np.full((max(w_c * h_c, 1), 4), min(255, cb_len - 1), np.uint8)
    cent[:P * (coeffs // 3)] = rng.integers(0, cb_len, (P * (coeffs // 3), 4), dtype=np.uint8)
    cent[:, 3] = 255
    tex["centroids"] = cent.reshape(max(h_c, 1), max(w_c, 1), 4) if w_c else cent.reshape(1, 1, 4)
    lab = np.zeros((n, 4), np.uint8)
    labels = rng.integers(0, P, n)
    lab[:, 0], lab[:, 1], lab[:, 3] = labels & 0xff, labels >> 8, 255
    tex["labels"] = lab


ROLE_FILES = {"means_l": "means_l.webp", "means_u": "means_u.webp", "quats": "quats.webp", "scales": "scales.webp",
              "sh0": "sh0.webp", "centroids": "shN_centroids.webp", "labels": "shN_labels.webp"}


def bundle(meta, tex, width=None, modes=None, raw_meta=None, extra=None, drop=()):
    """Bytes of a ZIP_STORED bundle: each role's pixels as a lossless WebP under the name meta gives it."""
    modes = modes or {}
    names = {"means_l": meta["means"]["files"][0], "means_u": meta["means"]["files"][1],
             "quats": meta["quats"]["files"][0], "scales": meta["scales"]["files"][0], "sh0": meta["sh0"]["files"][0]}
    if "shN" in meta and isinstance(meta["shN"].get("files"), list):
        names["centroids"], names["labels"] = meta["shN"]["files"][:2]
    members = {}
    for role, px in tex.items():
        if role in drop:
            continue
        img = px if px.ndim == 3 else rgba(px, width)
        members[names[role]] = sro.webp(img, modes.get(role, "RGBA"))
    members.update(extra or {})
    return sro.zip_bundle(members, meta, raw_meta)


def write_sog_bundle(meta, tex, width):
    """The same bundle through gsx.sog.write_sog (standard member names, writer's member order)."""
    from gsx.sog import write_sog
    t = {ROLE_FILES[r]: (px if px.ndim == 3 else rgba(px, width)) for r, px in tex.items()}
    with tempfile.TemporaryDirectory() as tmp:
        p = Path(tmp) / "b.sog"
        write_sog(p, t, meta)
        return p.read_bytes()


def hand_cases():
    out = {}
    # every u16 code on x (y and z rolled), texture 256 x 256
    n = 65536
    t = random_textures(n, 1)
    codes = np.arange(n, dtype=np.uint32)
    for ch, sh in enumerate((0, 1, 2)):
        c = np.roll(codes, 977 * sh)
        t["means_l"][:, ch], t["means_u"][:, ch] = c & 0xff, c >> 8
    t["means_l"][:, 3] = t["means_u"][:, 3] = 255
    for r in ("quats", "scales", "sh0"):
        t[r][:] = (252, 7, 3, 200)
    out["pos_all_codes"] = (write_sog_bundle(base_meta(n, mins=(-9.5, -0.25, 0.0), maxs=(8.0, 12.0, 1e-3)), t, 256),
                            "ok")
    # degenerate and non-finite bounds
    n = 256
    for tag, mins, maxs in (("equal", (1.5, -2.0, 0.0), (1.5, -2.0, 0.0)), ("negative", (-9.0, -7.0, -30.0),
                                                                            (-1.0, -6.5, -29.0)),
                            ("inf", (-np.inf, 0.0, -np.inf), (np.inf, np.inf, 1.0)),
                            ("nan", (np.nan, 0.0, 1.0), (1.0, np.nan, np.nan)), ("huge", (-800.0, 0.0, 700.0),
                                                                                  (800.0, 710.0, 720.0))):
        t = plain_textures(n)
        t["means_l"][:, :3], t["means_u"][:, :3] = random_textures(n, 2)["means_l"][:, :3], np.arange(n)[:, None] // 2
        t["means_l"][:4, :3], t["means_u"][:4, :3] = [[0] * 3, [255] * 3, [0] * 3, [255] * 3], \
            [[0] * 3, [255] * 3, [128] * 3, [127] * 3]
        out[f"pos_{tag}"] = (bundle(base_meta(n, mins, maxs), t), "ok")
    # every quaternion byte triple component and alphas 252 .. 255 and others
    t = plain_textures(256 * 12)
    b = np.arange(256 * 12) % 256
    t["quats"][:, 0], t["quats"][:, 1], t["quats"][:, 2] = b, (b * 7 + 3) % 256, (b * 13 + 5) % 256
    t["quats"][:, 3] = np.repeat([252, 253, 254, 255, 0, 251, 1, 128, 256 - 4, 253, 252, 255], 256)[:len(b)]
    out["quats_bytes"] = (bundle(base_meta(len(b)), t), "ok")
    # every opacity byte
    t = random_textures(256, 4)
    t["sh0"][:, 3] = np.arange(256)
    out["opacity_bytes"] = (bundle(base_meta(256), t), "ok")
    # short codebooks with in-range indices
    t = random_textures(500, 5)
    t["scales"][:, :3] %= 10
    t["sh0"][:, :3] %= 3
    m = base_meta(500, scb=[-5.0, -4.0, -3.5, -3.0, -2.0, -1.5, -1.0, 0.0, 1.0, 1e30], ccb=[-1.0, 0.0, 0.5])
    add_shn(m, t, 500, 2, 70, 6, cb_len=5)
    out["short_codebooks"] = (bundle(m, t), "ok")
    # palettes of 1, 64, 65 and 200 entries at every band count
    for bands in (0, 1, 2, 3):
        for P in (1, 64, 65, 200):
            n = 100
            t = random_textures(n, 10 * bands + P)
            m = base_meta(n)
            add_shn(m, t, n, bands, P, 100 * bands + P)
            fn = write_sog_bundle if bands else bundle
            out[f"palette_b{bands}_p{P}"] = (fn(m, t, 12) if bands else fn(m, t), "ok")
    # members wider or narrower than the writer's texture (the reader indexes flat pixels)
    t = random_textures(100, 7)
    m = base_meta(100)
    add_shn(m, t, 100, 1, 30, 8)
    tex = {r: (rgba(px, {"means_l": 100, "means_u": 3, "quats": 7, "scales": 101, "sh0": 1, "labels": 50}[r])
               if r != "centroids" else px) for r, px in t.items()}
    out["member_widths"] = (bundle(m, tex), "ok")
    # RGB-mode members: all-255 alpha (opens as RGB) and members saved as RGB
    t = random_textures(400, 9)
    for r in ("means_l", "means_u", "scales"):
        t[r][:, 3] = 255
    out["rgb_members"] = (bundle(base_meta(400), t, modes={"quats": "RGB", "sh0": "RGB"}), "ok")
    # custom member names, one file read for two roles
    t = random_textures(200, 10)
    names = {"means_l": "pos/low.webp", "means_u": "pos/high.webp", "quats": "q", "scales": "shared.webp",
             "sh0": "shared.webp"}
    m = base_meta(200, names=names)
    t["sh0"] = t["scales"]
    add_shn(m, t, 200, 3, 90, 11, names=("cent.webp", "lab.webp"))
    out["custom_names"] = (bundle(m, t), "ok")
    # no splats
    t = {r: np.zeros((0, 4), np.uint8) for r in ("means_l", "means_u", "quats", "scales", "sh0")}
    out["count0"] = (bundle(base_meta(0), {r: rgba(px) for r, px in t.items()}), "ok")
    t0 = dict(t)
    m = base_meta(0)
    add_shn(m, t0, 0, 1, 3, 12)
    t0 = {r: (rgba(px) if px.ndim == 2 else px) for r, px in t0.items()}
    out["count0_shn"] = (bundle(m, t0), "ok")
    # refusals
    good_t = random_textures(16, 13)
    good_m = base_meta(16)
    add_shn(good_m, good_t, 16, 1, 4, 14)

    def variant(edit=None, tex_edit=None, **kw):
        m, tx = json.loads(json.dumps(good_m)), {k: v.copy() for k, v in good_t.items()}
        if edit:
            edit(m)
        if tex_edit:
            tex_edit(tx)
        return bundle(m, tx, **kw)

    out["refuse_not_zip"] = (b"PK\x03\x04 this is not a zip" + bytes(64), "refuse")
    out["refuse_no_meta"] = (sro.zip_bundle({"means_l.webp": sro.webp(rgba(good_t["means_l"]))}, None), "refuse")
    out["refuse_bad_json"] = (variant(raw_meta=b"{not json"), "refuse")
    out["refuse_missing_member"] = (variant(drop=("quats",)), "refuse")
    out["refuse_not_image"] = (variant(drop=("sh0",), extra={"sh0.webp": b"RIFF\x00\x00\x00\x00WEBPnope"}), "refuse")
    out["refuse_count_float"] = (variant(lambda m: m.update(count=16.0)), "refuse")
    out["refuse_count_negative"] = (variant(lambda m: m.update(count=-1)), "refuse")
    out["refuse_count_string"] = (variant(lambda m: m.update(count="16")), "refuse")
    out["refuse_two_mins"] = (variant(lambda m: m["means"].update(mins=[0.0, 1.0])), "refuse")
    out["refuse_too_small"] = (variant(lambda m: m.update(count=17)), "refuse")
    out["refuse_centroids_small"] = (variant(lambda m: m["shN"].update(count=130)), "refuse")
    out["refuse_shn_no_bands"] = (variant(lambda m: m["shN"].pop("bands")), "refuse")
    out["refuse_shn_no_count"] = (variant(lambda m: m["shN"].pop("count")), "refuse")
    out["refuse_shn_count0"] = (variant(lambda m: m["shN"].update(count=0)), "refuse")
    out["refuse_shn_count_negative"] = (variant(lambda m: m["shN"].update(count=-3)), "refuse")
    out["refuse_bands4"] = (variant(lambda m: m["shN"].update(bands=4)), "refuse")
    for bands in (-1, -3):   # the reference accepts these through negative list indexing (45 and 9 coefficients)
        t = random_textures(16, 15)
        m = base_meta(16)
        add_shn(m, t, 16, {-1: 3, -3: 1}[bands], 4, 16)
        m["shN"]["bands"] = bands
        out[f"refuse_bands{bands}"] = (bundle(m, t), "refuse")

    def oob(role, ch, v):
        def f(tx):
            tx[role][7, ch] = v
        return f
    out["refuse_scales_oob"] = (variant(lambda m: m["scales"].update(codebook=m["scales"]["codebook"][:200]),
                                        oob("scales", 1, 200)), "refuse")
    out["refuse_sh0_oob"] = (variant(lambda m: m["sh0"].update(codebook=m["sh0"]["codebook"][:9]),
                                     oob("sh0", 2, 9)), "refuse")
    out["refuse_shn_codebook_oob"] = (variant(lambda m: m["shN"].update(codebook=m["shN"]["codebook"][:100])), "refuse")
    out["refuse_label_oob"] = (variant(tex_edit=oob("labels", 0, 4)), "refuse")
    out["refuse_empty_codebook"] = (variant(lambda m: m["scales"].update(codebook=[])), "refuse")
    return out


def writer_cases(mod):
    """Bundles of the reference writer itself: real Pillow, the oracle's Lloyd for gpu_ops.kmeans."""
    from gsx import synth
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        p = Path(tmp) / "w.sog"
        for n, deg, level in ((1, 0, 0), (300, 0, 0), (300, 1, 0), (300, 2, 7), (300, 3, 0), (3_000, 1, 7)):
            a = synth.structured(n, "mixed", sh_degree=deg)
            np.random.seed(n + deg + level)
            mod.SogFormat().write(a, str(p), compression_level=level)
            out[f"writer_n{n}_d{deg}_l{level}"] = (p.read_bytes(), "ok")
    return out


def main(ref_root):
    mod = import_reference_sog(ref_root)
    cases = writer_cases(mod)
    cases.update(hand_cases())
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp) / "in.sog"
        for name, (blob, expect) in cases.items():
            path.write_bytes(blob)
            out[f"{name}_file"] = np.frombuffer(blob, np.uint8)
            try:
                with np.errstate(all="ignore"):
                    got = mod.SogFormat().read(str(path))
            except Exception as e:  # noqa: BLE001
                out[f"{name}_raises"] = np.array(type(e).__name__)
                expect = "refuse"                              # where the reference raises, gsx refuses
                try:
                    sro.read(blob)
                except Exception as o:  # noqa: BLE001
                    assert type(o).__name__ == type(e).__name__, f"{name}: oracle raises {o!r}, reference {e!r}"
                else:
                    raise AssertionError(f"{name}: the reference raises {e!r}, the oracle does not")
            else:
                b = np.ascontiguousarray(got).tobytes()
                out[f"{name}_len"] = np.array(len(b))
                out[f"{name}_sha256"] = np.array(sro.digest(b))
                out[f"{name}_dtype"] = np.array(str(got.dtype.descr))
                want = sro.read(blob)
                assert sro.digest(np.ascontiguousarray(want).tobytes()) == sro.digest(b), f"{name}: the oracle differs"
                assert str(want.dtype.descr) == str(got.dtype.descr), name
            out[f"{name}_expect"] = np.array(expect)
            try:
                sro.decode(blob)
            except ValueError:
                assert expect == "refuse", f"{name}: the oracle refuses a bundle gsx decodes"
            else:
                assert expect == "ok", f"{name}: the oracle decodes a bundle gsx refuses"
            print(name, expect, len(blob), str(out.get(f"{name}_raises", "")))
    np.savez_compressed(OUT, **out)
    print(OUT, OUT.stat().st_size)


if __name__ == "__main__":
    main(sys.argv[1])

"""CPU: the NumPy SOG reader oracle against the reference reader's own results (g14), meta.json and ZIP parsing, the
host tables, the refusals gsx.sog_reader raises before any device work, and the quaternion rule the kernel uses
against the reference's NumPy expression over every byte triple."""
import io
import json
import sys
import zipfile
from pathlib import Path

import numpy as np
import pytest

import sog_reader_oracle as sro

GOLDEN = Path(__file__).resolve().parent / "golden" / "g14_reference_sog_reader_small.npz"

# refused on the device by the kernels' index checks, not before the upload
KERNEL_REFUSALS = {"refuse_scales_oob", "refuse_sh0_oob", "refuse_shn_codebook_oob", "refuse_label_oob",
                   "refuse_empty_codebook"}


def golden_cases():
    z = np.load(GOLDEN)
    return sorted(k[: -len("_file")] for k in z.files if k.endswith("_file"))


def blob_of(z, case) -> bytes:
    return z[f"{case}_file"].tobytes()


@pytest.mark.parametrize("case", golden_cases())
def test_oracle_reproduces_reference_golden(case):
    z = np.load(GOLDEN)
    blob = blob_of(z, case)
    if f"{case}_raises" in z.files:   # the oracle's plain read raises what the reference raised
        with pytest.raises(Exception) as e:
            sro.read(blob)
        assert type(e.value).__name__ == str(z[f"{case}_raises"])
    if str(z[f"{case}_expect"]) == "refuse":
        with pytest.raises(ValueError):
            sro.decode(blob)
        if f"{case}_sha256" not in z.files:
            return
        a = sro.read(blob)            # accepted by the reference, refused by gsx
    else:
        a = sro.decode(blob)
    b = np.ascontiguousarray(a).tobytes()
    assert len(b) == int(z[f"{case}_len"]) and sro.digest(b) == str(z[f"{case}_sha256"])
    assert str(a.dtype.descr) == str(z[f"{case}_dtype"])


def test_golden_covers_the_edge_cases():
    z = np.load(GOLDEN)
    cases = golden_cases()
    ok = [c for c in cases if str(z[f"{c}_expect"]) == "ok"]
    assert len(ok) >= 30 and sum(c.startswith("writer_") for c in ok) == 6
    raises = {str(z[f"{c}_raises"]) for c in cases if f"{c}_raises" in z.files}
    assert {"KeyError", "IndexError", "ValueError", "TypeError", "UnidentifiedImageError"} <= raises
    for c in ("refuse_bands-1", "refuse_bands-3"):   # the reference accepts negative bands; gsx refuses them
        assert f"{c}_sha256" in z.files and str(z[f"{c}_expect"]) == "refuse"
    meta = json.loads(zipfile.ZipFile(io.BytesIO(blob_of(z, "writer_n3000_d1_l7"))).read("meta.json"))
    assert meta["shN"]["count"] > 64 and meta["shN"]["bands"] == 1     # the reader's palette indexing matters
    assert sro.digest(np.ascontiguousarray(sro.decode(blob_of(z, "palette_b2_p200"))).tobytes()) == \
        str(z["palette_b2_p200_sha256"])


def test_meta_and_zip_parsing(gsx_lib):
    from gsx import sog_reader
    z = np.load(GOLDEN)
    zf, meta = sog_reader.open_bundle(blob_of(z, "custom_names"))
    lay = sog_reader.parse_meta(meta)
    assert lay.count == 200 and lay.bands == 3 and lay.coeffs == 45 and lay.palette_size == 90
    assert lay.files["scales"] == lay.files["sh0"] == "shared.webp" and lay.files["quats"] == "q"
    assert lay.members() == {"pos/low.webp": 200, "pos/high.webp": 200, "shared.webp": 200, "q": 200,
                             "lab.webp": 200, "cent.webp": 64 * 45 * 2}
    flat = sog_reader.decode_members(zf, lay.members(), threads=1)
    assert np.array_equal(flat, sog_reader.decode_members(zf, lay.members(), threads=4))
    off = 0
    for name, need in lay.members().items():   # the pixels read_webp_to_flat keeps
        want, _ = sro.webp_pixels(zf, name)
        assert np.array_equal(flat[off:off + 4 * need], want[:4 * need]), name
        off += 4 * need
    lay0 = sog_reader.parse_meta(json.loads(zipfile.ZipFile(io.BytesIO(blob_of(z, "palette_b0_p65"))).read("meta.json")))
    assert lay0.bands == 0 and lay0.coeffs == 0 and lay0.pixels_needed()["centroids"] == 0
    assert sog_reader.parse_meta({**meta, "shN": {**meta["shN"], "bands": 0}}).bands == 0


def test_host_tables(gsx_lib):
    from gsx import sog_reader
    q, op = sog_reader.byte_tables()
    u = np.arange(256, dtype=np.uint8)
    assert q.dtype == op.dtype == np.float32
    assert np.array_equal(q, (u.astype(np.float32) / 255.0 - 0.5) * 2.0)
    codes = np.arange(65536, dtype=np.uint16)
    for mins, maxs in (((-2.0, 0, 3), (5.0, 0, 3.5)), ((np.nan, -np.inf, 1), (1.0, np.inf, 1)), ((-700, 1, 2), (700, 1, 2))):
        tab = sog_reader.position_tables(list(mins), list(maxs))
        for i in range(3):
            with np.errstate(all="ignore"):
                l = (codes / 65535.0) * (maxs[i] - mins[i]) + mins[i]
                want = (np.sign(l) * (np.exp(np.abs(l)) - 1.0)).astype(np.float32)
            assert np.array_equal(tab[i].view(np.uint32), want.view(np.uint32)), (mins, maxs, i)


@pytest.mark.parametrize("case", [c for c in golden_cases() if c.startswith("refuse_") and c not in KERNEL_REFUSALS])
def test_refused_before_the_device(case, gsx_lib):
    """Every malformed bundle is refused on the host: no device is needed to get the ValueError."""
    from gsx import sog_reader
    z = np.load(GOLDEN)
    with pytest.raises(ValueError):
        sog_reader.decode(blob_of(z, case), device="cuda")


@pytest.mark.parametrize("edit", [
    lambda m: m.update(count=True), lambda m: m.update(count=2 ** 31), lambda m: m["means"].update(maxs=[0, 1, "x"]),
    lambda m: m["means"].update(files="means_l.webp"), lambda m: m["scales"].update(codebook=[[1.0], [2.0]]),
    lambda m: m["shN"].update(bands=True), lambda m: m["shN"].update(bands=1.0), lambda m: m["shN"].pop("codebook"),
    lambda m: m.update(shN=None), lambda m: m["shN"].update(files=["only_one.webp"])])
def test_meta_refusals(edit, gsx_lib):
    from gsx import sog_reader
    z = np.load(GOLDEN)
    meta = json.loads(zipfile.ZipFile(io.BytesIO(blob_of(z, "palette_b1_p65"))).read("meta.json"))
    edit(meta)
    with pytest.raises(ValueError):
        sog_reader.parse_meta(meta)


def test_refused_without_pillow(gsx_lib, monkeypatch):
    from gsx import sog_reader
    z = np.load(GOLDEN)
    monkeypatch.setitem(sys.modules, "PIL", None)
    with pytest.raises(ValueError, match="Pillow"):
        sog_reader.decode(blob_of(z, "opacity_bytes"), device="cuda")


def test_kernel_argument_errors(gsx_lib):
    """Rejected before any device work: fake (never dereferenced) device pointers are enough."""
    import ctypes as C
    p = C.c_void_p(4096)
    tex = (C.c_void_p * 6)(*[4096 + 64 * k for k in range(6)])
    no_labels = (C.c_void_p * 6)(*[4096 + 64 * k for k in range(5)], None)
    assert gsx_lib.gsx_sog_decode(tex, 10, p, p, 256, 256, p, 5, 10, p, p, None) == -2            # coeffs
    assert gsx_lib.gsx_sog_decode(tex, 1 << 31, p, p, 256, 256, p, 5, 9, p, p, None) == -4
    assert gsx_lib.gsx_sog_decode(tex, -1, p, p, 256, 256, p, 5, 9, p, p, None) == -2
    assert gsx_lib.gsx_sog_decode(no_labels, 10, p, p, 256, 256, p, 5, 9, p, p, None) == -2      # SH, no labels
    assert gsx_lib.gsx_sog_decode(tex, 10, p, p, 256, 256, p, 0, 9, p, p, None) == -2            # labels, P = 0
    odd = (C.c_void_p * 6)(4097, 4160, 4224, 4288, 4352, None)
    assert gsx_lib.gsx_sog_decode(odd, 10, p, p, 256, 256, None, 0, 0, p, p, None) == -2         # misaligned
    assert gsx_lib.gsx_sog_decode(no_labels, 0, None, None, 0, 0, None, 0, 45, None, None, None) == 0
    assert gsx_lib.gsx_sog_decode(None, 1, p, p, 256, 256, p, 5, 9, p, p, None) == -2
    assert gsx_lib.gsx_sog_decode_palette(p, 10, 8, p, 256, p, p, None) == -2
    assert gsx_lib.gsx_sog_decode_palette(p, 1 << 27, 45, p, 256, p, p, None) == -4
    assert gsx_lib.gsx_sog_decode_palette(None, 0, 45, None, 256, None, None, None) == 0
    assert gsx_lib.gsx_sog_decode_palette(None, 10, 0, None, 256, None, None, None) == 0


def test_quaternion_rule_every_byte_triple():
    """The kernel's rule -- sqrt(max(1 - ((a*a + b*b) + c*c), 0)) in float32, one rounding per operation -- against
    the reference's np.sqrt(np.maximum(1.0 - np.sum(q_rest**2, axis=1), 0.0)) over all 2^24 byte triples."""
    u = np.arange(256, dtype=np.uint8)
    t = (u.astype(np.float32) / 255.0 - 0.5) * 2.0
    bad = 0
    for start in range(0, 1 << 24, 1 << 22):
        i = np.arange(start, start + (1 << 22), dtype=np.uint32)
        q = np.stack([t[i & 255], t[(i >> 8) & 255], t[i >> 16]], 1)
        want = np.sqrt(np.maximum(1.0 - np.sum(q ** 2, axis=1), 0.0))
        a, b, c = q[:, 0], q[:, 1], q[:, 2]
        s = (a * a + b * b) + c * c
        got = np.sqrt(np.maximum(np.float32(1) - s, np.float32(0)))
        assert got.dtype == want.dtype == np.float32
        bad += int(np.count_nonzero(got.view(np.uint32) != want.view(np.uint32)))
    assert bad == 0

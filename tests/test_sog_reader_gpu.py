"""GPU: the SOG reader on the device (gsx.sog_reader) against the reference reader's own results (g14) and the NumPy
oracle (sog_reader_oracle.py): every fixture bundle, every quaternion byte triple, every position code, every opacity
byte, the index checks, a 1 M-splat SH-3 round trip through the device writer, the records view and the drop-in."""

import numpy as np
import pytest

import sog_reader_oracle as sro
from test_sog_reader_cpu import GOLDEN, blob_of, golden_cases

pytestmark = pytest.mark.gpu


def assert_same(got: np.ndarray, want: np.ndarray, what: str):
    assert got.dtype == want.dtype and len(got) == len(want), what
    g, w = np.frombuffer(got.tobytes(), np.uint8), np.frombuffer(np.ascontiguousarray(want).tobytes(), np.uint8)
    d = np.flatnonzero(g != w)
    assert d.size == 0, f"{what}: {d.size} bytes differ, first at {d[:8]} (rows {d[:4] // got.dtype.itemsize})"


@pytest.mark.parametrize("case", golden_cases())
def test_device_matches_reference_golden(case, cuda, gsx_lib):
    from gsx import sog_reader
    z = np.load(GOLDEN)
    blob = blob_of(z, case)
    if str(z[f"{case}_expect"]) == "refuse":
        with pytest.raises(ValueError):
            sog_reader.decode(blob, cuda)
        return
    d = sog_reader.decode(blob, cuda)
    a = d.to_host()
    assert d.metadata is None and str(a.dtype.descr) == str(z[f"{case}_dtype"])
    if sro.digest(np.ascontiguousarray(a).tobytes()) != str(z[f"{case}_sha256"]):
        assert_same(a, sro.decode(blob), case)
        pytest.fail(f"{case}: equal to the oracle but not to the reference's digest")


# ------------------------------------------------------------------------------------- decode_textures on raw pixels
def textures(n, seed=0):
    rng = np.random.default_rng(seed)
    t = {k: rng.integers(0, 256, (n, 4), dtype=np.uint8) for k in ("means_l.webp", "means_u.webp", "quats.webp",
                                                                      "scales.webp", "sh0.webp")}
    t["quats.webp"][:, 3] = rng.integers(252, 256, n)
    return t


def meta_for(n, mins=(-2.0, -1.0, 0.5), maxs=(3.0, 2.5, 4.0), scb=256, ccb=256):
    rng = np.random.default_rng(n)
    return {"count": n, "means": {"mins": list(mins), "maxs": list(maxs), "files": ["means_l.webp", "means_u.webp"]},
            "scales": {"codebook": sorted(rng.normal(-4, 1, scb).tolist()), "files": ["scales.webp"]},
            "quats": {"files": ["quats.webp"]},
            "sh0": {"codebook": sorted(rng.normal(0, 1, ccb).tolist()), "files": ["sh0.webp"]}}


def add_shn(meta, tex, n, bands, P, seed=1, cb=256):
    rng = np.random.default_rng(seed)
    coeffs = sro.COEFFS[bands]
    meta["shN"] = {"count": P, "bands": bands, "codebook": sorted(rng.normal(0, 0.3, cb).tolist()),
                   "files": ["shN_centroids.webp", "shN_labels.webp"]}
    tex["shN_centroids.webp"] = rng.integers(0, cb, (64 * coeffs * -(-P // 64), 4), dtype=np.uint8)
    lab = rng.integers(0, P, n)
    tex["shN_labels.webp"] = np.stack([lab & 0xff, lab >> 8, np.zeros(n), np.full(n, 255)], 1).astype(np.uint8)


def run(tex, meta, cuda):
    import torch
    from gsx import sog_reader
    dev = {k: torch.from_numpy(np.ascontiguousarray(v).reshape(-1)).to(cuda) for k, v in tex.items()}
    got = sog_reader.decode_textures(dev, meta).to_host()
    with np.errstate(all="ignore"):
        want = sro.from_pixels(sro.pixels_reader({k: np.asarray(v).reshape(-1) for k, v in tex.items()}), meta)
    return got, want


def test_every_quaternion_triple(cuda, gsx_lib):
    n = 1 << 24
    t = textures(n, 1)
    i = np.arange(n, dtype=np.uint32)
    t["quats.webp"] = np.stack([i & 255, i >> 8 & 255, i >> 16, np.array([252, 253, 254, 255, 7])[i % 5]],
                               1).astype(np.uint8)
    got, want = run(t, meta_for(n), cuda)
    for k in range(4):
        assert np.array_equal(got[f"rot_{k}"].view(np.uint32), want[f"rot_{k}"].view(np.uint32)), k
    assert_same(got, want, "quaternion triples")


@pytest.mark.parametrize("mins, maxs", [((-2.0, -0.5, 0.0), (6.0, 0.5, 1e-6)), ((1.0, -3.0, 0.0), (1.0, -3.0, 0.0)),
                                        ((-np.inf, np.nan, -9.0), (np.inf, 1.0, -8.0)),
                                        ((-710.0, 700.0, 5.0), (710.0, 720.0, -5.0))])
def test_every_position_code(mins, maxs, cuda, gsx_lib):
    n = 65536
    t = textures(n, 2)
    c = np.arange(n, dtype=np.uint32)
    for ch in range(3):
        r = np.roll(c, 4099 * ch)
        t["means_l.webp"][:, ch], t["means_u.webp"][:, ch] = r & 0xff, r >> 8
    got, want = run(t, meta_for(n, mins, maxs), cuda)
    assert_same(got, want, f"positions {mins} {maxs}")


def test_every_opacity_byte_and_sh(cuda, gsx_lib):
    for bands in (0, 1, 2, 3):
        n = 256 * 3
        t = textures(n, 3 + bands)
        t["sh0.webp"][:, 3] = np.arange(n) % 256
        m = meta_for(n)
        add_shn(m, t, n, bands, 700, seed=bands)
        got, want = run(t, m, cuda)
        assert_same(got, want, f"bands {bands}")


def test_index_checks(cuda, gsx_lib):
    n = 1000
    base = textures(n, 5)
    m = meta_for(n)
    add_shn(m, base, n, 2, 300)
    base["shN_labels.webp"][0, :2] = (299 & 0xff, 299 >> 8)                              # the largest label

    def refused(edit_meta=None, edit_tex=None):
        import copy
        mm, tt = copy.deepcopy(m), {k: v.copy() for k, v in base.items()}
        if edit_meta:
            edit_meta(mm)
        if edit_tex:
            edit_tex(tt)
        with pytest.raises(ValueError):
            run(tt, mm, cuda)

    got, want = run(base, m, cuda)
    assert_same(got, want, "in range")
    refused(lambda mm: mm["scales"].update(codebook=mm["scales"]["codebook"][:255]),
            lambda tt: tt["scales.webp"].__setitem__((999, 2), 255))
    refused(lambda mm: mm["sh0"].update(codebook=mm["sh0"]["codebook"][:17]))
    refused(lambda mm: mm["shN"].update(codebook=mm["shN"]["codebook"][:128]))
    refused(edit_tex=lambda tt: tt["shN_labels.webp"].__setitem__((500, 1), 2))          # label 512 + x >= 300
    refused(lambda mm: mm["shN"].update(count=299))                                      # label 299 >= P


def test_no_splats(cuda, gsx_lib):
    for shn in (False, True):
        t = {k: np.zeros((0, 4), np.uint8) for k in ("means_l.webp", "means_u.webp", "quats.webp", "scales.webp",
                                                     "sh0.webp")}
        m = meta_for(0)
        if shn:
            add_shn(m, t, 0, 3, 5)
        got, want = run(t, m, cuda)
        assert len(got) == 0 and got.dtype == want.dtype


# ------------------------------------------------------------------------------------------------- at scale
def cheap_fit(values):
    """256 quantiles of the palette values: a codebook fit that does not dominate a 1 M-splat test."""
    return np.quantile(values.reshape(-1), np.linspace(0, 1, 256)).reshape(-1, 1)


def test_round_trip_1m_sh3(cuda, gsx_lib, tmp_path):
    """synth records -> gsx.sog.encode -> write_sog -> decode, against the oracle on the same bytes (not against the
    written records: the reader's palette indexing differs from the writer's layout)."""
    from gsx import records, sog, sog_reader, synth
    a = synth.structured(1 << 20, "mixed")
    np.random.seed(3)
    tex = sog.encode(records.DeviceRecords.from_structured(a, cuda), codebook_fit=cheap_fit)
    p = tmp_path / "r.sog"
    sog.write_sog(p, tex.to_host(), tex.meta)
    blob = p.read_bytes()
    d = sog_reader.decode(blob, cuda)
    with np.errstate(all="ignore"):
        want = sro.decode(blob)
    assert_same(d.to_host(), want, "1 M SH-3 round trip")
    assert tex.meta["shN"]["count"] == 65536


def test_records_feed_the_device_writers(cuda, gsx_lib):
    from gsx import records, sog_reader, splat
    z = np.load(GOLDEN)
    d = sog_reader.decode(blob_of(z, "writer_n300_d3_l0"), cuda)
    r = d.records()
    assert r.rows.data_ptr() == d.rows.data_ptr()                    # zero-copy view
    host = records.DeviceRecords.from_structured(d.to_host(), cuda)
    with np.errstate(all="ignore"):
        assert splat.encode(r).to_host() == splat.encode(host).to_host()


class StandIn:
    def __init__(self):
        self.calls = []

    def read(self, path, *args, **kwargs):
        self.calls.append((path, args, kwargs))
        return "reference"


def test_dropin_read_on_stand_in_class(cuda, gsx_lib, tmp_path):
    from gsx import dropin, sog_reader
    z = np.load(GOLDEN)
    cls = type("StandInSog", (StandIn,), {})
    dropin.install_reader(cls, sog_reader.decode, webp="host")
    dropin.install_reader(cls, sog_reader.decode, webp="host")       # idempotent
    assert cls._gsx_reference_read is StandIn.read and cls.read is not StandIn.read
    r = cls()
    p = tmp_path / "a.sog"
    p.write_bytes(blob_of(z, "custom_names"))
    got = r.read(str(p))
    assert r.calls == [] and isinstance(got, np.ndarray)
    assert_same(got, sro.decode(p.read_bytes()), "drop-in")
    for bad in ("refuse_bands-1", "refuse_label_oob"):                # refused: the original read, original arguments
        q = tmp_path / f"{bad}.sog"
        q.write_bytes(blob_of(z, bad))
        r.calls.clear()
        assert r.read(str(q), 7, level=4) == "reference"
        assert r.calls == [(str(q), (7,), {"level": 4})]


def test_patch_rejects_unknown_sog_reader(gsx_lib):
    from gsx import dropin
    with pytest.raises(ValueError):
        dropin.patch(sog_reader="gpu")

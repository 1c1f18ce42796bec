"""GPU: gsx.webp's lossless WebP encoder against the NumPy restatement (webp_oracle.py), byte for byte, and the SOG
bundle written from device textures against the Pillow bundle: same pixels, same meta.json, same decoded rows."""
import io
import json
import zipfile

import numpy as np
import pytest

import webp_oracle as wo

pytestmark = pytest.mark.gpu

CASES = wo.cases()


def device_encode(img, cuda, info=None):
    import torch
    from gsx import webp
    h, w = img.shape[:2]
    t = torch.from_numpy(np.ascontiguousarray(img).reshape(-1, 4)).to(cuda)
    return webp.encode_lossless(t, w, h, info=info)


def check_case(img, cuda):
    want_info, got_info = {}, {}
    want = wo.encode(img, info=want_info)
    got = device_encode(img, cuda, got_info)
    assert got_info["candidate"] == want_info["candidate"]
    assert got_info["bits"] == want_info["bits"]
    if want_info["modes"] is None:
        assert got_info["modes"] is None
    else:
        assert np.array_equal(got_info["modes"], want_info["modes"])
    if got != want:
        diff = next(i for i, (a, b) in enumerate(zip(got, want)) if a != b) if len(got) == len(want) else None
        raise AssertionError(f"device file ({len(got)} B) differs from the oracle's ({len(want)} B) at byte {diff}")
    return got


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_bytes_equal_oracle(name, cuda, gsx_lib):
    check_case(CASES[name], cuda)


def test_device_bytes_equal_oracle_on_sog_textures(cuda, gsx_lib):
    for img in wo.sog_textures().values():
        check_case(img, cuda)


def test_refusals_before_any_launch(cuda, gsx_lib):
    import torch
    from gsx import webp
    before = gsx_lib.gsx_kernel_launches()
    ok = torch.zeros((4, 4), dtype=torch.uint8, device=cuda)
    with pytest.raises(ValueError):
        webp.encode_lossless(torch.zeros((16385, 4), dtype=torch.uint8, device=cuda), 16385, 1)
    with pytest.raises(ValueError):
        webp.encode_lossless(torch.zeros((16385, 4), dtype=torch.uint8, device=cuda), 1, 16385)
    with pytest.raises(ValueError):
        webp.encode_lossless(ok.float(), 2, 2)
    with pytest.raises(ValueError):
        webp.encode_lossless(ok.cpu(), 2, 2)
    with pytest.raises(ValueError):
        webp.encode_lossless(ok, 3, 2)
    with pytest.raises(ValueError):
        webp.encode_lossless(ok, 0, 4)
    assert gsx_lib.gsx_kernel_launches() == before


def quantile_fit(values):
    return np.quantile(values.reshape(-1), np.linspace(0, 1, 256)).astype(np.float32)


@pytest.fixture(scope="module")
def sog_1m(cuda):
    from gsx import records, sog, synth
    a = synth.structured(1_000_000, "mixed", 3)
    np.random.seed(3)
    return sog.encode(records.DeviceRecords.from_structured(a, cuda), 0, codebook_fit=quantile_fit)


def test_device_bytes_equal_oracle_on_1m_sog_textures(sog_1m, cuda, gsx_lib):
    host = sog_1m.to_host()
    for name, t in sog_1m.textures.items():
        w, h = sog_1m.sizes[name]
        from gsx import webp
        assert webp.encode_lossless(t, w, h) == wo.encode(host[name]), name


def decode_member(zf, name):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(zf.read(name))).convert("RGBA"))


def same_pixels(a, b):
    """Equal alpha everywhere and equal RGB where alpha > 0: libwebp keeps no RGB under alpha 0 (its predictor leaves
    the predicted value there, gsx leaves 0), so those bytes carry nothing either file promises."""
    visible = a[..., 3] > 0
    return np.array_equal(a[..., 3], b[..., 3]) and np.array_equal(a[visible], b[visible])


def test_write_sog_device_bundle_matches_pillow_bundle(sog_1m, cuda, gsx_lib, tmp_path):
    from gsx import sog, sog_reader
    sog.write_sog(tmp_path / "dev.sog", sog_1m, sog_1m.meta)
    sog.write_sog(tmp_path / "pil.sog", sog_1m.to_host(), sog_1m.meta)
    ratios = {}
    with zipfile.ZipFile(tmp_path / "dev.sog") as zd, zipfile.ZipFile(tmp_path / "pil.sog") as zp:
        assert zd.namelist() == zp.namelist()
        assert all(i.compress_type == zipfile.ZIP_STORED for i in zd.infolist())
        assert json.loads(zd.read("meta.json")) == json.loads(zp.read("meta.json"))
        for name in zd.namelist()[:-1]:
            assert same_pixels(decode_member(zd, name), decode_member(zp, name)), name
            ratios[name] = zd.getinfo(name).file_size / zp.getinfo(name).file_size
    dev, pil = (tmp_path / "dev.sog").stat().st_size, (tmp_path / "pil.sog").stat().st_size
    print("device / Pillow bytes per member:", {k: round(v, 3) for k, v in ratios.items()},
          f"bundle {dev} / {pil} = {dev / pil:.3f}")
    a = sog_reader.decode(tmp_path / "dev.sog", cuda)
    b = sog_reader.decode(tmp_path / "pil.sog", cuda)
    assert a.dtype == b.dtype and bytes(a.rows.cpu().numpy()) == bytes(b.rows.cpu().numpy())
    assert dev <= 1.2 * pil, f"device bundle {dev} B is {dev / pil:.3f}x the Pillow bundle {pil} B"


def test_dropin_write_device_webp_on_stand_in_class(cuda, gsx_lib, tmp_path):
    from gsx import dropin, sog, sog_reader, synth

    class StandIn:
        def write(self, data, path, **kwargs):
            raise AssertionError("the original write must not run for packed float32 records")

    class HostWebp(StandIn):
        pass

    dropin.install_writer(StandIn, sog.prepare_write, webp="device")
    dropin.install_writer(HostWebp, sog.prepare_write, webp="host")
    a = synth.structured(3_000, "mixed")
    np.random.seed(8)
    StandIn().write(a, tmp_path / "dev.sog", compression_level=7)
    np.random.seed(8)
    HostWebp().write(a, tmp_path / "pil.sog", compression_level=7)
    with zipfile.ZipFile(tmp_path / "dev.sog") as zd, zipfile.ZipFile(tmp_path / "pil.sog") as zp:
        assert zd.namelist() == zp.namelist()
        assert zd.read("meta.json") == zp.read("meta.json")
        names = zd.namelist()[:-1]
        assert any(zd.read(n) != zp.read(n) for n in names)        # gsx's bytes, not libwebp's
        for n in names:
            assert same_pixels(decode_member(zd, n), decode_member(zp, n)), n
    ra = sog_reader.decode(tmp_path / "dev.sog", cuda)
    rb = sog_reader.decode(tmp_path / "pil.sog", cuda)
    assert bytes(ra.rows.cpu().numpy()) == bytes(rb.rows.cpu().numpy())


def test_dropin_patch_sog_webp_option():
    from gsx import dropin
    with pytest.raises(ValueError):
        dropin.patch(sog_webp="device")                           # needs sog="device"
    with pytest.raises(ValueError):
        dropin.patch(sog="device", sog_webp="cuda")

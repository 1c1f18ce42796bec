"""GPU: gsx.webp_decode.decode_lossless against Pillow's convert('RGBA'), byte for byte, on every CPU case at the
default chunk size, at tiny chunks (false starts, group mismatches, re-decode rounds) and with the serial fallback;
the malformed streams; and the SOG reader with its WebP members decoded on the device against the host decode."""
import io
import zipfile

import numpy as np
import pytest

import vp8l_model as M
from test_sog_reader_cpu import GOLDEN, blob_of, golden_cases
from test_vp8l_cpu import CASES, malformed

pytestmark = pytest.mark.gpu


def device_rgba(data, cuda, **kw):
    from gsx.webp_decode import decode_lossless
    return decode_lossless(data, cuda, **kw).cpu().numpy()


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_pillow(name, cuda, gsx_lib):
    data = CASES[name]
    want = M.pillow_rgba(data)
    for kw in ({}, {"chunk_bits": 64}, {"chunk_bits": 64, "max_rounds": 0}):
        got = device_rgba(data, cuda, **kw)
        assert got.shape == want.shape and np.array_equal(got, want), (name, kw, np.argwhere(got != want)[:4])


def test_chain_paths_are_taken(cuda, gsx_lib):
    """Tiny chunks on a multi-group stream: false starts, group mismatches and rounds; max_rounds=0: the serial
    decode from the frontier."""
    data = CASES["half_m4_q100"]
    st = {}
    device_rgba(data, cuda, chunk_bits=32, stats=st)
    assert st["groups"] > 1 and st["chunks"] > 8
    assert st["false_starts"] + st["group_mismatches"] > 0 and st["rounds"] > 0, st
    st = {}
    assert np.array_equal(device_rgba(data, cuda, chunk_bits=32, max_rounds=0, stats=st), M.pillow_rgba(data))
    assert st["serial_fallbacks"] == 1 and st["rounds"] == 0


def test_large_images(cuda, gsx_lib):
    """1000 x 700 noise and gradient images (both multi-group with libwebp at method 4) at the default chunks."""
    rng = np.random.default_rng(9)
    y, x = np.mgrid[0:700, 0:1000]
    a = np.stack([x & 255, y & 255, (x * y) & 255, np.full_like(x, 255)], -1).astype(np.uint8)
    a[300:400] = rng.integers(0, 256, (100, 1000, 4))
    for m in (1, 4):
        data = M.pillow_file(a, method=m)
        st = {}
        assert np.array_equal(device_rgba(data, cuda, stats=st), M.pillow_rgba(data)), (m, st)


@pytest.mark.parametrize("name", sorted(malformed()))
def test_malformed_streams_raise(name, cuda, gsx_lib):
    with pytest.raises(ValueError):
        device_rgba(malformed()[name], cuda)


def test_not_lossless_is_refused(cuda, gsx_lib):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(b, "WEBP", quality=80)
    with pytest.raises(ValueError):
        device_rgba(b.getvalue(), cuda)


def test_parallel_only_routes_by_header(cuda, gsx_lib):
    """Streams with several groups or a colour cache come back as None; one-group cache-free ones decode."""
    from gsx.webp_decode import decode_lossless
    assert decode_lossless(CASES["half_m4_q100"], cuda, parallel_only=True) is None      # 2 groups, cache 7
    assert decode_lossless(CASES["all_cache"], cuda, parallel_only=True) is None         # cache 6
    got = decode_lossless(CASES["all_copies"], cuda, parallel_only=True)
    assert np.array_equal(got.cpu().numpy(), M.pillow_rgba(CASES["all_copies"]))


def same_rows(blob, cuda):
    from gsx import sog_reader
    host = sog_reader.decode(blob, cuda).to_host()
    dev = sog_reader.decode(blob, cuda, webp="device").to_host()
    assert host.dtype == dev.dtype and host.tobytes() == dev.tobytes()


@pytest.mark.parametrize("case", [c for c in golden_cases() if c.startswith("writer")])
def test_sog_reader_webp_device_on_pillow_bundles(case, cuda, gsx_lib):
    z = np.load(GOLDEN)
    blob = blob_of(z, case)
    if f"{case}_raises" in z.files:
        pytest.skip("the reference raises on this bundle")
    same_rows(blob, cuda)


def test_sog_reader_webp_device_on_gsx_bundles(cuda, gsx_lib, tmp_path):
    from gsx import records, sog, synth
    from test_sog_reader_gpu import cheap_fit
    a = synth.structured(50_000, "mixed")
    np.random.seed(3)
    tex = sog.encode(records.DeviceRecords.from_structured(a, cuda), codebook_fit=cheap_fit)
    for k, how in enumerate((tex, tex.to_host())):      # members by gsx.webp on the device, then by Pillow
        p = tmp_path / f"r{k}.sog"
        sog.write_sog(p, how, tex.meta)
        same_rows(p.read_bytes(), cuda)


def test_dropin_falls_back_on_a_bad_member(cuda, gsx_lib, tmp_path):
    from gsx import dropin, sog_reader

    class StandIn:
        def read(self, path, *args, **kwargs):
            return "reference"

    z = np.load(GOLDEN)
    src = io.BytesIO(blob_of(z, "writer_n300_d0_l0"))
    out = io.BytesIO()
    with zipfile.ZipFile(src) as zi, zipfile.ZipFile(out, "w") as zo:
        for name in zi.namelist():
            b = zi.read(name)
            zo.writestr(name, b[:len(b) // 2] if name == "quats.webp" else b)
    p = tmp_path / "bad.sog"
    p.write_bytes(out.getvalue())
    with pytest.raises(ValueError):
        sog_reader.decode(out.getvalue(), cuda, webp="device")
    dropin.install_reader(StandIn, sog_reader.decode, webp="device")
    assert StandIn().read(str(p)) == "reference"

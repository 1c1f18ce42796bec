"""GPU: compressed PLY encode on the device (Morton order, chunk bounds, gsx_cply_pack) against the NumPy oracle
(compressed_ply_oracle.py) and the reference writer's own output (g10)."""
from pathlib import Path

import numpy as np
import pytest

import compressed_ply_oracle as cpo

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "g10_reference_compressed_ply_small.npz"


def device_encode(a, cuda, order=None):
    import torch
    from gsx import compressed_ply, records
    r = records.DeviceRecords.from_structured(a, cuda)
    if order is not None:
        order = torch.from_numpy(np.asarray(order, np.int32)).to(cuda)
    enc = compressed_ply.encode(r, order)
    return enc, enc.to_host()


def check_against_oracle(a, cuda, order=None):
    enc, got = device_encode(a, cuda, order)
    o = enc.order.cpu().numpy()
    assert np.array_equal(np.sort(o), np.arange(len(a)))
    if order is not None:
        assert np.array_equal(o, order)
    want = cpo.encode(a, o)
    cpo.assert_packed_equal(got, want)
    assert list(enc.sh_names) == (list(want[2].dtype.names) if want[2] is not None else [])
    return enc, got


def test_encode_300k_mixed(cuda, gsx_lib):
    from gsx import synth
    enc, (chunk, vertex, sh) = check_against_oracle(synth.structured(300_000, "mixed"), cuda)
    assert len(chunk) == (300_000 + 255) // 256 and sh is not None and len(sh.dtype.names) == 45


@pytest.mark.parametrize("tag", ["mixed", "deg1"])
def test_encode_matches_reference_golden(tag, cuda, gsx_lib):
    z = np.load(GOLDEN)
    a = cpo.golden_inputs()[tag]
    assert cpo.digest(a) == str(z[f"{tag}_input_sha256"])
    enc, got = device_encode(a, cuda)
    assert np.array_equal(enc.order.cpu().numpy(), z[f"{tag}_order"])
    want = (z[f"{tag}_chunk"], z[f"{tag}_vertex"], z[f"{tag}_sh"] if f"{tag}_sh" in z.files else None)
    cpo.assert_packed_equal(got, want)
    assert list(enc.sh_names) == list(z[f"{tag}_sh_names"])


def test_encode_blobs_recurse(cuda, gsx_lib):
    from gsx import synth
    a = synth.structured(200_000, "mixed")
    rng = np.random.default_rng(5)
    for start, cnt, sigma in ((1000, 400, 1e-3), (50_000, 1500, 1e-4), (120_000, 300, 1e-3), (150_000, 700, 0.0)):
        for f in ("x", "y", "z"):
            a[f][start:start + cnt] = a[f][start] + rng.normal(0, sigma, cnt).astype(np.float32)
    check_against_oracle(a, cuda)


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 513])
def test_encode_sizes(n, cuda, gsx_lib):
    from gsx import synth
    enc, (chunk, vertex, sh) = check_against_oracle(synth.structured(n, "mixed"), cuda)
    assert len(chunk) == (n + 255) // 256 and len(vertex) == n
    assert (sh is None) == (n == 0)


def edge_cloud():
    """Identity order, so every chunk is what it is built to be: equal positions; an extent of exactly f32(1e-5); one
    just below; quaternion, scale, f_rest and opacity extremes."""
    from gsx import synth
    a = synth.structured(6 * 256 + 17, "mixed")
    a["x"][:256], a["y"][:256], a["z"][:256] = 0.75, -1.5, 3.0
    e = np.float32(1e-5)
    for c, hi in ((1, e), (2, np.nextafter(e, np.float32(0)))):
        sl = slice(c * 256, (c + 1) * 256)
        for f in ("x", "y", "z", "scale_0", "scale_1", "scale_2"):
            v = np.zeros(256, np.float32)
            v[7], v[100] = hi, hi / 2
            a[f][sl] = v
        for f in ("f_dc_0", "f_dc_1", "f_dc_2"):
            a[f][sl] = 0.25
    base = 3 * 256
    quats = [(0, 0, 0, 0), (0.5, 0.5, 0.5, 0.5), (-0.5, 0.5, -0.5, 0.5), (0.3, -0.3, 0.3, 0.2), (-0.9, 0.1, 0.2, 0.3),
             (0.1, 0.2, -0.95, -0.1), (0.0, 0.0, 0.0, -2.0), (1e-30, 0, 0, 0), (7.0, -7.0, 1.0, 0.0)]
    for k, q in enumerate(quats):
        for i in range(4):
            a[f"rot_{i}"][base + k] = q[i]
    for k, v in enumerate((25.0, -25.0, 20.0, -20.0, 20.5, -1e9, 1e9, 19.999)):
        a[f"scale_{k % 3}"][base + 20 + k] = v
    for k, v in enumerate((4.0, -4.0, -4.01, 3.999, 50.0, -50.0, 1e30, -1e30, 1e-40, -0.0)):
        a[f"f_rest_{(11 * k) % 45}"][base + 40 + k] = v
    for k, v in enumerate((200.0, -200.0, 150.0, -150.0, 0.0, -0.0)):
        a["opacity"][base + 60 + k] = v
    return a


def test_encode_edge_rows(cuda, gsx_lib):
    a = edge_cloud()
    _, (chunk, vertex, _) = check_against_oracle(a, cuda, order=np.arange(len(a)))
    assert np.all(vertex["packed_position"][:256] == 0)
    assert chunk["max_x"][1] - chunk["min_x"][1] == np.float32(1e-5)
    assert np.any(vertex["packed_position"][256:512] != 0)                 # f32(1e-5) is not degenerate
    assert np.all(vertex["packed_position"][512:768] == 0)                 # just below it is
    assert vertex["packed_rotation"][3 * 256] == (512 << 20 | 512 << 10 | 512)


def sh_cloud(n=1000):
    from gsx import synth
    a = synth.structured(n, "mixed")
    for i in range(45):
        a[f"f_rest_{i}"] = 0.0
    return a


def test_sh_degree_detection(cuda, gsx_lib):
    a = sh_cloud()
    a["f_rest_0"] = 0.5
    a["f_rest_9"][-1] = 0.25                         # the only non-zero f_rest_>=9, in the last row -> degree 2
    enc, (_, _, sh) = check_against_oracle(a, cuda)
    assert len(enc.sh_names) == 24 and sh.dtype.names[-1] == "f_rest_23"
    a = sh_cloud()
    a["f_rest_30"][500] = -1.0                       # degree 3, no narrowing
    enc, _ = check_against_oracle(a, cuda)
    assert len(enc.sh_names) == 45
    a = sh_cloud()
    a["f_rest_3"][2] = 1.0                           # degree 1
    enc, _ = check_against_oracle(a, cuda)
    assert len(enc.sh_names) == 9


def test_sh_all_zero_and_negative_zero(cuda, gsx_lib):
    enc, (_, _, sh) = check_against_oracle(sh_cloud(), cuda)
    assert sh is None and enc.sh is None and enc.sh_names == ()
    a = sh_cloud()
    a["f_rest_44"] = -0.0
    a["f_rest_5"][::3] = -0.0
    enc, (_, _, sh) = check_against_oracle(a, cuda)
    assert sh is None


def test_no_f_rest_fields(cuda, gsx_lib):
    from gsx import synth
    full = synth.structured(700, "mixed", sh_degree=0)
    assert not any(f.startswith("f_rest_") for f in full.dtype.names)
    enc, (_, _, sh) = check_against_oracle(full, cuda)
    assert sh is None
    # f_rest_ columns are taken by index, wherever they sit in the row and with gaps in the numbering
    a = synth.structured(600, "mixed")
    keep = [f for f in a.dtype.names if f not in ("f_rest_2", "f_rest_30")][::-1]
    b = np.zeros(len(a), dtype=[(f, "f4") for f in keep])
    for f in keep:
        b[f] = a[f]
    enc, (_, _, sh) = check_against_oracle(b, cuda)
    assert len(sh.dtype.names) == 43 and "f_rest_2" not in sh.dtype.names


def test_gathered_survivors(cuda, gsx_lib):
    import torch
    from gsx import compressed_ply, records, synth
    a = synth.structured(100_000, "mixed")
    r = records.DeviceRecords.from_structured(a, cuda)
    _, op = r.xyz_opacity()
    survivors = torch.nonzero(op > -1.0).flatten().to(torch.int32)
    enc = compressed_ply.encode(r.gather(survivors))
    s = survivors.cpu().numpy()
    assert 0 < len(s) < len(a)
    cpo.assert_packed_equal(enc.to_host(), cpo.encode(a[s], enc.order.cpu().numpy()))


def test_dropin_write_on_stand_in_class(cuda, gsx_lib, tmp_path):
    import torch
    from gsx import compressed_ply, dropin, morton, synth

    class StandIn:
        def __init__(self):
            self.calls = []

        def write(self, data, path, **kwargs):
            self.calls.append(("original", data, path, kwargs))

        def _write_ply_file(self, path, chunk_data, vertex_data, sh_data):
            self.calls.append(("file", path, chunk_data, vertex_data, sh_data))

    original = StandIn.write
    dropin.install_writer(StandIn, compressed_ply.prepare_write)
    dropin.install_writer(StandIn, compressed_ply.prepare_write)     # idempotent
    assert StandIn._gsx_reference_write is original and StandIn.write is not original
    a = synth.structured(5_000, "mixed")
    w = StandIn()
    w.write(a, tmp_path / "a.ply")
    assert [c[0] for c in w.calls] == ["file"]
    xyz = torch.from_numpy(np.ascontiguousarray(np.c_[a["x"], a["y"], a["z"]])).to(cuda)
    order = morton.morton_order(xyz).cpu().numpy()
    _, path, chunk, vertex, sh = w.calls[0]
    assert path == tmp_path / "a.ply"
    cpo.assert_packed_equal((chunk, vertex, sh), cpo.encode(a, order))
    # u1 colour fields: not packed float32 records -> the original write, untouched
    b = np.zeros(10, dtype=[("x", "f4"), ("y", "f4"), ("z", "f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    w2 = StandIn()
    w2.write(b, "b.ply", level=3)
    assert len(w2.calls) == 1 and w2.calls[0][0] == "original" and w2.calls[0][1] is b and w2.calls[0][3] == {"level": 3}
    # packed float32 but without the fields the format needs: gsx raises, the original write runs
    c = np.zeros(10, dtype=[("x", "f4"), ("y", "f4"), ("z", "f4")])
    w3 = StandIn()
    w3.write(c, "c.ply")
    assert [x[0] for x in w3.calls] == ["original"]

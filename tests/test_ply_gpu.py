"""GPU: the plain 3DGS and CloudCompare PLY readers and writers on the device (gsx.ply decode / encode) against the
reference's own results (g15) and the NumPy oracle (ply_oracle.py) at 1 M and 10 M splats; gsx_ply_transcode at every
row stride residue, partial last tiles and 1024-byte rows; every float32 pattern and the integer and float64 edges of
its casts; round trips between the flavours; a decode -> filters -> gather -> encode chain that never builds the host
array; and the drop-in.  Bytes are compared, not values."""

import numpy as np
import pytest

import ply_oracle as po
import splat_codecs_oracle as sco
from test_ply_cpu import GOLDEN, expected, golden_cases, writer_input

pytestmark = pytest.mark.gpu


def assert_same(got: np.ndarray, want: np.ndarray, what: str):
    assert str(got.dtype.descr) == str(want.dtype.descr) and len(got) == len(want), what
    g = np.frombuffer(np.ascontiguousarray(got).tobytes(), np.uint8)
    w = np.frombuffer(np.ascontiguousarray(want).tobytes(), np.uint8)
    d = np.flatnonzero(g != w)
    assert d.size == 0, f"{what}: {d.size} bytes differ, first at {d[:8]} (rows {d[:4] // got.dtype.itemsize})"


@pytest.mark.parametrize("case", golden_cases())
def test_device_matches_reference_golden(case, cuda, gsx_lib):
    from gsx import ply
    z = np.load(GOLDEN)
    flavor = str(z[f"{case}_flavor"])
    if case.startswith("read_"):
        run = lambda: ply.decode(z[f"{case}_file"].tobytes(), flavor, cuda)  # noqa: E731
    else:
        run = lambda: ply.encode(writer_input(z, case), flavor, bool(z[f"{case}_crop"]), cuda)  # noqa: E731
    if expected(z, case) == "refuse":
        with pytest.raises(ValueError):
            run()
        return
    a = run().to_host()
    b = np.ascontiguousarray(a).tobytes()
    assert str(a.dtype.descr) == str(z[f"{case}_dtype"])
    assert len(b) == int(z[f"{case}_len"]) and sco.digest(b) == str(z[f"{case}_sha256"]), case


@pytest.mark.parametrize("n", [1 << 20, 10_000_000])
@pytest.mark.parametrize("flavor", ["3dgs", "cc"])
def test_synth_cloud_decode_and_encode(n, flavor, cuda, gsx_lib):
    """A gsx.synth cloud written by the oracle writer, decoded and re-encoded on the device (from Decoded rows and
    from its DeviceRecords view), against the oracle reader and writer."""
    import torch
    from gsx import ply, synth
    blob = po.file(po.write(synth.structured(n, "mixed"), flavor))
    dec = ply.decode(blob, flavor, cuda)
    want = po.read(blob, flavor)
    del blob
    assert_same(dec.to_host(), want, f"decode {flavor}")
    enc_want = po.write(want, flavor, crop_sh=True)
    del want
    assert_same(ply.encode(dec, flavor, crop_sh=True).to_host(), enc_want, f"encode {flavor} from Decoded")
    assert_same(ply.encode(dec.records(), flavor, crop_sh=True).to_host(), enc_want, f"encode {flavor} from records")
    del dec
    torch.cuda.empty_cache()


def transcode_case(src_row, dst_row, n, seed, cuda):
    """Random source rows with fields at odd offsets of every type, the kernel's result and NumPy's field assignment
    into zeroed destination rows."""
    import torch
    from gsx import ply
    from gsx.hostcopy import to_device, to_host
    rng = np.random.default_rng(seed)
    kinds = ["i1", "u1", "<i2", "<u2", "<i4", "<u4", "<f4", "<f8"]
    pairs, s_off, d_off = [], 1, 3
    while True:   # one field of each type, then float32 -> float32 copies, at increasing unaligned offsets
        k = kinds[len(pairs)] if len(pairs) < len(kinds) else "<f4"
        d = {"<f8": "<f4"}.get(k, k) if len(pairs) % 3 else ("u1" if k in ("<f4", "<f8", "<u2") else k)
        ws, wd = np.dtype(k).itemsize, np.dtype(d).itemsize
        if s_off + ws > src_row or d_off + wd > dst_row:
            break
        pairs.append((k, s_off, d, d_off))
        s_off += ws + int(rng.integers(0, 3))
        d_off += wd + int(rng.integers(0, 2))
    sdt = np.dtype({"names": [f"s{i}" for i in range(len(pairs))], "formats": [p[0] for p in pairs],
                    "offsets": [p[1] for p in pairs], "itemsize": src_row})
    ddt = np.dtype({"names": [f"d{i}" for i in range(len(pairs))], "formats": [p[2] for p in pairs],
                    "offsets": [p[3] for p in pairs], "itemsize": dst_row})
    raw = rng.integers(0, 256, n * src_row + 7, dtype=np.uint8)
    src = np.frombuffer(raw[7:].tobytes(), sdt)
    want = np.zeros(n, ddt)
    with np.errstate(all="ignore"):
        for i in range(len(pairs)):
            want[f"d{i}"] = src[f"s{i}"]
    table = ply.field_table(sdt, ddt, [(f"s{i}", f"d{i}") for i in range(len(pairs))], "test")
    dev = to_device(raw, cuda)
    got = to_host(ply.transcode(dev, 7, n, src_row, dst_row, table))
    torch.cuda.synchronize()
    return got.reshape(-1), np.frombuffer(want.tobytes(), np.uint8), len(pairs)


@pytest.mark.parametrize("src_row", list(range(248, 264)) + [1, 9, 71, 1023, 1024])
def test_transcode_every_row_stride(src_row, cuda, gsx_lib):
    """Source rows at every residue mod 16 and narrow and 1024-byte rows, destination rows of a different residue,
    64 * k + 37 rows (a partial last tile), the source 7 bytes into its allocation."""
    wider = src_row + 3 if src_row + 3 <= 1024 else src_row - 9
    for dst_row, n in ((wider, 64 * 40 + 37), (1024, 64 + 1), (max(1, src_row - 5), 37)):
        got, want, nf = transcode_case(src_row, dst_row, n, src_row * 31 + dst_row, cuda)
        d = np.flatnonzero(got != want)
        assert d.size == 0, f"rows {src_row} -> {dst_row}, {nf} fields: {d.size} bytes differ, first at {d[:8]}"


def test_f4_to_u1_every_float32(cuda, gsx_lib):
    """Every float32 bit pattern through the f4 -> u1 cast (the `red` of a file that stores colours as float), against
    the truncation to int32 and its low byte computed with torch on the device (0 for NaN and out-of-range values),
    the rule NumPy's strided field assignment follows on x86 for all 2^32 patterns."""
    import torch
    from gsx import ply
    m = 1 << 28
    bad, start = 0, 0
    table = [1, ply.TYPE_CODES[("f", 4)], 0, ply.TYPE_CODES[("u", 1)]]
    buf = torch.empty(m * 5, dtype=torch.uint8, device=cuda)
    while start < (1 << 32):
        bits = torch.arange(start, start + m, dtype=torch.int64, device=cuda)
        bits = torch.where(bits < (1 << 31), bits, bits - (1 << 32)).to(torch.int32)
        buf.view(m, 5)[:, 1:5] = bits.view(torch.uint8).view(m, 4)
        got = ply.transcode(buf, 0, m, 5, 1, table).view(-1)
        v = bits.view(torch.float32).to(torch.float64)
        t = torch.trunc(v)
        ok = torch.isfinite(t) & (t >= -2147483648.0) & (t < 2147483648.0)
        want = torch.where(ok, torch.where(ok, t, 0.0).to(torch.int64) & 0xff, 0).to(torch.uint8)
        bad += int((got != want).sum())
        start += m
    assert bad == 0, f"{bad} of 2^32 float32 -> uint8 casts differ"


def cast_edges():
    f8 = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -5e-324, 1e-46, 1.4e-45, 7e-46, 0.7e-45,
                   1.1754942e-38, 3.4028235e38, 3.4028235677973366e38, 3.4028236e38, 1e39, -1e300, 0.1, 0.5, 1.5,
                   2.5, -0.5, 255.5, 255.99, 256.0, -1.0, -1.5, 2147483647.5, 2147483648.0, -2147483648.5,
                   -2147483649.0, 4294967295.0, 4294967296.0, 1e19, 16777217.0, 16777219.0], np.float64)
    rng = np.random.default_rng(7)
    bits = np.concatenate([f8.view(np.uint64), rng.integers(0, 1 << 64, 200_000, dtype=np.uint64, endpoint=False),
                           np.array([0x7ff0000000000001, 0x7ff4000000000000, 0xfff0000020000000, 0x7ff8000000000001,
                                     0x000fffffffffffff, 0x3ff0000010000000, 0x3ff0000030000000], np.uint64)])
    return {"f8": bits.view(np.float64),
            "i1": np.arange(-128, 128, dtype=np.int8), "u1": np.arange(256, dtype=np.uint8),
            "i2": np.arange(-32768, 32768, dtype=np.int16), "u2": np.arange(65536, dtype=np.uint16),
            "i4": np.concatenate([np.array([-2 ** 31, 2 ** 31 - 1, 16777217, -16777217, 16777219, 33554435], np.int32),
                                  rng.integers(-2 ** 31, 2 ** 31, 200_000, dtype=np.int32)]),
            "u4": np.concatenate([np.array([2 ** 32 - 1, 2 ** 31, 16777217, 4294967040, 4294967168], np.uint32),
                                  rng.integers(0, 2 ** 32, 200_000, dtype=np.uint32)])}


@pytest.mark.parametrize("src", ["i1", "u1", "i2", "u2", "i4", "u4", "f8"])
def test_cast_edges(src, cuda, gsx_lib):
    """Integer and float64 sources into float32 and uint8 fields, against NumPy's strided field assignment."""
    from gsx import ply
    from gsx.hostcopy import to_device, to_host
    vals = cast_edges()[src]
    sdt = np.dtype({"names": ["v"], "formats": [vals.dtype.newbyteorder("<")], "offsets": [3], "itemsize": 13})
    ddt = np.dtype({"names": ["f", "u"], "formats": ["<f4", "u1"], "offsets": [1, 6], "itemsize": 7})
    a = np.zeros(len(vals), sdt)
    a["v"] = vals
    want = np.zeros(len(vals), ddt)
    with np.errstate(all="ignore"):
        want["f"], want["u"] = a["v"], a["v"]
    table = ply.field_table(sdt, ddt, [("v", "f"), ("v", "u")], "test")
    raw = to_device(np.frombuffer(a.tobytes(), np.uint8), cuda)
    got = to_host(ply.transcode(raw, 0, len(a), 13, 7, table)).reshape(-1)
    w = np.frombuffer(want.tobytes(), np.uint8)
    d = np.flatnonzero(got != w)
    assert d.size == 0, f"{src}: {d.size} bytes differ, first rows {np.unique(d // 7)[:8]}: " \
                        f"{vals[np.unique(d // 7)[:4]]}"


def test_round_trip_3dgs_cc_3dgs(cuda, gsx_lib, tmp_path):
    """3DGS file -> decode -> encode("cc") -> write_ply -> decode("cc") -> encode("3dgs"), against the oracle's chain,
    with RGB and extras riding along."""
    from gsx import ply, synth
    a = synth.structured(200_003, "mixed")
    rng = np.random.default_rng(3)
    extra = np.zeros(len(a), a.dtype.descr + [("red", "u1"), ("green", "u1"), ("blue", "u1"), ("conf", "<f8"),
                                               ("seg", "<i2")])
    for f in a.dtype.names:
        extra[f] = a[f]
    for f in ("red", "green", "blue"):
        extra[f] = rng.integers(0, 256, len(a))
    extra["conf"], extra["seg"] = rng.normal(size=len(a)), rng.integers(-300, 300, len(a))
    blob = po.file(po.write(extra, "3dgs"))
    cc = ply.encode(ply.decode(blob, "3dgs", cuda), "cc")
    p = tmp_path / "cc.ply"
    ply.write_ply(p, cc)
    want_cc = po.write(po.read(blob, "3dgs"), "cc")
    assert p.read_bytes() == po.file(want_cc)
    back = ply.encode(ply.decode(p, "cc", cuda), "3dgs", crop_sh=True)
    assert_same(back.to_host(), po.write(po.read(po.file(want_cc), "cc"), "3dgs", crop_sh=True), "3dgs again")


def test_filter_chain_end_to_end(cuda, gsx_lib, tmp_path):
    """decode(3DGS) -> records() -> FilterChain (bbox, alpha, density, SOR) -> DeviceRecords.gather -> encode("cc"),
    no host structured array in between, against the oracle's host chain."""
    import oracle
    from gsx import ply, synth
    from gsx.pipeline import FilterChain
    blob = po.file(po.write(synth.structured(300_000, "mixed"), "3dgs"))
    r = ply.decode(blob, "3dgs", cuda).records()
    xyz, op = r.xyz_opacity()
    ch = FilterChain(xyz, op, cuda)
    ch.crop_by_bbox(-11, -11, -11, 11, 11, 11)
    ch.alpha(5)
    ch.density(sensitivity=0.5, keep_multicluster=True)
    ch.sor(16, 2.0, hash_mode="i32wrap")
    enc = ply.encode(r.gather(ch.idx) if ch.idx is not None else r, "cc")
    ply.write_ply(tmp_path / "out.ply", enc)
    cur = po.read(blob, "3dgs")
    idx = np.arange(len(cur))
    for step in ("bbox", "alpha", "density", "sor"):
        c = cur[idx]
        pts = np.column_stack((c["x"], c["y"], c["z"]))
        if step == "bbox":
            m = oracle.bbox_mask(c["x"], c["y"], c["z"], -11, -11, -11, 11, 11, 11)
        elif step == "alpha":
            m = oracle.alpha_mask(c["opacity"], 5)
        elif step == "density":
            m = oracle.density_mask(pts, sensitivity=0.5, keep_multicluster=True)[0]
        else:
            m = oracle.sor_taichi_mask(pts, 16, 2.0)
        idx = idx[m]
    assert 0 < len(idx) < len(cur)
    want = po.write(cur[idx], "cc")
    assert_same(enc.to_host(), want, "chain")
    assert (tmp_path / "out.ply").read_bytes() == po.file(want)


class StandIn:
    def __init__(self):
        self.calls = []
        self.extra_elements = "untouched"

    def read(self, path, *args, **kwargs):
        self.calls.append(("read", path, args, kwargs))
        return "reference"

    def write(self, data, path, *args, **kwargs):
        self.calls.append(("write", path, args, kwargs))


def test_dropin_on_stand_in_classes(cuda, gsx_lib, tmp_path):
    from gsx import dropin, ply
    z = np.load(GOLDEN)
    for flavor in ("3dgs", "cc"):
        cls = type(f"StandIn_{flavor}", (StandIn,), {})
        for _ in range(2):                                     # idempotent
            dropin.install_reader(cls, ply.decode, after=dropin._vertex_only, flavor=flavor)
            dropin.install_writer(cls, ply.prepare_write, flavor=flavor)
        assert cls._gsx_reference_read is StandIn.read and cls._gsx_reference_write is StandIn.write
        assert cls.read is not StandIn.read and cls.write is not StandIn.write
        r = cls()
        good = z[f"read_{flavor}_extras_file"].tobytes()
        p = tmp_path / f"{flavor}.ply"
        p.write_bytes(good)
        got = r.read(str(p))
        assert r.calls == [] and r.extra_elements == []
        assert_same(got, po.read(good, flavor), "drop-in read")
        q = tmp_path / f"{flavor}_bad.ply"
        q.write_bytes(z["read_3dgs_refuse_camera_element_file"].tobytes())
        assert r.read(str(q), 7, level=4) == "reference"
        assert r.calls[-1] == ("read", str(q), (7,), {"level": 4})
        out = tmp_path / f"{flavor}_out.ply"
        r.write(got, str(out), crop_sh=True)
        assert len(r.calls) == 1 and out.read_bytes() == po.file(po.write(got, flavor, crop_sh=True))
        r.write(got, str(out), extra_elements=["camera"])      # kept elements: the reference's write
        assert r.calls[-1] == ("write", str(out), (), {"extra_elements": ["camera"]})
        bad = np.zeros(3, [("x", "<f4"), ("flag", "?")])
        r.write(bad, str(out), crop_sh=False)                   # refused: the reference's write
        assert r.calls[-1] == ("write", str(out), (), {"crop_sh": False}) and len(r.calls) == 3


def test_patch_refuses_unknown_ply_value(gsx_lib):
    from gsx import dropin
    with pytest.raises(ValueError):
        dropin.patch(ply="gpu", require_cuda=False)

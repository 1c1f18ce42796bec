"""GPU: the .splat / .ksplat / .spz / compressed PLY readers on the device (gsx.splat, gsx.ksplat, gsx.spz,
gsx.compressed_ply `decode`) against the reference readers' own results (g13) and the NumPy oracle
(readers_oracle.py) at 1 M splats, a device round trip through each writer, NumPy's float32 log over every float32 bit
pattern, every float16 pattern, and the drop-in readers."""
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

import readers_oracle as ro
import splat_codecs_oracle as sco

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
from make_readers_golden import cply_arrays, ksplat_file, ply_bytes, sec, spz_body  # noqa: E402
from test_readers_cpu import GOLDEN, golden_cases, meta_repr  # noqa: E402

pytestmark = pytest.mark.gpu


def decoders():
    from gsx import compressed_ply, ksplat, splat, spz
    return {"splat": splat.decode, "ksplat": ksplat.decode, "spz": spz.decode, "cply": compressed_ply.decode}


@pytest.mark.parametrize("case", golden_cases())
def test_device_matches_reference_golden(case, cuda, gsx_lib):
    z = np.load(GOLDEN)
    blob, fmt = z[f"{case}_file"].tobytes(), str(z[f"{case}_format"])
    dec = decoders()[fmt]
    if str(z[f"{case}_expect"]) == "refuse":
        with pytest.raises(ValueError):
            dec(blob, cuda)
        return
    d = dec(blob, cuda)
    a = d.to_host()
    b = np.ascontiguousarray(a).tobytes()
    assert str(a.dtype.descr) == str(z[f"{case}_dtype"]) and meta_repr(d.metadata) == str(z[f"{case}_meta"])
    if sco.digest(b) != str(z[f"{case}_sha256"]):
        with np.errstate(all="ignore"):
            want = np.ascontiguousarray(ro.READERS[fmt](blob)[0]).tobytes()
        diff = np.flatnonzero(np.frombuffer(b, np.uint8) != np.frombuffer(want, np.uint8))
        pytest.fail(f"{case}: {diff.size} bytes differ, first at {diff[:8]} (row {diff[:1] // a.dtype.itemsize})")


def assert_same(got: np.ndarray, want: np.ndarray, what: str):
    assert got.dtype == want.dtype and len(got) == len(want), what
    g, w = np.frombuffer(got.tobytes(), np.uint8), np.frombuffer(np.ascontiguousarray(want).tobytes(), np.uint8)
    d = np.flatnonzero(g != w)
    assert d.size == 0, f"{what}: {d.size} bytes differ, first at {d[:8]} (rows {d[:4] // got.dtype.itemsize})"


def check(fmt, blob, cuda):
    d = decoders()[fmt](blob, cuda)
    with np.errstate(all="ignore"):
        want, meta = ro.READERS[fmt](blob)
    assert_same(d.to_host(), want, fmt)
    assert meta_repr(d.metadata) == meta_repr(meta)


N = 1 << 20


def test_splat_at_scale(cuda, gsx_lib):
    rng = np.random.default_rng(1)
    check("splat", rng.integers(0, 256, N * 32 + 5, dtype=np.uint8).tobytes(), cuda)


@pytest.mark.parametrize("level", [0, 1, 2, 3])
def test_ksplat_at_scale(level, cuda, gsx_lib):
    s = [sec(N - 1000, 256, deg=2, maxn=N), sec(1000, 64, deg=1, partial=[10, 0, 990], fb=0)]
    check("ksplat", ksplat_file(level, s), cuda)


@pytest.mark.parametrize("version", [1, 2, 3])
def test_spz_at_scale(version, cuda, gsx_lib):
    check("spz", spz_body(version, N + 3, 3, seed=version), cuda)


def test_compressed_ply_at_scale(cuda, gsx_lib, tmp_path):
    arrays = cply_arrays(N + 17, (N + 17 + 255) // 256, 45, seed=3)
    check("cply", ply_bytes(tmp_path / "c.ply", *arrays), cuda)


def test_round_trip_through_each_writer(cuda, gsx_lib, tmp_path):
    """synth records -> device writer -> decode(file).records() -> the same writer, against the oracle writer applied
    to the oracle reader's output."""
    from gsx import compressed_ply, ksplat, records, splat, spz, synth
    import compressed_ply_oracle as cpo
    a = synth.structured(300_000, "mixed")
    r = records.DeviceRecords.from_structured(a, cuda)
    with np.errstate(all="ignore"):
        blob = splat.encode(r).to_host()
        got = splat.encode(splat.decode(blob, cuda).records()).to_host()
        assert got == sco.splat_file(ro.splat(blob)[0]), "splat"
        for lv in (0, 1, 2):
            blob = ksplat.encode(r, lv).to_host()
            got = ksplat.encode(ksplat.decode(blob, cuda).records(), lv).to_host()
            assert got == sco.ksplat_file(ro.ksplat(blob)[0], lv), f"ksplat level {lv}"
        payload = spz.encode(r).to_host()
        got = spz.encode(spz.decode(payload, cuda).records()).to_host()
        assert got == sco.spz_payload(ro.spz(payload)[0]), "spz"
        p = tmp_path / "c.ply"
        compressed_ply.write_ply(p, *compressed_ply.encode(r).to_host())
        dec = compressed_ply.decode(p, cuda)
        enc = compressed_ply.encode(dec.records())
        back = ro.compressed_ply(p.read_bytes())[0]
        cpo.assert_packed_equal(enc.to_host(), cpo.encode(back, enc.order.cpu().numpy()))


def test_numpy_logf_every_float32(cuda, gsx_lib):
    """Every float32 bit pattern through the .splat reader's scale fields (gsx_splat_decode on device-built records),
    compared with np.log(np.maximum(x, 1e-6)) on the host, NaN included."""
    import torch
    from gsx import splat
    from gsx._abi import check as gcheck, lib
    from gsx.hostcopy import to_host
    from gsx.readers import tables_on
    from gsx._abi import _ptr, _stream
    m = 1 << 24
    rec = torch.zeros((m, 32), dtype=torch.uint8, device=cuda)
    rows = torch.empty((m, 71), dtype=torch.uint8, device=cuda)
    tabs = tables_on(rec.device, *splat.read_tables())
    bad, start = 0, -(1 << 31)
    while start < (1 << 31):
        cnt = min(3 * m, (1 << 31) - start)
        k = (cnt + 2) // 3
        bits = torch.arange(start, start + 3 * k, dtype=torch.int64, device=cuda)
        bits = torch.where(bits < (1 << 31), bits, bits - (1 << 32)).to(torch.int32)
        rec[:k].view(torch.int32)[:, 3:6] = bits.view(k, 3)
        gcheck(lib.gsx_splat_decode(_ptr(rec), k, _ptr(tabs), _ptr(rows), _stream()), "gsx_splat_decode")
        got = to_host(rows[:k, 40:52].contiguous()).reshape(-1).view(np.uint32)[:cnt]   # scale_0 .. scale_2
        x = np.arange(start, start + cnt, dtype=np.int64).astype(np.int32).view(np.float32)
        with np.errstate(all="ignore"):
            want = np.log(np.maximum(x, 1e-6)).view(np.uint32)
        bad += int(np.count_nonzero(got != want))
        start += cnt
    assert bad == 0, f"{bad} of 2^32 float32 log values differ from np.log"


def test_every_float16_pattern(cuda, gsx_lib):
    """All 65 536 float16 patterns through ksplat level-1 scales and SH and SPZ v1 positions."""
    from gsx import ksplat, spz
    h = np.arange(65536, dtype=np.uint16)
    want = h.view(np.float16).astype(np.float32).view(np.uint32)
    recs = np.zeros((65536, 42), np.uint8)
    for k in range(3):
        recs[:, 6 + 2 * k:8 + 2 * k] = np.roll(h, k).view(np.uint8).reshape(-1, 2)
    for k in range(9):
        recs[:, 24 + 2 * k:26 + 2 * k] = np.roll(h, 3 + k).view(np.uint8).reshape(-1, 2)
    s = sec(65536, 1 << 20, deg=1, fb=0, partial=[65536])
    s["records"] = recs.tobytes()
    a = ksplat.decode(ksplat_file(1, [s]), cuda).to_host()
    for k in range(3):
        assert np.array_equal(a[f"scale_{k}"].view(np.uint32), np.roll(want, k)), k
    for k in range(9):
        assert np.array_equal(a[f"f_rest_{k}"].view(np.uint32), np.roll(want, 3 + k)), k
    body = spz_body(1, 65536, 0, seed=4, patterns=np.stack([h, np.roll(h, 1), np.roll(h, 2)], 1).tobytes())
    b = spz.decode(body, cuda).to_host()
    for k, f in enumerate("xyz"):
        assert np.array_equal(b[f].view(np.uint32), np.roll(want, k)), f


class StandIn:
    def __init__(self):
        self.calls = []
        self.metadata = "untouched"

    def read(self, path, *args, **kwargs):
        self.calls.append((path, args, kwargs))
        return "reference"


def test_dropin_reads_on_stand_in_classes(cuda, gsx_lib, tmp_path):
    from gsx import compressed_ply, dropin, ksplat, splat, spz
    z = np.load(GOLDEN)
    good = {"splat": "splat_writer_edge", "ksplat": "ksplat_multisection", "spz": "spz_writer_edge",
            "cply": "cply_order"}
    bad = {"ksplat": "ksplat_version", "spz": "spz_truncated", "cply": "cply_no_chunk"}
    for fmt, mod in (("splat", splat), ("ksplat", ksplat), ("spz", spz), ("cply", compressed_ply)):
        cls = type(f"StandIn_{fmt}", (StandIn,), {})
        dropin.install_reader(cls, mod.decode)
        dropin.install_reader(cls, mod.decode)                # idempotent
        assert cls._gsx_reference_read is StandIn.read and cls.read is not StandIn.read
        r = cls()
        p = tmp_path / fmt
        blob = z[f"{good[fmt]}_file"].tobytes()
        p.write_bytes(blob)
        got = r.read(str(p))
        with np.errstate(all="ignore"):
            want, meta = ro.READERS[fmt](blob)
        assert r.calls == [] and isinstance(got, np.ndarray)
        assert_same(got, want, fmt)
        assert r.metadata == ("untouched" if meta is None else meta) or meta_repr(r.metadata) == meta_repr(meta)
        if fmt in bad:   # refused: the original read, with the original arguments
            q = tmp_path / f"{fmt}.bad"
            q.write_bytes(z[f"{bad[fmt]}_file"].tobytes())
            assert r.read(str(q), 7, level=4) == "reference"
            assert r.calls == [(str(q), (7,), {"level": 4})]

"""GPU: the .ksplat / .spz / .splat writers on the device (gsx.ksplat, gsx.spz, gsx.splat) against the reference
writers' own files (g12) and the NumPy oracle (splat_codecs_oracle.py), the trailing-field upload, the drop-ins, and
NumPy's float32 exp over every float32 bit pattern."""
import gzip

import numpy as np
import pytest

import splat_codecs_oracle as sco
from test_splat_codecs_cpu import GOLDEN, TAGS

pytestmark = pytest.mark.gpu


def device_files(a, cuda, records=None):
    """{case: bytes} of the three device writers, or the exception type name for a refused case."""
    from gsx import ksplat, records as rec, splat, spz
    r = records if records is not None else rec.DeviceRecords.from_writer_input(a, cuda)
    jobs = {sco.ksplat_tag(c): (lambda c=c: ksplat.encode(r, *c).to_host()) for c in sco.KSPLAT_CASES}
    jobs["spz"] = lambda: spz.encode(r).to_host()
    jobs["splat"] = lambda: splat.encode(r).to_host()
    out = {}
    for k, job in jobs.items():
        try:
            out[k] = job()
        except ValueError as e:
            out[k] = type(e).__name__
    return out


@pytest.mark.parametrize("tag", TAGS)
def test_device_matches_reference_golden(tag, cuda, gsx_lib):
    z = np.load(GOLDEN)
    a = sco.golden_inputs()[tag]
    for name, got in device_files(a, cuda).items():
        key = f"{tag}_{name}"
        if f"{key}_raises" in z.files:
            assert got == "ValueError", key
            continue
        assert isinstance(got, bytes) and len(got) == int(z[f"{key}_len"]), key
        if sco.digest(got) != str(z[f"{key}_sha256"]):
            with np.errstate(all="ignore"):
                want = sco.ksplat_file(a, *next(c for c in sco.KSPLAT_CASES if sco.ksplat_tag(c) == name)) \
                    if name.startswith("ksplat") else sco.spz_payload(a) if name == "spz" else sco.splat_file(a)
            d = np.flatnonzero(np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8))
            pytest.fail(f"{key}: {d.size} bytes differ, first at {d[:8]}")


def assert_same(got: bytes, want: bytes, what: str):
    assert len(got) == len(want), what
    g, w = np.frombuffer(got, np.uint8), np.frombuffer(want, np.uint8)
    d = np.flatnonzero(g != w)
    assert d.size == 0, f"{what}: {d.size} bytes differ, first at {d[:8]}"


def check_against_oracle(a, cuda):
    got = device_files(a, cuda)
    with np.errstate(all="ignore"):
        for c in sco.KSPLAT_CASES:
            assert_same(got[sco.ksplat_tag(c)], sco.ksplat_file(a, *c), sco.ksplat_tag(c))
        assert_same(got["spz"], sco.spz_payload(a), "spz")
        assert_same(got["splat"], sco.splat_file(a), "splat")
    return got


def test_300k_mixed(cuda, gsx_lib):
    from gsx import synth
    check_against_oracle(synth.structured(300_000, "mixed"), cuda)


def test_edge_cloud_at_scale(cuda, gsx_lib):
    """The golden's edge rows spread over a 100 k cloud: NaN / inf rows in many CTAs and buckets."""
    from gsx import synth
    a = synth.structured(100_003, "mixed")
    edge = sco.golden_inputs()["mixed3"][:200]
    for k in range(0, len(a) - 200, 9_973):
        a[k:k + 200] = edge
    check_against_oracle(a, cuda)


def test_splat_order_is_stable_argsort(cuda, gsx_lib):
    from gsx import records, splat, synth
    a = synth.structured(50_000, "mixed")
    a["scale_0"][::3], a["opacity"][::3] = -4.0, 0.5          # a third of the rows share one metric
    a["opacity"][7::11] = np.nan
    enc = splat.encode(records.DeviceRecords.from_structured(a, cuda))
    assert np.array_equal(enc.order.cpu().numpy(), sco.splat_order(a))


def with_rgb(a):
    """`a` with the converter's trailing red/green/blue u1 fields (converter.py:244-253)."""
    dt = a.dtype.descr + [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    b = np.zeros(len(a), dtype=dt)
    for f in a.dtype.names:
        b[f] = a[f]
    b["red"], b["green"], b["blue"] = 7, 8, 9
    return b


def test_trailing_rgb_fields_do_not_change_the_bytes(cuda, gsx_lib):
    from gsx import records, synth
    a = synth.structured(20_001, "mixed")
    b = with_rgb(a)
    assert not records.is_packed_f32(b)
    r = records.DeviceRecords.from_writer_input(b, cuda)
    assert r.names == a.dtype.names
    assert np.array_equal(r.rows.cpu().numpy().view(np.uint32), a.view(np.float32).reshape(len(a), -1).view(np.uint32))
    assert device_files(b, cuda) == device_files(a, cuda)
    # a non-float32 field between float32 fields, and a field at an odd byte offset
    c = np.zeros(len(a), dtype=[("tag", "u1")] + a.dtype.descr[:5] + [("pad", "<i2")] + a.dtype.descr[5:])
    for f in a.dtype.names:
        c[f] = a[f]
    assert device_files(c, cuda) == device_files(a, cuda)


class StandIn:
    def __init__(self):
        self.calls = []

    def write(self, data, path, *args, **kwargs):
        self.calls.append((data, path, args, kwargs))


def test_dropin_writes_on_stand_in_classes(cuda, gsx_lib, tmp_path):
    from gsx import dropin, ksplat, splat, spz, synth
    a = with_rgb(synth.structured(3_000, "mixed"))
    plain = sco.golden_inputs()["fields0"]
    for mod in (ksplat, spz, splat):
        cls = type(f"StandIn_{mod.__name__}", (StandIn,), {})
        opts = {"gzip": "host"} if mod is spz else {}
        dropin.install_writer(cls, mod.prepare_write, **opts)
        dropin.install_writer(cls, mod.prepare_write, **opts)         # idempotent
        assert cls._gsx_reference_write is StandIn.write and cls.write is not StandIn.write
        w = cls()
        p = tmp_path / mod.__name__
        if mod is ksplat:
            w.write(a, p, 2, bucket_size=7, sh_level=1)
            want = sco.ksplat_file(a, 2, 1, 7)
        elif mod is spz:
            w.write(a, p, compression_level=6)
            want = sco.spz_payload(a)
        else:
            w.write(a, p)
            with np.errstate(all="ignore"):
                want = sco.splat_file(a)
        assert w.calls == []
        got = p.read_bytes()
        assert_same(gzip.decompress(got) if mod is spz else got, want, mod.__name__)
        # refused: a missing field -> the original write, with the original arguments
        b = plain[[f for f in plain.dtype.names if f != "rot_3"]]
        args = (3,) if mod is ksplat else ()
        w.write(b, "b.out", *args, level=4)
        assert len(w.calls) == 1 and w.calls[0][0] is b and w.calls[0][1:] == ("b.out", args, {"level": 4})
    # the degree-1 field set with SH content: the reference SPZ writer raises, and so does the drop-in's fallback
    cls = type("StandInSpz", (StandIn,), {})
    dropin.install_writer(cls, spz.prepare_write, gzip="host")
    w = cls()
    d1 = sco.golden_inputs()["fields1"]
    w.write(d1, tmp_path / "d1.spz", compression_level=0)
    assert len(w.calls) == 1 and w.calls[0][0] is d1 and w.calls[0][3] == {"compression_level": 0}


def test_numpy_expf_every_float32(cuda, gsx_lib):
    """Every float32 bit pattern through the product path: the scale fields of ksplat level 0 hold the raw float32
    exp bytes, in row order.  Compared with np.exp on the host, NaN included."""
    import torch
    from gsx import ksplat, records
    from gsx.compressed_ply import PACK_FIELDS
    from gsx.hostcopy import to_host
    m = 1 << 24                                        # rows per chunk: 3 * 2^24 values
    rows = torch.zeros((m, 14), dtype=torch.float32, device=cuda)
    s0 = PACK_FIELDS.index("scale_0")
    bad, start, total = 0, -(1 << 31), 1 << 32
    while start < (1 << 31):
        cnt = min(3 * m, (1 << 31) - start)
        k = (cnt + 2) // 3
        bits = torch.arange(start, start + 3 * k, dtype=torch.int64, device=cuda)
        bits = torch.where(bits < (1 << 31), bits, bits - (1 << 32)).to(torch.int32)
        rows[:k, s0:s0 + 3] = bits.view(torch.float32).view(k, 3)
        enc = ksplat.encode(records.DeviceRecords(rows[:k], PACK_FIELDS, None), 0)
        got = to_host(enc.records[:, 12:24].contiguous()).reshape(-1).view(np.uint32)[:cnt]
        x = (np.arange(start, start + cnt, dtype=np.int64).astype(np.int32)).view(np.float32)
        with np.errstate(all="ignore"):
            want = np.exp(x).view(np.uint32)
        bad += int(np.count_nonzero(got != want))
        start += cnt
    assert start - (-(1 << 31)) == total
    assert bad == 0, f"{bad} of 2^32 float32 exp values differ from np.exp"

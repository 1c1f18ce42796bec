"""GPU: gsx.deflate's .gz files against the NumPy restatement (deflate_oracle.py), byte for byte, their CRC-32 against
zlib, a payload past 2^32 bytes, and the .spz writers that gzip on the device."""
import gzip
import zlib

import numpy as np
import pytest

import deflate_oracle as do
import splat_codecs_oracle as sco

pytestmark = pytest.mark.gpu

CASES = do.cases()


def device_gzip(x, cuda, level, breaks=(), mtime=0):
    import torch
    from gsx import deflate
    return deflate.gzip(torch.from_numpy(np.ascontiguousarray(x)).to(cuda), level, mtime=mtime, breaks=breaks)


def check(x, cuda, level, breaks=()):
    want = do.gzip_file(x, level, 0, breaks)
    got = device_gzip(x, cuda, level, breaks)
    if got != want:
        diff = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
        raise AssertionError(f"device file ({len(got)} B) differs from the oracle's ({len(want)} B) at byte {diff}")
    assert got[-8:-4] == zlib.crc32(x).to_bytes(4, "little")
    assert gzip.decompress(got) == x.tobytes()


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("level", [0, 1, 9])
def test_device_bytes_equal_oracle(name, level, cuda, gsx_lib):
    x, breaks = CASES[name]
    check(x, cuda, level, breaks)


@pytest.mark.parametrize("n", do.STORED_SIZES)
def test_stored_sizes(n, cuda, gsx_lib):
    check(np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8), cuda, 0)


SIZES = (4095, 4096, 4097, 8191, 8193, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, (2 << 20) + 4099)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["random", "runs"])
def test_random_payloads_around_tile_and_block(n, kind, cuda, gsx_lib):
    rng = np.random.default_rng(n)
    if kind == "random":
        x = rng.integers(0, 256, n, dtype=np.uint8)
    else:   # runs of 1..600 equal bytes: some cross the 4 KiB tiles, the 1 MiB blocks and the break
        lens = rng.integers(1, 600, n // 2 + 1)
        x = np.repeat(rng.integers(0, 6, len(lens), dtype=np.uint8), lens)[:n]
    check(x, cuda, 6, (n // 3,))


def test_crc_equals_zlib(cuda, gsx_lib):
    import torch
    from gsx import deflate
    rng = np.random.default_rng(32)
    for n in (0, 1, 15, 16, 17, 4095, 4096, 4097, 65536 * 3 + 7, 5_000_011):
        x = rng.integers(0, 256, n + 3, dtype=np.uint8)
        t = torch.from_numpy(x).to(cuda)[3:]          # an input that is not 16-byte aligned
        f = deflate.gzip(t, 0, mtime=0)
        assert f[-8:] == zlib.crc32(x[3:]).to_bytes(4, "little") + n.to_bytes(4, "little")


def spz_payloads():
    from gsx import synth
    out = {}
    for tag, a in sco.golden_inputs().items():
        out[f"g12_{tag}"] = a
    for n in (100_000, 1_000_000):
        for d in range(4):
            out[f"synth_{n}_sh{d}"] = synth.structured(n, "mixed", d)
        a = synth.structured(n, "mixed", 3)
        zero = np.random.default_rng(2024).random(n) < 0.9
        for i in range(45):
            a[f"f_rest_{i}"][zero] = 0
        out[f"synth_{n}_sparse"] = a
    return out


def test_spz_payloads_equal_oracle(cuda, gsx_lib):
    from gsx import records, spz
    checked = 0
    for name, a in spz_payloads().items():
        try:
            enc = spz.encode(records.DeviceRecords.from_writer_input(a, cuda))
        except ValueError:
            continue
        x = enc.payload.cpu().numpy()
        for level in (0, 6):
            got = enc.compress(level, mtime=0)
            want = do.gzip_file(x, level, 0, enc.sections())
            assert got == want, (name, level)
        checked += 1
    assert checked >= 14


def test_payload_past_2_to_32(cuda, gsx_lib):
    """4 GiB + 12345 bytes made on the device from a seed: runs of 128 equal bytes, every 64th MiB random."""
    import torch
    from gsx import deflate
    n, step = (1 << 32) + 12345, 1 << 26

    def chunk(lo, hi, dev):
        i = torch.arange(lo, hi, dtype=torch.int64, device=dev)
        runs = ((i >> 7) * 2654435761 + 12345) >> 11
        noise = (i * 6364136223846793005 + 1442695040888963407) >> 33
        return torch.where(((i >> 20) & 63) == 5, noise, runs).to(torch.uint8)

    x = torch.empty(n, dtype=torch.uint8, device=cuda)
    for lo in range(0, n, step):
        x[lo:min(n, lo + step)] = chunk(lo, min(n, lo + step), cuda)
    f = deflate.gzip(x, 6, mtime=0, breaks=(16, 1 << 32))
    del x
    torch.cuda.empty_cache()
    d = zlib.decompressobj(-15)
    crc, at, src = 0, 0, memoryview(f)[10:-8]
    while not d.eof:
        out = d.decompress(src, step)
        src = d.unconsumed_tail
        want = chunk(at, at + len(out), cuda).cpu().numpy().tobytes()
        assert out == want, f"bytes {at}..{at + len(out)} differ"
        crc = zlib.crc32(want, crc)
        at += len(out)
        assert out or src or d.eof, "the stream ends before its final block"
    assert d.eof and at == n
    assert f[-8:] == crc.to_bytes(4, "little") + (n & 0xFFFFFFFF).to_bytes(4, "little")
    assert int.from_bytes(f[-4:], "little") == 12345


def test_write_spz_device_reads_back(cuda, gsx_lib, tmp_path):
    from gsx import records, spz, synth
    a = synth.structured(20_000, "mixed", 3)
    enc = spz.encode(records.DeviceRecords.from_writer_input(a, cuda))
    for level in (0, 1, 9):
        spz.write_spz(tmp_path / "host.spz", enc, level)
        spz.write_spz(tmp_path / "dev.spz", enc, level, where="device")
        host, dev = (tmp_path / "host.spz").read_bytes(), (tmp_path / "dev.spz").read_bytes()
        assert gzip.decompress(host) == gzip.decompress(dev)
        assert host[8:10] == dev[8:10]                 # XFL and OS: CPython's header at this level
        ra, rb = spz.decode(tmp_path / "host.spz", cuda), spz.decode(tmp_path / "dev.spz", cuda)
        assert bytes(ra.rows.cpu().numpy()) == bytes(rb.rows.cpu().numpy())
    with pytest.raises(ValueError):
        spz.write_spz(tmp_path / "x.spz", enc, 6, where="gpu")


def test_dropin_write_device_gzip_on_stand_in_class(cuda, gsx_lib, tmp_path):
    from gsx import dropin, spz, synth

    class StandIn:
        def write(self, data, path, **kwargs):
            raise AssertionError("the original write must not run for packed float32 records")

    class HostGzip:
        def write(self, data, path, **kwargs):
            raise AssertionError("the original write must not run for packed float32 records")

    dropin.install_writer(StandIn, spz.prepare_write, gzip="device")
    dropin.install_writer(HostGzip, spz.prepare_write, gzip="host")
    a = synth.structured(3_000, "mixed")
    StandIn().write(a, tmp_path / "dev.spz", compression_level=6)
    HostGzip().write(a, tmp_path / "host.spz", compression_level=6)
    dev, host = (tmp_path / "dev.spz").read_bytes(), (tmp_path / "host.spz").read_bytes()
    assert dev != host and gzip.decompress(dev) == gzip.decompress(host)
    ra, rb = spz.decode(tmp_path / "dev.spz", cuda), spz.decode(tmp_path / "host.spz", cuda)
    assert bytes(ra.rows.cpu().numpy()) == bytes(rb.rows.cpu().numpy())


def test_refusals(cuda, gsx_lib):
    import torch
    from gsx import deflate
    x = torch.zeros(10, dtype=torch.uint8, device=cuda)
    for bad in (-2, 10):
        with pytest.raises(ValueError):
            deflate.gzip(x, bad)
    with pytest.raises(ValueError):
        deflate.gzip(x.float(), 6)
    with pytest.raises(ValueError):
        deflate.gzip(x.cpu(), 6)
    with pytest.raises(ValueError):
        deflate.gzip(x, 6, breaks=(5, 3))

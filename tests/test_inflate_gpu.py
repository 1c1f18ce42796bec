"""GPU: gsx.deflate.gunzip against gzip.decompress, byte for byte or by exception class, over the seeded corpus of
inflate_model.py (zlib levels, strategies, memLevels, window bits and flushes, gsx's encoder, multi-member files,
header flags, the finder's decoys, hand-built malformed members, truncations, bit flips) at several chunk sizes; the
device's chain against the model's; SPZ payloads of 1 M synth splats; a payload past 2^32 bytes; and gsx.spz.decode
of gzipped files against the reference rows."""
import gzip
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

import inflate_model as m

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
from make_readers_golden import spz_body  # noqa: E402
from test_readers_gpu import check as check_reader  # noqa: E402

pytestmark = pytest.mark.gpu


def gunzip(data, cuda, chunk_bytes=None, stats=None):
    from gsx import deflate
    from gsx.hostcopy import to_host
    try:
        return to_host(deflate.gunzip(data, cuda, chunk_bytes, stats)).tobytes()
    except (EOFError, gzip.BadGzipFile, zlib.error) as e:
        return type(e)


@pytest.fixture(scope="module")
def corpus():
    c = m.streams()
    c.update(m.malformed())
    c.update(m.corrupted())
    return {k: (v, m.expect(v)) for k, v in c.items()}


@pytest.mark.parametrize("chunk_bytes", [64, 333, 4096, None])
def test_gunzip_equals_gzip(corpus, chunk_bytes, cuda, gsx_lib):
    bad = []
    for name, (data, want) in corpus.items():
        got = gunzip(data, cuda, chunk_bytes)
        if got != want:
            bad.append((name, got if isinstance(got, type) else len(got),
                        want if isinstance(want, type) else len(want)))
    assert not bad, f"chunk_bytes {chunk_bytes}: {bad[:10]} ({len(bad)} cases)"


def test_device_chain_equals_model(corpus, cuda, gsx_lib):
    """The device verifies the same chain as the model: the same (start, stop) bit of every piece."""
    for name in ("text_l6", "records_gsx6", "decoy_stored_zlib", "zeros_l9", "period32769_l1", "text_fixed",
                 "multi_member", "random_l0"):
        data = corpus[name][0]
        for cb in (64, 1024):
            want, got = {}, {}
            m.gunzip(data, cb, want)
            gunzip(data, cuda, cb, got)
            assert got["chain"] == want["chain"], (name, cb)
            assert got["chunks"] == want["chunks"], (name, cb)


def test_tensor_input(cuda, gsx_lib):
    import torch
    data = m.streams()["multi_member"]
    t = torch.from_numpy(np.frombuffer(data, np.uint8).copy()).to(cuda)
    assert gunzip(t, cuda, 256) == gzip.decompress(data)


@pytest.fixture(scope="module")
def spz_payload(cuda):
    from gsx import records, spz, synth
    a = synth.structured(1 << 20, "mixed", 3)
    return spz.encode(records.DeviceRecords.from_writer_input(a, cuda)).to_host()


@pytest.mark.parametrize("level", [1, 6])
def test_spz_payload_1m(spz_payload, level, cuda, gsx_lib):
    blob = gzip.compress(spz_payload, level, mtime=0)
    assert gunzip(blob, cuda) == spz_payload


def test_gsx_gzip_spz_payload(spz_payload, cuda, gsx_lib):
    """gsx's own encoder: 1 MiB dynamic blocks, many chunks with no block boundary in them."""
    import torch
    from gsx import deflate
    blob = deflate.gzip(torch.from_numpy(np.frombuffer(spz_payload, np.uint8).copy()).to(cuda), 6)
    st = {}
    assert gunzip(blob, cuda, 4096, st) == spz_payload
    assert st["chunks"] > 1000


@pytest.mark.parametrize("level", [0, 6])
def test_past_4gib(level, cuda, gsx_lib):
    """64-bit sizes and offsets: 2^32 + 12345 bytes through gsx.deflate.gzip and back, compared on the device; the
    trailer's ISIZE is the size mod 2^32."""
    import torch
    from gsx import deflate
    n = (1 << 32) + 12345
    x = torch.empty(n, dtype=torch.uint8, device=cuda)
    for s in range(0, n, 1 << 28):                  # skewed bytes with short runs, not periodic; built in slices
        i = torch.arange(s, min(s + (1 << 28), n), device=cuda, dtype=torch.int64)
        x[s:s + len(i)] = (((i * 2654435761) >> 13) % 16 + (i // 5) % 3).to(torch.uint8)
    del i
    blob = deflate.gzip(x, level)
    out = deflate.gunzip(blob, cuda)
    assert out.numel() == n and torch.equal(out, x)


@pytest.mark.parametrize("level", [0, 1, 9])
def test_spz_decode_gzipped(level, cuda, gsx_lib):
    """gsx.spz.decode gunzips on the device: the rows equal the reference reader's (readers_oracle)."""
    check_reader("spz", gzip.compress(spz_body(3, (1 << 20) + 3, 3, seed=level), level, mtime=0), cuda)
    check_reader("spz", gzip.compress(spz_body(2, 5000, 1, seed=level), level, mtime=0), cuda)

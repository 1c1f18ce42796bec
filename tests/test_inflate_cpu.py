"""CPU: the chunked DEFLATE decoder's model (inflate_model.py) against gzip.decompress over the seeded corpus -- zlib
levels, strategies, memLevels, window bits and flushes, gsx's own encoder, multi-member files, header flags, the
finder's decoys, hand-built malformed members, truncations and bit flips -- at chunk sizes from 64 B to 64 KiB: the
same bytes, or the same exception class."""
import re

import pytest

import inflate_model as m

CHUNKS = (64, 256, 1024, 4096, 65536)


@pytest.fixture(scope="module")
def corpus():
    c = m.streams(8000)
    c.update(m.malformed())
    c.update(m.corrupted())
    return {k: (v, m.expect(v)) for k, v in c.items()}


@pytest.mark.slow
@pytest.mark.parametrize("chunk_bytes", CHUNKS)
def test_model_equals_gzip(corpus, chunk_bytes):
    bad = []
    for name, (data, want) in corpus.items():
        try:
            got = m.gunzip(data, chunk_bytes)
        except (EOFError, m.gzip.BadGzipFile, m.zlib.error) as e:
            got = type(e)
        if got != want:
            bad.append(name)
    assert not bad, f"chunk_bytes {chunk_bytes}: {bad}"


def test_chain_stats():
    """Many chunks without a block boundary (gsx's 1 MiB blocks) need no re-decode, and an all-zero payload that
    overflows the first capacity takes the overflow path."""
    data = m.streams(8000)
    st = {}
    assert m.gunzip(data["text_gsx6"], 64, st) == m.expect(data["text_gsx6"])
    assert st["chunks"] > 10 and st["redecoded"] == 0
    st = {}
    z = m.gz(m.raw_deflate(bytes(200_000), 9))
    assert m.gunzip(z, 64, st) == bytes(200_000)
    assert st["overflow_reruns"] > 0


def test_model_is_test_only():
    """The product never imports the model."""
    from pathlib import Path
    pkg = Path(__file__).resolve().parent.parent / "3dgsconverter_b200"
    imports = re.compile(r"^\s*(import|from)\s+\S*inflate_model", re.M)
    assert not [p for p in pkg.rglob("*.py") if imports.search(p.read_text())]


def test_malformed_cases_hit_their_check():
    """Each hand-built member fails the zlib check it is named after (zlib's message), so the decoder's copy of that
    check is what refuses it."""
    want = {"block_type_3": "invalid block type", "stored_nlen": "invalid stored block lengths",
            "fixed_lit_286": "invalid literal/length code", "fixed_lit_287": "invalid literal/length code",
            "fixed_dist_30": "invalid distance code", "fixed_dist_31": "invalid distance code",
            "too_many_lengths": "too many length or distance symbols",
            "too_many_distances": "too many length or distance symbols",
            "cl_oversubscribed": "invalid code lengths set", "cl_incomplete": "invalid code lengths set",
            "repeat_first": "invalid bit length repeat", "repeat_past_end": "invalid bit length repeat",
            "missing_eob": "invalid code -- missing end-of-block",
            "lit_oversubscribed": "invalid literal/lengths set", "lit_incomplete": "invalid literal/lengths set",
            "dist_incomplete": "invalid distances set", "dist_oversubscribed": "invalid distances set",
            "far_chunk0": "invalid distance too far back", "far_later_chunk": "invalid distance too far back"}
    cases = m.malformed()
    for name, msg in want.items():
        with pytest.raises(m.zlib.error, match=re.escape(msg)):
            m.gzip.decompress(cases[name])
        with pytest.raises(m.zlib.error):
            m.gunzip(cases[name], 64)


def test_first_block_stored():
    """spz.decode gunzips on the host exactly when the first member starts with a stored block (zlib level 0)."""
    from gsx.deflate import first_block_stored
    text = m.payloads(4000)["text"]
    assert first_block_stored(m.gzip.compress(text, 0))
    assert not any(first_block_stored(m.gzip.compress(text, level)) for level in (1, 6, 9))
    assert first_block_stored(m.gz(m.raw_deflate(text, 0), 31, b"x", b"name", b"comment"))
    assert not first_block_stored(b"\x1f\x8b\x08")                  # cut short: the device path raises EOFError
    assert not first_block_stored(m.gzip.compress(b"", 6)[:10])

"""CPU: deflate_oracle's .gz files (the restatement of gsx.deflate) decompress to their input with CPython's gzip and
raw zlib, their headers are CPython's, and on SPZ payloads they are no larger than zlib's levels 6 and 1."""
import gzip
import zlib

import numpy as np
import pytest

import deflate_oracle as do
import splat_codecs_oracle as sco
import webp_oracle as wo

CASES = do.cases()


def roundtrip(x, level, breaks=(), info=None):
    f = do.gzip_file(x, level, 0, breaks, info)
    assert gzip.decompress(f) == x.tobytes()
    d = zlib.decompressobj(-15)
    assert d.decompress(f[10:-8]) == x.tobytes() and d.eof and d.unused_data == b""
    return f


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("level", [0, 1, 6])
def test_oracle_files_decompress(name, level):
    x, breaks = CASES[name]
    roundtrip(x, level, breaks)


@pytest.mark.parametrize("n", do.STORED_SIZES)
def test_stored_block_sizes(n):
    x = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8)
    f = roundtrip(x, 0)
    assert len(f) == 10 + 5 * max(1, -(-n // 65535)) + n + 8


def test_runs_become_copies_at_four():
    for r, copies in ((3, 0), (258, 1), (259, 1), (260, 1), (262, 1)):
        info = {}
        roundtrip(CASES[f"run_{r}"][0], 6, info=info)
        assert info["copies"] == [copies], r
    x = np.full(100_000, 4, np.uint8)
    info = {}
    f = roundtrip(x, 6, info=info)
    assert info["copies"] == [1] and len(f) < 1000


def test_blocks_cut_at_breaks_and_every_mib():
    assert do.block_starts(0) == [0]
    assert do.block_starts(10, (0, 0, 3, 3, 10, 10)) == [0, 3]
    assert do.block_starts(3 << 20, (5,)) == [0, 5, 5 + (1 << 20), 5 + (2 << 20)]
    info = {}
    roundtrip(CASES["run_across_1mib"][0], 6, CASES["run_across_1mib"][1], info=info)
    assert len(info["copies"]) == 2 and info["copies"] == [1, 1]
    info = {}
    roundtrip(CASES["run_across_break"][0], 6, CASES["run_across_break"][1], info=info)
    assert len(info["copies"]) == 3


def test_length_limit_and_code_length_codes():
    x = CASES["fibonacci"][0]
    counts = np.bincount(x, minlength=286)
    counts[256] = 1
    assert wo.huffman_lengths(counts, 99).max() > 15          # the floor loop has to run
    info = {}
    roundtrip(x, 6, info=info)
    assert 0 < info["lit_len"][0].max() <= 15
    info = {}
    roundtrip(CASES["code_length_runs"][0], 6, info=info)
    syms = {s for s, _ in info["runs"][0]}
    assert {16, 17, 18} <= syms
    assert (18, 138 - 11) in info["runs"][0]


@pytest.mark.parametrize("level", range(-1, 10))
@pytest.mark.parametrize("mtime", [0, 1, 2**32 - 1])
def test_header_is_cpythons(level, mtime):
    want = gzip.compress(b"", level, mtime=mtime)[:10]
    assert do.header(level, mtime) == want
    from gsx import deflate
    assert deflate.header(level, mtime) == want


def test_levels_outside_zlib_refused():
    from gsx import deflate
    for bad in (-2, 10, 1.0, True, "6"):
        with pytest.raises(ValueError):
            deflate.header(bad, 0)
    with pytest.raises(ValueError):
        deflate.blocks(10, (4, 2))
    with pytest.raises(ValueError):
        deflate.blocks(10, (11,))
    assert deflate.blocks(3 << 20, (5,)).tolist() == do.block_starts(3 << 20, (5,))


def spz_payload(n, sparse=False):
    from gsx import synth
    a = synth.structured(n, "mixed", 3)
    if sparse:
        zero = np.random.default_rng(2024).random(n) < 0.9
        for i in range(45):
            a[f"f_rest_{i}"][zero] = 0
    return np.frombuffer(sco.spz_payload(a), np.uint8)


def spz_breaks(x, dim=15):
    n = (len(x) - 16) // (20 + 3 * dim)
    return tuple(np.cumsum([16, 9 * n, n, 3 * n, 3 * n, 4 * n]).tolist())


@pytest.mark.slow
@pytest.mark.parametrize("n, sparse, zlib_level", [(1_000_000, False, 6), (300_000, True, 1)])
def test_size_against_zlib_on_spz_payloads(n, sparse, zlib_level):
    """Recorded: 1 M mixed SH-3, 0.5157 of the payload (zlib level 6: 0.5590); 300 k sparse SH-3 (90 % of the splats
    with zero f_rest), 0.2975 (zlib level 1: 0.3165)."""
    x = spz_payload(n, sparse)
    f = roundtrip(x, 6, spz_breaks(x))
    z = gzip.compress(x.tobytes(), zlib_level, mtime=0)
    print(f"n={n} sparse={sparse}: gsx {len(f) / len(x):.4f}, zlib level {zlib_level} {len(z) / len(x):.4f}")
    assert len(f) <= len(z)


def test_dropin_patch_spz_gzip_option():
    from gsx import dropin
    with pytest.raises(ValueError):
        dropin.patch(spz_gzip="device")                           # needs codecs="device"
    with pytest.raises(ValueError):
        dropin.patch(codecs="device", spz_gzip="cuda")
    with pytest.raises(ValueError):
        dropin.patch(codecs="host", spz_gzip="device")

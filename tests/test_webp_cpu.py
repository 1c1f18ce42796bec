"""CPU: the NumPy restatement of the lossless WebP encoder (webp_oracle.py) writes files that Pillow decodes to the
input with RGB cleared where alpha is 0, for every shape and symbol statistic the device encoder is tested on."""
import io

import numpy as np
import pytest

import webp_oracle as wo

CASES = wo.cases()


def decode(data: bytes) -> np.ndarray:
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    assert im.format == "WEBP"
    return np.asarray(im.convert("RGBA"))


def expected(img: np.ndarray) -> np.ndarray:
    out = img.copy()
    out[out[..., 3] == 0, :3] = 0
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_file_decodes_to_input(name):
    img = CASES[name]
    info = {}
    data = wo.encode(img, info=info)
    assert data[:4] == b"RIFF" and data[8:16] == b"WEBPVP8L" and int.from_bytes(data[4:8], "little") == len(data) - 8
    assert np.array_equal(decode(data), expected(img))
    if name in wo.WINNERS:
        assert info["candidate"] == wo.WINNERS[name], info["bits"]
    assert info["bits"][info["candidate"]] == min(info["bits"])


def test_sog_textures_decode():
    for name, img in wo.sog_textures().items():
        assert np.array_equal(decode(wo.encode(img)), expected(img)), name


def test_constant_image_codes_take_no_bits():
    info = {}
    wo.encode(CASES["constant"], info=info)
    assert info["candidate"] == 0
    img = wo.Image(wo.to_argb(CASES["constant"]))
    # red, blue, alpha and distance: one symbol each, a simple code read with 0 bits
    for t in img.trees[1:]:
        assert t[0].parts[:2] == [(1, 1), (0, 1)] and not t[1].any()
    assert img.tok.max() == img.tok.size - 1           # one literal, then one copy of the rest


def test_two_symbol_trees_are_simple():
    img = wo.Image(wo.to_argb(CASES["two_symbols"]))
    for t in img.trees[1:4]:
        assert t[0].parts[0] == (1, 1) and t[0].parts[1] == (1, 1)     # simple code, two symbols


def test_fibonacci_histogram_hits_the_length_limit():
    img = wo.Image(wo.to_argb(CASES["fibonacci"]))
    assert max(int(t[1].max()) for t in img.trees) <= 15
    assert max(int(wo.huffman_lengths(h, 64).max()) for h in img.hist) > 15


def test_long_runs_split_at_4096_and_cross_rows():
    img = wo.Image(wo.to_argb(CASES["long_run"]))
    heads = img.tok[img.tok >= 3]
    assert heads.max() == wo.MAX_COPY and len(heads) >= 2
    rows = wo.Image(wo.to_argb(CASES["runs_across_rows"]))
    starts = np.nonzero(rows.tok >= 3)[0]
    assert any((s % 7) + rows.tok[s] > 7 for s in starts)


def test_some_tokens_straddle_three_words():
    """Tokens of the Fibonacci image reach 60 bits, so some span three 32-bit words of the emit buffer."""
    info = {}
    data = wo.encode(CASES["fibonacci"], info=info)
    bits = info["pixel_bits"]
    header = info["bits"][info["candidate"]] - int(bits.sum())
    off = 160 + header + np.concatenate([[0], np.cumsum(bits)[:-1]])
    words = (off + bits - 1) // 32 - off // 32 + 1
    assert len(data) > 0 and (words[bits > 0] == 3).any() and (words[bits > 0] == 2).any()


def test_length_prefix_codes():
    code, nbits, extra = wo.length_prefix(np.arange(1, 4097))
    for L, c, n, e in zip(range(1, 4097), code, nbits, extra):
        if c < 4:
            assert L == c + 1 and n == 0
        else:
            off = (2 + (c & 1)) << ((c - 2) >> 1)
            assert n == (c - 2) >> 1 and L == off + e + 1
    assert code.max() == 23


def test_refuses_oversize():
    with pytest.raises(ValueError):
        wo.encode(np.zeros((1, 16385, 4), np.uint8))

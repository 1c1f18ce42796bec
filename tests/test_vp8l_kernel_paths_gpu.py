"""The VP8L decoder's paths (csrc/gsx_vp8l.cu, gsx/webp_decode.py), one hand-built stream each: a colour-cached
sub-image whose first token reads the empty cache, more prefix-code groups than the first header workspace holds,
a job's token capacity overflowing, the 2048-entry colour cache, the predictor's modes 14 and 15, and copy chains as
deep as the image under k_vp8l_jump.  Then the prefix codes (simple codes in both forms and with a symbol past the
distance alphabet, lengths past the 8-bit table in every alphabet, one used symbol at lengths 1..15, a one-symbol
code-length code, max_symbol, repeats before the first length and ending at the alphabet), cache bits 1..11 and the
refused values, transform tiles at bits 2..9 on ragged widths, every palette bundling, a palette index past the
palette, a palette under the other three transforms, the predictor wavefront over heights and widths at its edges,
the rightmost column's TR under every mode, the entropy image (bits 2..9, group 300, gaps), all 120 plane codes at
widths 1..9 and cache tokens and copies across 32-bit chunks.

Each case has a seeded builder (vp8l_model.compose).  An unmarked CPU test proves through vp8l_model (its Header and
COUNTERS) that the stream has the feature the case is named after, and that the model decodes it to Pillow's pixels:
the model restates the decoder, so only Pillow, which neither of them wrote, catches a bug they share.  A `gpu` test
asserts the device pixels equal Pillow's byte for byte and, where the host sees it, that the path was taken."""
import numpy as np
import pytest

import vp8l_model as M


def cached_palette(seed=0):
    """A 4-colour palette coded with a 3-bit cache whose first token is cache index 0 (the empty cache's
    0x00000000); the main image uses every index."""
    rng = np.random.default_rng(seed)
    a, b = (int(v) | 0x01010101 for v in rng.integers(0, 2 ** 32, 2, dtype=np.uint64))
    pal = [("cache", 0), ("lit", a), ("lit", b), ("cache", M.cache_index(a, 3))]
    main = [("lit", 0xFF000000 | 0x1B << 8)] + [("lit", int(g) << 8) for g in rng.integers(0, 256, 2 * 8 - 1)]
    return M.compose(8, 8, main, transforms=[("palette", 4, pal, 3)])


def many_groups(ngroups=12, seed=1):
    """A 64 x 16 image with 4-pixel tiles cycling through `ngroups` prefix-code groups."""
    rng = np.random.default_rng(seed)
    ent = [k % ngroups for k in range(16 * 4)]
    main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, 64 * 16, dtype=np.uint64)]
    return M.compose(64, 16, main, meta=(2, ent, 16))


def zero_bit_tokens(side=300):
    """A solid image of literals whose five codes each have one symbol: every token takes 0 bits, so the lone chunk
    holds more tokens than its first capacity."""
    return M.compose(side, side, [("lit", 0xFF336699)] * (side * side))


def full_cache(seed=2):
    """An 11-bit cache (2048 slots): distinct literals, then a cache token for every slot they filled."""
    rng = np.random.default_rng(seed)
    vals = [int(v) for v in rng.integers(0, 2 ** 32, 3000, dtype=np.uint64)]
    slots = {}
    for v in vals:
        slots[M.cache_index(v, 11)] = v
    toks = [("lit", v) for v in vals] + [("cache", s) for s in sorted(slots)]
    toks += [("lit", 0)] * (-len(toks) % 64)
    return M.compose(64, len(toks) // 64, toks, cache_bits=11)


def sentinel_modes(seed=3):
    """A predictor transform on 4-pixel tiles whose modes are 14, 15, 13 and 0."""
    rng = np.random.default_rng(seed)
    tiles = [("lit", 0xFF000000 | m << 8) for m in (14, 15, 13, 0)]
    main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, 64, dtype=np.uint64)]
    return M.compose(8, 8, main, transforms=[("predictor", 2, tiles, 0)])


def deep_chain(side=512):
    """One literal, then copies of the pixel to the left (distance code 121) over the whole image: pixel i's source
    chain is i long."""
    n = side * side
    toks = [("lit", 0xFF0A0B0C)]
    left = n - 1
    while left:
        k = min(4096, left)
        toks.append(("copy", k, 121))
        left -= k
    return M.compose(side, side, toks)


CASES = {"cached_palette": cached_palette, "many_groups": many_groups, "zero_bit_tokens": zero_bit_tokens,
         "full_cache": full_cache, "sentinel_modes": sentinel_modes, "deep_chain": deep_chain}


def header(data):
    return M.Header(M.container(data)[0])


def test_cases_reach_their_paths():
    M.COUNTERS.clear()
    h = header(cached_palette())
    assert h.transforms[0][0] == M.COLOUR_INDEXING and M.COUNTERS.get("cache", 0) == 1      # the palette's cache
    assert header(many_groups()).ngroups == 12                                             # > the first 8
    assert header(full_cache()).cache_bits == 11
    h = header(zero_bit_tokens())
    assert all(c.single is not None for c in h.groups[0]) and 8 * len(M.container(zero_bit_tokens())[0]) < 1 << 14
    M.COUNTERS.clear()
    M.decode(sentinel_modes())
    assert M.COUNTERS.get("mode_14", 0) and M.COUNTERS.get("mode_15", 0)
    assert M.COUNTERS.get("cache_hit", 0) == 0


@pytest.mark.parametrize("name", [n for n in CASES if n != "deep_chain"])
def test_model_matches_pillow(name):
    data = CASES[name]()
    assert np.array_equal(M.decode(data, chunk_bits=256), M.pillow_rgba(data))


def test_deep_chain_is_a_chain():
    data = deep_chain()
    h = header(data)
    assert h.cache_bits == 0 and h.ngroups == 1 and not h.transforms
    assert (M.pillow_rgba(data) == [0x0A, 0x0B, 0x0C, 0xFF]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_matches_pillow(name, cuda, gsx_lib):
    from gsx.webp_decode import decode_lossless
    data = CASES[name]()
    st = {}
    got = decode_lossless(data, cuda, stats=st).cpu().numpy()
    assert np.array_equal(got, M.pillow_rgba(data)), name
    if name == "many_groups":
        assert st["groups"] == 12
    if name == "zero_bit_tokens":
        assert st["chunks"] == 1 and st["overflow_reruns"] > 0
    if name == "full_cache":
        assert st["cache_bits"] == 11


@pytest.mark.gpu
def test_sub_image_cache_is_cleared(cuda, gsx_lib):
    """The header workspace is reused from the allocator: a stream whose palette cache held other colours runs
    first, then the stream whose palette reads the empty cache."""
    from gsx.webp_decode import decode_lossless
    for seed in (5, 6, 7):
        decode_lossless(cached_palette(seed), cuda)
        data = cached_palette(0)
        assert np.array_equal(decode_lossless(data, cuda).cpu().numpy(), M.pillow_rgba(data))


# ------------------------------------------------------------------------------------------------ prefix codes
ALPHABETS = (280, 256, 256, 256, 40)


class Lengths:
    """A normal prefix code of given lengths, described by the code-length symbols `seq` ((symbol, extra) pairs; by
    default each length literally), with max_symbol = (nb, value) when given."""

    def __init__(self, lengths, seq=None, max_symbol=None):
        from gsx.webp import BitWriter, code_lengths, reversed_codes
        self.lengths, self.codes = list(lengths), reversed_codes(lengths)
        seq = [(ln, 0) for ln in lengths] if seq is None else seq
        cl_counts = np.bincount([s for s, _ in seq], minlength=19)
        cl_len = code_lengths(cl_counts, 7)
        cl_code = reversed_codes(cl_len)
        lone = sum(1 for x in cl_len if x) == 1
        d = self.desc = BitWriter()
        n = max([i + 1 for i, s in enumerate(M.CL_ORDER) if cl_len[s]] + [4])
        d.put(0, 1)
        d.put(n - 4, 4)
        for s in M.CL_ORDER[:n]:
            d.put(cl_len[s], 3)
        d.put(max_symbol is not None, 1)
        if max_symbol is not None:
            nb, v = max_symbol
            d.put(nb, 3)
            d.put(v, 2 + 2 * nb)
        for s, x in seq:
            d.put(cl_code[s], 0 if lone else cl_len[s])
            if s >= 16:
                d.put(x, (2, 3, 7)[s - 16])


class Simple:
    """A simple prefix code's description: `syms` as written (1 or 2 of them; wide: the first in 8 bits)."""

    def __init__(self, syms, wide=True):
        from gsx.webp import BitWriter
        d = self.desc = BitWriter()
        d.put(1, 1)
        d.put(len(syms) - 1, 1)
        d.put(int(wide), 1)
        d.put(syms[0], 8 if wide else 1)
        if len(syms) == 2:
            d.put(syms[1], 8)
        self.lengths = [0] * 256
        self.codes = [0] * 256
        if len(set(syms)) == 2 and max(syms) < 256:      # canonical: the smaller symbol is code 0
            self.lengths[syms[0]] = self.lengths[syms[1]] = 1
            self.codes[max(syms)] = 1


def stream(width, height, tokens, codes=None, cache_bits=0, cache_field=None):
    """A RIFF WEBP file of one group and no transforms: codes[k] (a Lengths / Simple / Tree) replaces the Tree built
    from the tokens' counts for alphabet k.  cache_field: the raw 4-bit cache-bits value after a set flag."""
    from gsx.webp import BitWriter, Tree
    size = (1 << cache_bits) if cache_bits else 0
    counts = [[0] * a for a in (280 + size, 256, 256, 256, 40)]
    for t in tokens:
        if t[0] == "lit":
            v = t[1]
            for k, c in ((0, (v >> 8) & 255), (1, (v >> 16) & 255), (2, v & 255), (3, v >> 24)):
                counts[k][c] += 1
        elif t[0] == "copy":
            counts[0][256 + M._prefix(t[1])[0]] += 1
            counts[4][M._prefix(t[2])[0]] += 1
        else:
            counts[0][280 + t[1]] += 1
    trees = []
    for k, c in enumerate(counts):
        if codes and k in codes:
            trees.append(codes[k])
            continue
        if not any(c):
            c[0] = 1
        trees.append(Tree(c))
    w = BitWriter()
    w.put(0x2F, 8), w.put(width - 1, 14), w.put(height - 1, 14), w.put(1, 1), w.put(0, 3)
    w.put(0, 1)
    if cache_field is not None:
        w.put(1, 1), w.put(cache_field, 4)
    else:
        w.put(1 if cache_bits else 0, 1)
        if cache_bits:
            w.put(cache_bits, 4)
    w.put(0, 1)
    for t in trees:
        w.extend(t.desc)

    def sym(k, s):
        if sum(1 for ln in trees[k].lengths if ln) > 1:
            w.put(trees[k].codes[s], trees[k].lengths[s])

    for t in tokens:
        if t[0] == "lit":
            v = t[1]
            sym(0, (v >> 8) & 255), sym(1, (v >> 16) & 255), sym(2, v & 255), sym(3, v >> 24)
        elif t[0] == "copy":
            p, nb, x = M._prefix(t[1])
            sym(0, 256 + p)
            w.put(x, nb)
            p, nb, x = M._prefix(t[2])
            sym(4, p)
            w.put(x, nb)
        else:
            sym(0, 280 + t[1])
    return M.riff(w.value.to_bytes((w.size + 7) // 8 + 4, "little"))


def simple_distance(syms):
    """2 x 1 pixels, all five codes simple: green (0x10, 0x20) picks each pixel's green, the distance code is `syms`.
    libwebp gives an 8-bit symbol past the 40-symbol alphabet no length, so only a code with none in the alphabet
    is refused."""
    return stream(2, 1, [("lit", 0xFF301040), ("lit", 0xFF302040)],
                  {0: Simple([0x10, 0x20]), 4: Simple(list(syms))})


def simple_forms():
    """Simple codes in both forms: green 1-bit (symbol 1), red 8-bit with two equal symbols, blue two symbols."""
    return stream(3, 1, [("lit", 0xFF070105), ("lit", 0xFF070109), ("lit", 0xFF070105)],
                  {0: Simple([1], wide=False), 1: Simple([7, 7]), 2: Simple([5, 9])})


SIMPLE_DISTANCE = {"5": (5,), "5_5": (5, 5), "5_200": (5, 200), "200_5": (200, 5), "39_40": (39, 40)}
SIMPLE_REFUSED = {"200": (200,)}


def long_code(k, seed=20):
    """Alphabet k's code has 16 symbols at lengths 1..14, 15, 15 (nine of them past the 8-bit table), every one used;
    the other codes are built from the counts.  For the distance code every copy is one pixel long."""
    rng = np.random.default_rng(seed + k)
    lens = [0] * ALPHABETS[k]
    syms = sorted(int(s) for s in rng.choice(40 if k == 4 else 256, 16, replace=False)) if k != 4 else list(range(16))
    for s, ln in zip(syms, list(range(1, 15)) + [15, 15]):
        lens[s] = ln
    shift = (8, 16, 0, 24)[k] if k < 4 else None
    toks = []
    for i in range(330):
        v = int(rng.integers(0, 4)) * 0x11111111 & ~(0xFF << shift) if shift is not None else 0xFF000000
        toks.append(("lit", v | (syms[i % 16] << shift if shift is not None else int(rng.integers(0, 4)) << 8)))
    if k == 4:
        for s in syms:                             # the smallest distance code of each prefix symbol
            toks.append(("copy", 1, s + 1 if s < 4 else ((2 + (s & 1)) << ((s - 2) >> 1)) + 1))
        toks += [("lit", 0xFF000000)] * (-len(toks) % 33)
    return stream(33, len(toks) // 33, toks, {k: Lengths(lens)})


def one_used(lens_of):
    """A red code of the given {symbol: length}: libwebp makes exactly one used symbol, of any length 1..15, a 0-bit
    code; one symbol at length 3 beside four at length 15 is an incomplete code, which it refuses."""
    lens = [0] * 256
    for s, ln in lens_of.items():
        lens[s] = ln
    return stream(4, 2, [("lit", 0xFF000000 | 0x20 << 8 | i) for i in range(8)], {1: Lengths(lens)})


ONE_USED = {"one_len_1": {7: 1}, "one_len_14": {7: 14}, "one_len_15": {7: 15}}
ONE_USED_REFUSED = {"len_3_and_15s": {7: 3, 100: 15, 101: 15, 102: 15, 103: 15}, "two_len_15": {7: 15, 9: 15}}


def lone_cl_code():
    """Red uses all 256 values once: every length is 8, so the code-length code has one symbol (read with 0 bits)."""
    toks = [("lit", 0xFF000000 | v << 16) for v in np.random.default_rng(21).permutation(256).tolist()]
    return stream(16, 16, toks)


def max_symbol(nb):
    """nb 0: red reads max_symbol 4 of its lengths (2, 2, 2, 2); nb 7: blue reads 102 (a complete code over 0..101)."""
    from gsx.webp import code_lengths
    if nb == 0:
        lens = [2, 2, 2, 2] + [0] * 252
        code = Lengths(lens, seq=[(2, 0)] * 4, max_symbol=(0, 2))
        toks = [("lit", 0xFF000000 | (i % 4) << 16) for i in range(12)]
        return stream(4, 3, toks, {1: code})
    lens = code_lengths([1] * 102, 15) + [0] * 154
    code = Lengths(lens, seq=[(ln, 0) for ln in lens[:102]], max_symbol=(7, 100))
    toks = [("lit", 0xFF000000 | i % 102) for i in range(204)]
    return stream(12, 17, toks, {2: code})


def repeats():
    """Red: code-length 16 repeats before any length (each repeats 8) for all 256 lengths, the code-length code one
    symbol; green: 256 literal lengths of 8, then an 18 ending exactly at 280; distance: lengths 1, 1, then an 18 and
    a 17 ending exactly at 40 (read, not used)."""
    red = Lengths([8] * 256, seq=[(16, 3)] * 42 + [(16, 1)])
    green = Lengths([8] * 256 + [0] * 24, seq=[(8, 0)] * 256 + [(18, 13)])
    dist = Lengths([1, 1] + [0] * 38, seq=[(1, 0), (1, 0), (18, 19), (17, 5)])
    rng = np.random.default_rng(22)
    toks = [("lit", 0xFF000000 | int(v) << 16 | int(g) << 8) for v, g in zip(rng.integers(0, 256, 64),
                                                                              rng.integers(0, 256, 64))]
    return stream(8, len(toks) // 8, toks, {0: green, 1: red, 4: dist})


# ------------------------------------------------------------------------------------------------ colour cache
def cache_bits_case(bits, seed=30):
    """A colour cache of `bits`: literals, then cache tokens naming the slots they filled, then more literals."""
    rng = np.random.default_rng(seed + bits)
    vals = [int(v) for v in rng.integers(0, 2 ** 32, 40, dtype=np.uint64)]
    slots = {M.cache_index(v, bits): v for v in vals}
    toks = [("lit", v) for v in vals] + [("cache", s) for s in list(slots)[:30]] + [("lit", v) for v in vals[:10]]
    toks += [("lit", 0)] * (-len(toks) % 9)
    return M.compose(9, len(toks) // 9, toks, cache_bits=bits)


def cache_field(v):
    """The cache flag set with a bits field of v (0 or 12..15 are refused)."""
    return stream(2, 2, [("lit", 1)] * 4, cache_field=v)


# ------------------------------------------------------------------------------------------------ transforms
def tiles_case(kind, bits, seed=40):
    """A predictor or cross-colour transform of `bits` tiles on a width that is not a multiple of the tile."""
    rng = np.random.default_rng(seed + bits + (kind == "cross") * 100)
    width, height = (1 << bits) + 3, 5
    tw, th = M.div(width, bits), M.div(height, bits)
    if kind == "predictor":
        tiles = [("lit", 0xFF000000 | int(m) << 8) for m in rng.integers(0, 14, tw * th)]
    else:
        tiles = [("lit", 0xFF000000 | int(v)) for v in rng.integers(0, 1 << 24, tw * th)]
    main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, width * height, dtype=np.uint64)]
    return M.compose(width, height, main, transforms=[(kind, bits, tiles, 0)])


def palette_case(n, width=13, height=3, past=False, then=(), seed=50):
    """A palette of n colours, every index used (past: one index beyond the palette, which reads colour 0); `then`
    adds transforms after it in reading order, on the packed width."""
    rng = np.random.default_rng(seed + n)
    cols = [int(v) for v in rng.integers(0, 2 ** 32, n, dtype=np.uint64)]
    deltas = [cols[0]] + [int((np.frombuffer(cols[i].to_bytes(4, "little"), np.uint8)
                               - np.frombuffer(cols[i - 1].to_bytes(4, "little"), np.uint8)).view("<u4")[0])
                          for i in range(1, n)]
    bits = 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3
    per, xs = 1 << bits, M.div(width, bits)
    idx = rng.integers(0, n, (height, width))
    idx.flat[: min(n, idx.size)] = np.arange(min(n, idx.size))
    if past:
        idx[0, 1] = (1 << (8 >> bits)) - 1
    main = []
    for y in range(height):
        for px in range(xs):
            g = 0
            for k in range(per):
                x = px * per + k
                if x < width:
                    g |= int(idx[y, x]) << (k * (8 >> bits))
            main.append(("lit", 0xFF000000 | g << 8))
    tr = [("palette", n, [("lit", d) for d in deltas], 0)]
    for t in then:
        if t == "green":
            tr.append(("green",))
        else:
            tiles = [("lit", 0xFF000000 | int(v) << 8 if t == "predictor" else int(v))
                     for v in rng.integers(0, 14 if t == "predictor" else 1 << 24, M.div(xs, 2) * M.div(height, 2))]
            tr.append((t, 2, tiles, 0))
    if then:     # the residuals the later transforms undo: random, on the packed width
        main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, xs * height, dtype=np.uint64)]
    return M.compose(width, height, main, transforms=tr)


PALETTES = (1, 2, 3, 4, 5, 16, 17, 256)


def repeated_transform():
    return M.compose(4, 4, [("lit", 1)] * 16, transforms=[("green",), ("green",)])


def wavefront(height, width, seed=60):
    """A predictor over height x width; more than 4096 pixels are 4093 literals and then copies 4093 back, so the
    stream stays small while every row differs."""
    rng = np.random.default_rng(seed + height * 64 + width)
    bits = 2 if height * width < 50_000 else 5
    tw, th = M.div(width, bits), M.div(height, bits)
    tiles = [("lit", 0xFF000000 | int(m) << 8) for m in rng.integers(0, 14, tw * th)]
    n = width * height
    main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, min(n, 4093), dtype=np.uint64)]
    left = n - len(main)
    while left:
        k = min(4096, left)
        main.append(("copy", k, 4093 + 120))
        left -= k
    return M.compose(width, height, main, transforms=[("predictor", bits, tiles, 0)])


WAVE_HEIGHTS, WAVE_WIDTHS = (1, 31, 32, 33, 65, 16384), (1, 2, 3, 61, 62, 63)


def right_column_modes(seed=61):
    """9 x 56 pixels, 4-pixel tiles: the rightmost tile column runs every mode 0..13 top to bottom, so every mode
    meets the rightmost pixel's TR (the leftmost pixel of the row)."""
    rng = np.random.default_rng(seed)
    tiles = []
    for ty in range(14):
        tiles += [("lit", 0xFF000000 | int(m) << 8) for m in rng.integers(0, 14, 2)] + [("lit", 0xFF000000 | ty << 8)]
    main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, 9 * 56, dtype=np.uint64)]
    return M.compose(9, 56, main, transforms=[("predictor", 2, tiles, 0)])


# ------------------------------------------------------------------------------------------------ entropy image
def meta_case(bits, groups=(0, 1, 2), seed=70):
    """Meta prefix codes of `bits` tiles on a ragged width, the tiles' groups drawn from `groups` (any not drawn are
    still read, as simple codes)."""
    rng = np.random.default_rng(seed + bits + len(groups))
    width, height = (1 << bits) + 5, 3
    tx, ty = M.div(width, bits), M.div(height, bits)
    ent = [int(g) for g in rng.choice(groups, tx * ty)]
    k = min(len(groups), len(ent))
    ent[:k] = sorted(groups, reverse=True)[:k]         # the largest first, then as many others as fit
    main = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, width * height, dtype=np.uint64)]
    return M.compose(width, height, main, meta=(bits, ent, tx))


# ------------------------------------------------------------------------------------------------ chain
def plane_codes(width, seed=80):
    """All 120 plane distance codes (copies of one pixel) at a narrow width, where some clamp to distance 1."""
    rng = np.random.default_rng(seed + width)
    toks = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, 90, dtype=np.uint64)]
    toks += [("copy", 1, c) for c in range(1, 121)]
    toks += [("lit", 0xFF000000)] * (-len(toks) % width)
    return M.compose(width, len(toks) // width, toks)


def cached_copies(seed=90):
    """Literals, cache tokens and copies mixed, with a 4-bit cache: at 32-bit chunks every kind crosses chunk ends."""
    rng = np.random.default_rng(seed)
    vals = [int(v) for v in rng.integers(0, 2 ** 32, 12, dtype=np.uint64)]
    toks, recent = [], []
    for i in range(600):
        r = rng.integers(0, 3)
        if r == 0 or not recent:
            v = vals[int(rng.integers(0, 12))]
            toks.append(("lit", v))
            recent.append(v)
        elif r == 1:
            toks.append(("cache", M.cache_index(recent[-1], 4)))
            recent.append(recent[-1])
        else:
            k = int(rng.integers(2, 20))
            toks.append(("copy", k, 1 + 120))
            recent += [recent[-1]] * k
    toks += [("lit", 0)] * (-len(recent) % 16)
    return M.compose(16, -(-len(recent) // 16), toks, cache_bits=4)


NEW = {
    **{f"simple_dist_{k}": (lambda v=v: simple_distance(v)) for k, v in SIMPLE_DISTANCE.items()},
    "simple_forms": simple_forms,
    **{f"long_code_{k}": (lambda k=k: long_code(k)) for k in range(5)},
    **{k: (lambda v=v: one_used(v)) for k, v in ONE_USED.items()},
    "lone_cl_code": lone_cl_code, "max_symbol_0": lambda: max_symbol(0), "max_symbol_7": lambda: max_symbol(7),
    "repeats": repeats,
    **{f"cache_bits_{b}": (lambda b=b: cache_bits_case(b)) for b in range(1, 12)},
    **{f"{k}_bits_{b}": (lambda k=k, b=b: tiles_case(k, b)) for k in ("predictor", "cross") for b in range(2, 10)},
    **{f"palette_{n}": (lambda n=n: palette_case(n)) for n in PALETTES},
    "palette_past": lambda: palette_case(5, past=True),
    "palette_then_all": lambda: palette_case(4, width=23, height=9, then=("predictor", "cross", "green")),
    "right_column_modes": right_column_modes,
    **{f"meta_bits_{b}": (lambda b=b: meta_case(b)) for b in range(2, 10)},
    "meta_group_300": lambda: meta_case(2, groups=(0, 3, 300)), "meta_gaps": lambda: meta_case(2, groups=(0, 4, 9)),
    **{f"plane_codes_w{w}": (lambda w=w: plane_codes(w)) for w in range(1, 10)},
    "cached_copies": cached_copies,
}
REFUSED = {
    **{f"simple_dist_{k}": (lambda v=v: simple_distance(v)) for k, v in SIMPLE_REFUSED.items()},
    **{k: (lambda v=v: one_used(v)) for k, v in ONE_USED_REFUSED.items()},
    **{f"cache_field_{v}": (lambda v=v: cache_field(v)) for v in (0, 12, 13, 14, 15)},
    "repeated_transform": repeated_transform,
}
WAVES = {f"wave_h{h}_w{w}": (lambda h=h, w=w: wavefront(h, w)) for h in WAVE_HEIGHTS for w in WAVE_WIDTHS}


@pytest.mark.parametrize("name", sorted(NEW))
def test_new_model_matches_pillow(name):
    data = NEW[name]()
    assert np.array_equal(M.decode(data, chunk_bits=64), M.pillow_rgba(data)), name


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_by_model_and_pillow(name):
    data = REFUSED[name]()
    with pytest.raises(ValueError):
        M.decode(data, chunk_bits=64)
    with pytest.raises(Exception):
        M.pillow_rgba(data)


def counters(*names):
    M.COUNTERS.clear()
    for n in names:
        M.decode(NEW[n](), chunk_bits=64)
    return dict(M.COUNTERS)


def test_new_cases_reach_their_paths():
    c = counters(*[f"simple_dist_{k}" for k in SIMPLE_DISTANCE])
    assert c.get("simple_code_past_alphabet", 0) == 3 and c.get("simple_code_8bit", 0)
    c = counters("simple_forms")
    assert c.get("simple_code_1bit", 0) and c.get("single_len_1", 0)
    for k in range(5):
        code = header(NEW[f"long_code_{k}"]()).groups[0][k]
        assert code.single is None and code.max == 15
    assert counters("one_len_15").get("single_len_15", 0)
    assert header(NEW["lone_cl_code"]()).groups[0][1].max == 8
    c = counters("repeats")
    assert c.get("repeat_before_first", 0)
    assert header(NEW["repeats"]()).groups[0][4].max == 1
    for b in range(1, 12):
        assert header(NEW[f"cache_bits_{b}"]()).cache_bits == b
        assert counters(f"cache_bits_{b}").get("cache_hit", 0) > 0
    for kind, t in (("predictor", M.PREDICTOR), ("cross", M.CROSS_COLOUR)):
        for b in range(2, 10):
            h = header(NEW[f"{kind}_bits_{b}"]())
            assert h.transforms[0][0] == t and h.transforms[0][2] == b and h.width % (1 << b)
    for n in PALETTES:
        h = header(NEW[f"palette_{n}"]())
        assert h.transforms[0][0] == M.COLOUR_INDEXING and h.xsize == M.div(h.width, h.transforms[0][2])
    h = header(NEW["palette_then_all"]())
    assert [t[0] for t in h.transforms] == [M.COLOUR_INDEXING, M.PREDICTOR, M.CROSS_COLOUR, M.SUBTRACT_GREEN]
    assert all(t[1] == h.xsize < h.width for t in h.transforms[1:])
    c = counters("right_column_modes")
    assert all(c.get(f"mode_{m}", 0) for m in range(14))
    for b in range(2, 10):
        h = header(NEW[f"meta_bits_{b}"]())
        assert h.meta_bits == b and h.ngroups == 3 and h.width % (1 << b)
    assert header(NEW["meta_group_300"]()).ngroups == 301
    h = header(NEW["meta_gaps"]())
    assert h.ngroups == 10 and set(np.unique(h.entropy)) == {0, 4, 9}
    for w in range(1, 10):
        clamps = sum(1 for dx, dy in M.PLANE if dx + dy * w < 1)
        assert (clamps > 0) == (w <= 7), w
    h = header(NEW["cached_copies"]())
    assert h.cache_bits == 4 and 8 * len(M.container(NEW["cached_copies"]())[0]) > 64 * 32


def test_cached_copies_walk():
    data = NEW["cached_copies"]()
    st = {}
    assert np.array_equal(M.decode(data, chunk_bits=32, max_rounds=0, stats=st), M.pillow_rgba(data))
    assert st["serial_fallbacks"] == 1


@pytest.mark.parametrize("name", [n for n in sorted(WAVES) if "16384" not in n])
def test_wavefront_model_matches_pillow(name):
    data = WAVES[name]()
    assert np.array_equal(M.decode(data, chunk_bits=1 << 12), M.pillow_rgba(data)), name


def test_wavefront_cases():
    for name, build in WAVES.items():
        h = header(build())
        assert h.transforms[0][0] == M.PREDICTOR and (h.height, h.width) == tuple(
            int(v) for v in name[6:].split("_w")), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(NEW))
def test_new_device_matches_pillow(name, cuda, gsx_lib):
    from gsx.webp_decode import decode_lossless
    data = NEW[name]()
    want = M.pillow_rgba(data)
    assert np.array_equal(decode_lossless(data, cuda).cpu().numpy(), want), name
    if name == "cached_copies":
        for cb, rounds in ((32, 0), (32, None), (64, 2)):
            st = {}
            got = decode_lossless(data, cuda, chunk_bits=cb, max_rounds=rounds, stats=st).cpu().numpy()
            assert np.array_equal(got, want), (cb, rounds)
            assert st["chunks"] > 8


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_on_device(name, cuda, gsx_lib):
    from gsx.webp_decode import decode_lossless
    with pytest.raises(ValueError):
        decode_lossless(REFUSED[name](), cuda)


@pytest.mark.gpu
@pytest.mark.parametrize("height", WAVE_HEIGHTS)
def test_wavefront_device_matches_pillow(height, cuda, gsx_lib):
    from gsx.webp_decode import decode_lossless
    for w in WAVE_WIDTHS:
        data = WAVES[f"wave_h{height}_w{w}"]()
        assert np.array_equal(decode_lossless(data, cuda).cpu().numpy(), M.pillow_rgba(data)), (height, w)

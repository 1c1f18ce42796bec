"""The VP8L decoder's paths (csrc/gsx_vp8l.cu, gsx/webp_decode.py), one hand-built stream each: a colour-cached
sub-image whose first token reads the empty cache, more prefix-code groups than the first header workspace holds,
a job's token capacity overflowing, the 2048-entry colour cache, the predictor's modes 14 and 15, and copy chains as
deep as the image under k_vp8l_jump.

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

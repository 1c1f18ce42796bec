"""The VP8L encoder kernels (csrc/gsx_webp.cu), path by path: k_webp_clean's alpha rules and grid-stride pass, every
predictor mode of k_webp_predict winning a tile in both candidates, its ties and arithmetic edges, the image sides
around a tile, the copy tokens of k_webp_tokens over every length prefix code and the 4096-pixel split, and the scan
chunks of k_webp_bits / k_webp_bases / k_webp_emit past 2^26 pixels.

Each case has a seeded builder.  An unmarked CPU test proves through webp_oracle (`info=`, `predict`, `tokens`) or a
NumPy restatement of the kernel's cost and dispatch that the case reaches the branch it is named after, and decodes
every oracle file it builds with Pillow: the oracle restates the kernel, so only a decoder neither of them wrote
catches a bug they share.  A `gpu` test asserts the device file equals the oracle's byte for byte, and the five
histograms and both candidates' tile modes equal the oracle's; for images the oracle cannot afford, the image is
built on the device and the file must decode with Pillow to it."""
import io

import numpy as np
import pytest

import webp_oracle as wo

TILE = 16
SCAN_CHUNK = 1 << 26          # kScanChunk: pixels per offset scan of k_webp_bits
CLEAN_GRID_PER_SM = 8         # grid_for(): at most 8 CTAs of 256 threads per SM
H100_SMS = (114, 132)         # H100 PCIe, H100 SXM


def decode(data: bytes) -> np.ndarray:
    from PIL import Image
    Image.MAX_IMAGE_PIXELS = None
    im = Image.open(io.BytesIO(data))
    assert im.format == "WEBP"
    return np.asarray(im.convert("RGBA"))


def expected(img: np.ndarray) -> np.ndarray:
    out = img.copy()
    out[out[..., 3] == 0, :3] = 0
    return out


def oracle_file(img, info=None) -> bytes:
    data = wo.encode(img, info=info)
    assert np.array_equal(decode(data), expected(img))
    return data


def rgba_of(argb: np.ndarray, h: int, w: int) -> np.ndarray:
    a = argb.astype(np.uint32)
    return np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255, a >> 24], -1).astype(np.uint8).reshape(h, w, 4)


def device_encode(img, cuda, info=None):
    import torch
    from gsx import webp
    h, w = img.shape[:2]
    return webp.encode_lossless(torch.from_numpy(np.ascontiguousarray(img).reshape(-1, 4)).to(cuda), w, h, info=info)


def device_analyze(img, cuda, gsx_lib):
    """(hist uint32 [5 * 1088 + 1], tile modes uint8 [2, tiles_y, tiles_x]) of gsx_webp_analyze."""
    import torch
    from gsx import webp
    from gsx._abi import _ptr, _stream, check
    h, w = img.shape[:2]
    t = torch.from_numpy(np.ascontiguousarray(img).reshape(-1, 4)).to(cuda)
    ty, tx = -(-h // TILE), -(-w // TILE)
    ws = torch.empty(gsx_lib.gsx_webp_workspace_bytes(w, h), dtype=torch.uint8, device=cuda)
    hist = torch.empty(5 * webp.TREE_SYMS + 1, dtype=torch.int32, device=cuda)
    modes = torch.empty(2 * tx * ty, dtype=torch.uint8, device=cuda)
    check(gsx_lib.gsx_webp_analyze(_ptr(t), w, h, _ptr(ws), ws.numel(), _ptr(hist), _ptr(modes), _stream()),
          "gsx_webp_analyze")
    return hist.cpu().numpy().view(np.uint32), modes.cpu().numpy().reshape(2, ty, tx)


def oracle_analyze(img):
    h, w = img.shape[:2]
    c = wo.candidates(img, w, h)
    images = [c[0][1], c[1][1], c[2][1], c[1][2], c[2][2]]
    hist = np.concatenate([np.concatenate(i.hist) for i in images] + [[int((img[..., 3] != 255).any())]])
    return hist.astype(np.uint32), np.stack([c[1][3], c[2][3]])


def check_device(img, cuda, gsx_lib):
    want_info, got_info = {}, {}
    want = wo.encode(img, info=want_info)
    got = device_encode(img, cuda, got_info)
    assert got_info["candidate"] == want_info["candidate"] and got_info["bits"] == want_info["bits"]
    hist, modes = device_analyze(img, cuda, gsx_lib)
    want_hist, want_modes = oracle_analyze(img)
    assert np.array_equal(modes, want_modes), "tile modes differ"
    assert np.array_equal(hist, want_hist), f"histograms differ at {np.flatnonzero(hist != want_hist)[:8]}"
    if got != want:
        diff = next(i for i, (a, b) in enumerate(zip(got, want)) if a != b) if len(got) == len(want) else None
        raise AssertionError(f"device file ({len(got)} B) differs from the oracle's ({len(want)} B) at byte {diff}")
    assert np.array_equal(decode(got), expected(img))


def tile_costs(src: np.ndarray, w: int, h: int) -> np.ndarray:
    """int64 [tiles, 14]: k_webp_predict's cost of every mode per tile (sum of |residual as int8| over the four
    channels of the tile's inner pixels; the edge pixels cost the same under every mode)."""
    c = wo.channels(src)
    n = w * h
    x, y = np.arange(n) % w, np.arange(n) // w
    tile = (y // TILE) * -(-w // TILE) + x // TILE
    inner = (x > 0) & (y > 0)
    out = []
    for pr in wo.mode_predictions(c, w):
        r = ((c - pr) & 0xFF).astype(np.uint8).view(np.int8).astype(np.int64)
        out.append(np.bincount(tile[inner], weights=np.abs(r[inner]).sum(1), minlength=-(-w // TILE) * -(-h // TILE)))
    return np.stack(out, 1).astype(np.int64)


def neighbours(src: np.ndarray, w: int):
    """int32 [n, 4] each: L, T, TR (the rightmost column's TR is the row's first pixel), TL of every pixel."""
    c = wo.channels(src)
    ext = np.concatenate([np.zeros((w + 1, 4), np.int32), c])
    i = np.arange(len(c)) + w + 1
    return ext[i - 1], ext[i - w], ext[np.minimum(i - w + 1, len(c) + w)], ext[i - w - 1]


# ------------------------------------------------------------------------------------------------ k_webp_clean
def alpha0_rgb_case():
    rng = np.random.default_rng(0)
    img = rng.integers(1, 256, (23, 29, 4), dtype=np.uint8)
    img[rng.random((23, 29)) < 0.4, 3] = 0
    return img


def alpha_last_pixel_case():
    """300 000 pixels (more than one pass of the 8 * SMs CTAs of 256 threads), alpha 255 but for the last pixel."""
    rng = np.random.default_rng(1)
    y, x = np.mgrid[:500, :600]
    img = np.stack([(3 * x + y) % 256, (x * y) % 256, rng.integers(0, 4, (500, 600)), np.full((500, 600), 255)], -1)
    img = img.astype(np.uint8)
    img[-1, -1, 3] = 7
    return img


def test_clean_cases_reach_their_paths():
    img = alpha0_rgb_case()
    hidden = (img[..., 3] == 0) & img[..., :3].any(-1)
    assert hidden.sum() > 100 and (wo.to_argb(img)[hidden.reshape(-1)] == 0).all()
    oracle_file(img)
    img = alpha_last_pixel_case()
    n = img.shape[0] * img.shape[1]
    assert np.flatnonzero(img[..., 3].reshape(-1) != 255).tolist() == [n - 1]
    for sms in H100_SMS:
        grid = min(-(-n // 256), CLEAN_GRID_PER_SM * sms)
        assert n - 1 >= grid * 256                      # the last pixel is read on a later pass of the loop
    info = {}
    data = oracle_file(img, info)
    assert (data[20 + 4] >> 4) & 1 == 1                # alpha_is_used: bit 8 + 14 + 14 of the VP8L stream


# ------------------------------------------------------------------------------------------------ k_webp_predict
def _avg(a, b):
    return (a + b) >> 1


def _predict_one(m, L, T, TR, TL):
    """RFC 9649's predictor m of one pixel (int [4] in A, R, G, B order)."""
    if m == 0:
        return np.array([255, 0, 0, 0])
    if m == 11:
        return L if np.abs(T - TL).sum() < np.abs(L - TL).sum() else T
    if m == 12:
        return np.clip(L + T - TL, 0, 255)
    if m == 13:
        a = _avg(L, T)
        d = a - TL
        return np.clip(a + np.where(d < 0, -((-d) >> 1), d >> 1), 0, 255)
    return {1: L, 2: T, 3: TR, 4: TL, 5: _avg(_avg(L, TR), T), 6: _avg(L, TL), 7: _avg(L, T), 8: _avg(TL, T),
            9: _avg(T, TR), 10: _avg(_avg(L, TL), _avg(T, TR))}[m]


# every mode twice; modes that read TR (3, 5, 9, 10) in the rightmost tile column
TILE_MODES = np.array([[0, 1, 2, 3, 4, 5, 9], [6, 7, 8, 11, 12, 13, 10], [13, 12, 11, 10, 7, 5, 3],
                       [1, 4, 6, 8, 2, 0, 9]])
TR_MODES = (3, 5, 9, 10)


def modes_case(green: bool):
    """112 x 64 pixels made in raster order: each inner pixel is its tile's mode's prediction from the pixels made
    before it, plus noise in -3..3 on R, G and B (alpha 255).  With green, that is the subtract-green image, and the
    pixels have green added back to red and blue."""
    th, tw = TILE_MODES.shape
    h, w = TILE * th, TILE * tw
    rng = np.random.default_rng(2)
    c = np.zeros((h, w, 4), np.int64)
    c[..., 0] = 255
    c[0, :, 1:] = rng.integers(0, 256, (w, 3))
    c[:, 0, 1:] = rng.integers(0, 256, (h, 3))
    for y in range(1, h):
        for x in range(1, w):
            tr = c[y - 1, x + 1] if x + 1 < w else c[y, 0]
            p = _predict_one(TILE_MODES[y // TILE, x // TILE], c[y, x - 1], c[y - 1, x], tr, c[y - 1, x - 1])
            e = rng.integers(-3, 4, 4)
            e[0] = 0
            c[y, x] = (p + e) & 0xFF
    if green:
        c[..., 1] = (c[..., 1] + c[..., 2]) & 0xFF
        c[..., 3] = (c[..., 3] + c[..., 2]) & 0xFF
    return np.stack([c[..., 1], c[..., 2], c[..., 3], c[..., 0]], -1).astype(np.uint8)


def ties_case():
    """A constant tile (every mode but 0 that does not read TR costs 0: mode 1 wins the tie) and a tile of vertical
    stripes (modes 2, 11 and 12 cost 0: mode 2 wins)."""
    rng = np.random.default_rng(3)
    img = np.empty((16, 32, 4), np.uint8)
    img[:, :16] = (40, 90, 140, 255)
    img[:, 16:] = rng.integers(0, 256, (1, 16, 4))
    img[..., 3] = 255
    return img


def src_of(img, green):
    p = wo.to_argb(img)
    return wo.subtract_green(p) if green else p


@pytest.mark.parametrize("green", [False, True])
def test_every_mode_wins_a_tile(green):
    img = modes_case(green)
    h, w = img.shape[:2]
    _, modes = wo.predict(src_of(img, green), w, h)
    assert np.array_equal(modes, TILE_MODES)
    assert np.array_equal(tile_costs(src_of(img, green), w, h).argmin(1).reshape(modes.shape), modes)
    info = {}
    oracle_file(img, info)
    assert info["candidate"] == 1 + green


@pytest.mark.parametrize("green", [False, True])
def test_predictor_arithmetic_edges_in_winning_tiles(green):
    img = modes_case(green)
    h, w = img.shape[:2]
    src = src_of(img, green)
    L, T, TR, TL = neighbours(src, w)
    n = w * h
    x, y = np.arange(n) % w, np.arange(n) // w
    mode = TILE_MODES[y // TILE, x // TILE]
    inner = (x > 0) & (y > 0)
    d = _avg(L, T) - TL                                     # clamp_half: odd negative differences truncate to zero
    assert ((d < 0) & (d % 2 == 1))[inner & (mode == 13)].sum() >= 100
    s = L + T - TL                                          # clamp_full clips at both ends
    assert (s < 0)[inner & (mode == 12)].sum() >= 10 and (s > 255)[inner & (mode == 12)].sum() >= 10
    pl, pt = np.abs(T - TL).sum(1), np.abs(L - TL).sum(1)   # select_pred's tie returns T, not L
    assert ((pl == pt) & (L != T).any(1) & inner & (mode == 11)).sum() >= 1
    right = inner & (x == w - 1) & np.isin(mode, TR_MODES)  # the rightmost column's TR wraps to the row's start
    c = wo.channels(src)
    assert right.sum() >= 40 and np.array_equal(TR[right], c[y[right] * w])
    assert (TR[right] != c[(y[right] - 1) * w]).any(1).all() and (TR[right] != T[right]).any(1).all()
    assert set(TILE_MODES[:, -1]) <= set(TR_MODES)


def test_ties_go_to_the_lower_mode():
    img = ties_case()
    cost = tile_costs(wo.to_argb(img), 32, 16)
    tied = [np.flatnonzero(c == c.min()).tolist() for c in cost]
    assert tied == [[1, 2, 4, 6, 7, 8, 11, 12, 13], [2, 11, 12]]
    _, modes = wo.predict(wo.to_argb(img), 32, 16)
    assert modes.reshape(-1).tolist() == [1, 2]
    oracle_file(img)


SIDES = (1, 15, 16, 17)


def sides_case(h, w):
    rng = np.random.default_rng(100 * h + w)
    y, x = np.mgrid[:h, :w]
    img = np.stack([(5 * x + 3 * y) % 256, (7 * y) % 256, rng.integers(0, 3, (h, w)), np.full((h, w), 255)], -1)
    return img.astype(np.uint8)


def test_sides_around_a_tile():
    for h in SIDES:
        for w in SIDES:
            img = sides_case(h, w)
            _, modes = wo.predict(wo.to_argb(img), w, h)
            assert modes.shape == (-(-h // TILE), -(-w // TILE))
            if h == 1 or w == 1:                          # no tile has an inner pixel: every mode costs 0
                assert not tile_costs(wo.to_argb(img), w, h).any() and not modes.any()
            info = {}
            oracle_file(img, info)
            if (h, w) == (16, 16):                        # a one-tile sub-image
                assert info["candidate"] in (1, 2) and modes.size == 1


PREDICT_CASES = {"alpha0_rgb": alpha0_rgb_case, "alpha_last_pixel": alpha_last_pixel_case,
                 "modes_raw": lambda: modes_case(False), "modes_green": lambda: modes_case(True),
                 "ties": ties_case}
PREDICT_CASES.update({f"sides_{h}x{w}": (lambda h=h, w=w: sides_case(h, w)) for h in SIDES for w in SIDES})


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PREDICT_CASES))
def test_clean_and_predict_match_oracle(name, cuda, gsx_lib):
    check_device(PREDICT_CASES[name](), cuda, gsx_lib)


# ------------------------------------------------------------------------------------------------ k_webp_tokens
def runs_image(followers, width, seed, tail=0):
    """Runs of 1 + f equal pixels for each f in `followers`, each after 5 noise pixels, then noise up to a row's
    end less `tail` and a run of `tail` pixels ending on the last pixel."""
    rng = np.random.default_rng(seed)
    parts, starts = [], []
    at = 0
    for k, f in enumerate(followers):
        parts.append(rng.integers(0, 1 << 24, 5) | 0xFF000000)
        starts.append(at + 5)
        parts.append(np.full(1 + f, 0xFF000000 | (0x10101 * (k % 200 + 20)), np.int64))
        at += 6 + f
    pad = -(at + tail) % width
    parts.append(rng.integers(0, 1 << 24, pad) | 0xFF000000)
    parts.append(np.full(tail, 0xFF0A0B0C, np.int64))
    p = np.concatenate(parts).astype(np.uint32)
    return rgba_of(p, len(p) // width, width), starts


FOLLOWERS = [4096 * k + j for k in (1, 2) for j in range(4)]


def followers_case():
    return runs_image(FOLLOWERS, 256, 4096, tail=700)


def length_codes_case():
    lengths = []
    for c in range(2, 24):
        if c < 4:
            lengths.append(c + 1)
        else:
            nb = (c - 2) >> 1
            off = (2 + (c & 1)) << nb
            lengths += [off + 1, off + (1 << nb)]
    return runs_image(lengths, 128, 23)


def test_followers_4096k_plus_0_to_3():
    img, starts = followers_case()
    h, w = img.shape[:2]
    tok = wo.tokens(wo.to_argb(img))
    for s, f in zip(starts, FOLLOWERS):
        k, j = divmod(f, 4096)
        assert tok[s] == 1 and tok[s - 1] == 1
        assert tok[s + 1 + 4096 * np.arange(k)].tolist() == [4096] * k
        tail = tok[s + 1 + 4096 * k:s + 1 + f].tolist()
        assert tail == ([3, 0, 0] if j == 3 else [1] * j)
        assert tok[s + 1 + f] == 1                      # the next pixel is noise
    assert tok[-700:].tolist() == [1, 699] + [0] * 698  # a run over rows, ending on the last pixel
    assert (h * w - 700) // w < (h * w - 1) // w
    info = {}
    oracle_file(img, info)
    assert info["candidate"] == 0


def test_every_length_prefix_code():
    img, _ = length_codes_case()
    tok = wo.tokens(wo.to_argb(img))
    code, nbits, _ = wo.length_prefix(tok[tok >= 3])
    assert set(code.tolist()) == set(range(2, 24))
    assert 10 in nbits[tok[tok >= 3] == 4096]
    info = {}
    oracle_file(img, info)
    assert info["candidate"] == 0


TOKEN_CASES = {"followers": lambda: followers_case()[0], "length_codes": lambda: length_codes_case()[0]}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TOKEN_CASES))
def test_tokens_match_oracle(name, cuda, gsx_lib):
    check_device(TOKEN_CASES[name](), cuda, gsx_lib)


# ------------------------------------------------------------------------------------------------ scan chunks
P_LAST = SCAN_CHUNK - 1       # the last pixel of scan chunk 0
RUN_ARGB = 0xFF123456
SCAN_RUNS = {"literal": None, "copy_head": (P_LAST - 1, P_LAST + 101), "inside_copy": (P_LAST - 50, P_LAST + 51)}


def noise_argb(i):
    """Opaque pixels from a hash of the pixel index (int64 NumPy array or torch tensor): neighbours differ."""
    h = (i * 2654435761) & 0xFFFFFFFF
    h = ((h ^ (h >> 15)) * 0x2C1B3C6D) & 0xFFFFFFFF
    return (h >> 8) | 0xFF000000


def scan_window(kind, lo, hi):
    p = noise_argb(np.arange(lo, hi, dtype=np.int64))
    if SCAN_RUNS[kind]:
        a, b = SCAN_RUNS[kind]
        p[a - lo:b - lo] = RUN_ARGB
    return p.astype(np.uint32)


@pytest.mark.parametrize("kind", sorted(SCAN_RUNS))
def test_scan_chunk_edge_tokens(kind):
    lo, hi = P_LAST - 4096, P_LAST + 4096
    p = scan_window(kind, lo, hi)
    assert p[0] != noise_argb(np.int64(lo - 1)) and p[-1] != noise_argb(np.int64(hi))   # the window's runs are whole
    tok = wo.tokens(p)
    want = {"literal": 1, "copy_head": 101, "inside_copy": 0}[kind]
    assert tok[P_LAST - lo] == want and tok[P_LAST - lo + 1] in (0, 1)
    assert 8192 * 8193 == SCAN_CHUNK + 8192 and 16384 * 16384 == 4 * SCAN_CHUNK


def device_noise_image(w, h, kind, cuda):
    import torch
    n = w * h
    out = torch.empty((n, 4), dtype=torch.uint8, device=cuda)
    step = 1 << 24
    for lo in range(0, n, step):
        p = noise_argb(torch.arange(lo, min(n, lo + step), dtype=torch.int64, device=cuda))
        out[lo:lo + step] = torch.stack([(p >> s) & 255 for s in (16, 8, 0, 24)], -1).to(torch.uint8)
    if kind and SCAN_RUNS[kind]:
        a, b = SCAN_RUNS[kind]
        out[a:b] = torch.tensor([0x12, 0x34, 0x56, 0xFF], dtype=torch.uint8, device=cuda)
    return out


def check_decodes(w, h, kind, cuda):
    import torch
    from gsx import webp
    t = device_noise_image(w, h, kind, cuda)
    info = {}
    data = webp.encode_lossless(t, w, h, info=info)
    assert info["candidate"] == 0                      # the tokens are those of the pixels themselves
    img = t.cpu().numpy().reshape(h, w, 4)
    del t
    torch.cuda.empty_cache()
    assert np.array_equal(decode(data), img)          # opaque: the same_pixels rule is plain equality


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(SCAN_RUNS))
def test_two_scan_chunks_decode(kind, cuda, gsx_lib):
    check_decodes(8192, 8193, kind, cuda)


@pytest.mark.gpu
def test_four_scan_chunks_decode(cuda, gsx_lib):
    check_decodes(16384, 16384, None, cuda)

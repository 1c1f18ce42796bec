"""NumPy restatement of gsx's lossless WebP (VP8L) encoder, written from RFC 9649.

Every decision the device encoder makes is restated here, so the two must agree byte for byte:

  * transparent pixels: RGB := 0 where alpha == 0;
  * three candidates: (0) no transform, (1) the predictor transform, (2) subtract-green then the predictor, with
    16x16 tiles (size_bits 4) and, per tile, the mode 0..13 with the smallest sum of |residual as int8| over the four
    channels of every pixel of the tile (lowest mode on a tie); the RFC's edge rules and the rightmost column's TR;
  * run copies: a backward reference with distance code 2 (the left pixel) over the coded pixels, greedy: after the
    literal that starts a run of equal pixels, its r followers become copies of min(4096, left) pixels while at least
    3 are left; fewer than 3 stay literals.  Runs cross rows;
  * one Huffman group, no colour cache, no meta prefix image.  Codes: `huffman_lengths` (limit 15, code-length code 7);
    a tree with at most two used symbols, all below 256, is a simple code; otherwise a normal code with no repeat
    codes (16/17/18) and max_symbol = the whole alphabet;
  * the candidate with the fewest total bits wins (earliest on a tie);
  * the predictor sub-image (mode in green, alpha 255) is coded like any entropy-coded image: its own runs and codes.
"""
from __future__ import annotations

import heapq

import numpy as np

TILE_BITS = 4
TILE = 1 << TILE_BITS
MAX_COPY = 4096
MIN_COPY = 3
MAX_SIDE = 16384
N_LEN = 24
ALPHABETS = (256 + N_LEN, 256, 256, 256, 40)        # green + lengths, red, blue, alpha, distance
CL_ORDER = (17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
LEFT_DIST_SYMBOL = 1                                  # plane code 2 = (xi 1, yi 0) -> prefix symbol 1, no extra bits


# ---------------------------------------------------------------------------------------------------- pixels


def to_argb(rgba: np.ndarray) -> np.ndarray:
    """uint8 [..., 4] RGBA -> uint32 ARGB, with RGB cleared where alpha is 0."""
    a = rgba.reshape(-1, 4).astype(np.uint32)
    argb = (a[:, 3] << 24) | (a[:, 0] << 16) | (a[:, 1] << 8) | a[:, 2]
    return np.where(a[:, 3] == 0, np.uint32(0), argb).astype(np.uint32)


def channels(p: np.ndarray) -> np.ndarray:
    """uint32 ARGB [n] -> int32 [n, 4] in the order A, R, G, B."""
    return np.stack([(p >> s) & 0xFF for s in (24, 16, 8, 0)], axis=-1).astype(np.int32)


def pack(c: np.ndarray) -> np.ndarray:
    c = c.astype(np.uint32) & 0xFF
    return (c[..., 0] << 24) | (c[..., 1] << 16) | (c[..., 2] << 8) | c[..., 3]


def subtract_green(p: np.ndarray) -> np.ndarray:
    c = channels(p)
    c[:, 1] = (c[:, 1] - c[:, 2]) & 0xFF
    c[:, 3] = (c[:, 3] - c[:, 2]) & 0xFF
    return pack(c)


def _avg(a, b):
    return (a + b) >> 1


def _half(d):
    """C's d / 2 (truncation toward zero)."""
    return np.where(d < 0, -((-d) >> 1), d >> 1)


def mode_predictions(c: np.ndarray, width: int):
    """The 14 predictions (int32 [n, 4] each) of every pixel from its L, T, TR, TL neighbours in the flat image.
    Only meaningful for pixels with x > 0 and y > 0; TR of the rightmost column is the row's first pixel."""
    n = len(c)
    pad = np.zeros((width + 1, 4), np.int32)
    ext = np.concatenate([pad, c])                  # ext[i + width + 1] == c[i]
    idx = np.arange(n) + width + 1
    L, T, TR, TL = ext[idx - 1], ext[idx - width], ext[np.minimum(idx - width + 1, n + width)], ext[idx - width - 1]
    black = np.zeros_like(c)
    black[:, 0] = 255
    sel = np.abs(T - TL).sum(1) < np.abs(L - TL).sum(1)
    avg_lt = _avg(L, T)
    return [black, L, T, TR, TL, _avg(_avg(L, TR), T), _avg(L, TL), avg_lt, _avg(TL, T), _avg(T, TR),
            _avg(_avg(L, TL), _avg(T, TR)), np.where(sel[:, None], L, T), np.clip(L + T - TL, 0, 255),
            np.clip(avg_lt + _half(avg_lt - TL), 0, 255)]


def predict(p: np.ndarray, width: int, height: int):
    """(residual uint32 [n], modes uint8 [tiles_y, tiles_x]) of the predictor transform over ARGB p."""
    n = width * height
    c = channels(p)
    x = np.arange(n) % width
    y = np.arange(n) // width
    tw, th = -(-width // TILE), -(-height // TILE)
    tile = (y >> TILE_BITS) * tw + (x >> TILE_BITS)
    # edge predictions, the same for every mode
    edge = np.zeros_like(c)
    edge[:, 0] = 255                                 # (0, 0): 0xff000000
    top, left = (y == 0) & (x > 0), (x == 0) & (y > 0)
    edge[top] = c[np.nonzero(top)[0] - 1]
    edge[left] = c[np.nonzero(left)[0] - width]
    inner = (x > 0) & (y > 0)
    best_cost = np.full(tw * th, np.iinfo(np.int64).max, np.int64)
    modes = np.zeros(tw * th, np.int64)
    preds = mode_predictions(c, width)
    for m, pr in enumerate(preds):
        pm = np.where(inner[:, None], pr, edge)
        r = ((c - pm) & 0xFF).astype(np.uint8).view(np.int8).astype(np.int64)
        cost = np.bincount(tile, weights=np.abs(r).sum(1), minlength=tw * th).astype(np.int64)
        better = cost < best_cost
        best_cost[better], modes[better] = cost[better], m
    pm = np.empty_like(c)
    pix_mode = modes[tile]
    for m, pr in enumerate(preds):
        sel = pix_mode == m
        pm[sel] = pr[sel]
    pm[~inner] = edge[~inner]
    return pack((c - pm) & 0xFF), modes.reshape(th, tw).astype(np.uint8)


def sub_image(modes: np.ndarray) -> np.ndarray:
    """ARGB of the predictor sub-image: alpha 255, the mode in green."""
    return (np.uint32(0xFF000000) | (modes.reshape(-1).astype(np.uint32) << 8)).astype(np.uint32)


# ---------------------------------------------------------------------------------------------------- runs


def tokens(sym: np.ndarray) -> np.ndarray:
    """int64 [n]: 1 = literal, L >= 3 = the first pixel of a copy of L pixels, 0 = a pixel inside a copy."""
    n = len(sym)
    brk = np.ones(n, bool)
    brk[1:] = sym[1:] != sym[:-1]
    starts = np.nonzero(brk)[0]
    ends = np.append(starts[1:], n)
    run = np.cumsum(brk) - 1
    i = np.arange(n)
    start, end = starts[run], ends[run]
    k = i - start - 1
    r = end - start - 1
    q = np.maximum(k, 0) // MAX_COPY
    chunk = np.minimum(MAX_COPY, r - q * MAX_COPY)
    copy = (i > start) & (chunk >= MIN_COPY)
    out = np.ones(n, np.int64)
    out[copy] = 0
    head = copy & (k % MAX_COPY == 0)
    out[head] = chunk[head]
    return out


def length_prefix(length):
    """(prefix code, extra bit count, extra value) of a copy length (1..4096), vectorised."""
    v = np.asarray(length, np.int64) - 1
    h = np.where(v >= 2, np.floor(np.log2(np.maximum(v, 1))).astype(np.int64), 0)
    small = v < 4
    second = np.where(small, 0, (v >> np.maximum(h - 1, 0)) & 1)
    code = np.where(small, v, 2 * h + second)
    nbits = np.where(small, 0, h - 1)
    extra = np.where(small, 0, v & ((1 << np.maximum(nbits, 0)) - 1))
    return code, nbits, extra


def histograms(sym: np.ndarray, tok: np.ndarray):
    """Symbol counts of the five trees over the tokens of one image."""
    lit = tok == 1
    cp = tok >= MIN_COPY
    c = channels(sym[lit])
    code, _, _ = length_prefix(tok[cp])
    green = np.bincount(np.concatenate([c[:, 2], 256 + code]), minlength=ALPHABETS[0])
    return [green, np.bincount(c[:, 1], minlength=256), np.bincount(c[:, 3], minlength=256),
            np.bincount(c[:, 0], minlength=256),
            np.bincount(np.full(int(cp.sum()), LEFT_DIST_SYMBOL), minlength=ALPHABETS[4])]


# ---------------------------------------------------------------------------------------------------- Huffman


def huffman_lengths(counts, limit: int) -> np.ndarray:
    """Code lengths of a Huffman code over `counts`, at most `limit` bits.  Merges the two lightest nodes, ordered by
    (weight, id); a leaf's id is its symbol and the k-th merged node's id is len(counts) + k.  While the deepest leaf
    exceeds `limit`, every used symbol's weight is raised to a floor that starts at 1 and doubles.  One used symbol
    gets length 1; none gives all zeros."""
    counts = np.asarray(counts, np.int64)
    used = [int(s) for s in np.nonzero(counts)[0]]
    out = np.zeros(len(counts), np.int64)
    if len(used) == 1:
        out[used[0]] = 1
    if len(used) < 2:
        return out
    floor = 1
    while True:
        heap = [(max(int(counts[s]), floor), s) for s in used]
        heapq.heapify(heap)
        parent = {}
        nid = len(counts)
        while len(heap) > 1:
            w1, a = heapq.heappop(heap)
            w2, b = heapq.heappop(heap)
            parent[a] = parent[b] = nid
            heapq.heappush(heap, (w1 + w2, nid))
            nid += 1
        depth = {heap[0][1]: 0}
        for node in range(nid - 1, len(counts) - 1, -1):   # merged nodes, root first
            if node in parent:
                depth[node] = depth[parent[node]] + 1
        for s in used:
            out[s] = depth[parent[s]] + 1
        if out.max() <= limit:
            return out
        floor *= 2


def canonical_codes(lengths) -> np.ndarray:
    """Canonical codes (DEFLATE order: by length, then symbol), bit-reversed for an LSB-first writer."""
    lengths = np.asarray(lengths, np.int64)
    codes = np.zeros(len(lengths), np.int64)
    code = 0
    for ln in range(1, 16):
        for s in np.nonzero(lengths == ln)[0]:
            codes[s] = int(format(code, f"0{ln}b")[::-1], 2)
            code += 1
        code <<= 1
    return codes


class Bits:
    """LSB-first bit writer for headers: a list of (value, count)."""

    def __init__(self):
        self.parts = []

    def put(self, value: int, count: int):
        if count:
            assert 0 <= value < (1 << count), (value, count)
            self.parts.append((int(value), int(count)))

    @property
    def size(self):
        return sum(c for _, c in self.parts)

    def bits(self) -> np.ndarray:
        out = []
        for v, c in self.parts:
            out.extend((v >> b) & 1 for b in range(c))
        return np.array(out, np.uint8)


def tree(counts, alphabet: int):
    """(header Bits, effective code lengths, codes) of one tree."""
    counts = np.asarray(counts, np.int64)
    w = Bits()
    used = np.nonzero(counts)[0]
    if len(used) <= 2 and (len(used) == 0 or used[-1] < 256):
        syms = list(used) if len(used) else [0]
        w.put(1, 1)
        w.put(len(syms) - 1, 1)
        if syms[0] < 2:
            w.put(0, 1)
            w.put(int(syms[0]), 1)
        else:
            w.put(1, 1)
            w.put(int(syms[0]), 8)
        if len(syms) == 2:
            w.put(int(syms[1]), 8)
        lengths = np.zeros(alphabet, np.int64)
        codes = np.zeros(alphabet, np.int64)
        if len(syms) == 2:
            lengths[syms] = 1
            codes[syms[1]] = 1
        return w, lengths, codes
    lengths = huffman_lengths(counts, 15)
    cl_lengths = huffman_lengths(np.bincount(lengths, minlength=19), 7)
    w.put(0, 1)
    last = max(i for i, s in enumerate(CL_ORDER) if cl_lengths[s]) if cl_lengths.any() else 0
    num = max(4, last + 1)
    w.put(num - 4, 4)
    for i in range(num):
        w.put(int(cl_lengths[CL_ORDER[i]]), 3)
    w.put(0, 1)                                       # max_symbol: the whole alphabet
    single = (cl_lengths > 0).sum() == 1
    cl_codes = canonical_codes(cl_lengths)
    for ln in lengths:
        w.put(int(cl_codes[ln]), 0 if single else int(cl_lengths[ln]))
    return w, lengths, canonical_codes(lengths)


def data_fields(sym, tok, codes):
    """(values, counts) of every field of the coded pixels, in stream order."""
    lit = tok == 1
    idx = np.nonzero(tok)[0]
    c = channels(sym)
    green_c, green_l = codes[0]
    vals, cnts = [], []
    lt = tok[idx]
    is_lit = lt == 1
    code, nbits, extra = length_prefix(np.where(is_lit, 1, lt))
    g_sym = np.where(is_lit, c[idx, 2], 256 + code)
    fields = [(green_c[g_sym], green_l[g_sym]),
              (np.where(is_lit, codes[1][0][c[idx, 1]], extra), np.where(is_lit, codes[1][1][c[idx, 1]], nbits)),
              (np.where(is_lit, codes[2][0][c[idx, 3]], codes[4][0][LEFT_DIST_SYMBOL]),
               np.where(is_lit, codes[2][1][c[idx, 3]], codes[4][1][LEFT_DIST_SYMBOL])),
              (np.where(is_lit, codes[3][0][c[idx, 0]], 0), np.where(is_lit, codes[3][1][c[idx, 0]], 0))]
    assert lit.sum() == is_lit.sum()
    vals = np.stack([f[0] for f in fields], 1).reshape(-1)
    cnts = np.stack([f[1] for f in fields], 1).reshape(-1)
    return vals.astype(np.int64), cnts.astype(np.int64)


def pixel_bits(sym, tok, codes) -> np.ndarray:
    """int64 [n]: the bits each pixel's token takes (0 inside a copy)."""
    _, cnts = data_fields(sym, tok, codes)
    out = np.zeros(len(tok), np.int64)
    out[np.nonzero(tok)[0]] = cnts.reshape(-1, 4).sum(1)
    return out


def bits_of(vals, cnts) -> np.ndarray:
    total = int(cnts.sum())
    pos = np.concatenate([[0], np.cumsum(cnts)[:-1]])
    out = np.zeros(total, np.uint8)
    for b in range(int(cnts.max()) if len(cnts) else 0):
        m = cnts > b
        out[pos[m] + b] = (vals[m] >> b) & 1
    return out


class Image:
    """One entropy-coded image: its symbols, tokens, histograms and codes."""

    def __init__(self, sym):
        self.sym = sym
        self.tok = tokens(sym)
        self.hist = histograms(sym, self.tok)
        self.trees = [tree(h, a) for h, a in zip(self.hist, ALPHABETS)]
        self.codes = [(t[2], t[1]) for t in self.trees]

    def header_bits(self) -> int:
        return sum(t[0].size for t in self.trees)

    def data_bits(self) -> int:
        _, cnts = data_fields(self.sym, self.tok, self.codes)
        return int(cnts.sum())

    def write(self, w: Bits, main: bool):
        w.put(0, 1)                                   # no colour cache
        if main:
            w.put(0, 1)                               # no meta prefix image
        for t in self.trees:
            w.parts.extend(t[0].parts)


def candidates(rgba: np.ndarray, width: int, height: int):
    """[(transforms, Image main, Image sub or None, modes or None)] for candidates 0, 1, 2."""
    p = to_argb(rgba)
    out = [((), Image(p), None, None)]
    for sg in (False, True):
        src = subtract_green(p) if sg else p
        res, modes = predict(src, width, height)
        out.append((("green", "pred") if sg else ("pred",), Image(res), Image(sub_image(modes)), modes))
    return out


def encode(rgba: np.ndarray, width: int | None = None, height: int | None = None, info: dict | None = None) -> bytes:
    """The RIFF WEBP/VP8L file of uint8 RGBA [height, width, 4] (or [height * width, 4] with width and height).
    info, if a dict, receives 'candidate', 'bits' (per candidate), 'modes' (the chosen tile modes or None) and
    'pixel_bits' (per pixel of the main image)."""
    rgba = np.ascontiguousarray(rgba, np.uint8)
    if width is None:
        height, width = rgba.shape[:2]
    assert rgba.size == width * height * 4
    if not (1 <= width <= MAX_SIDE and 1 <= height <= MAX_SIDE):
        raise ValueError("VP8L images are 1..16384 pixels on a side")
    cands = candidates(rgba, width, height)
    alpha_used = bool(np.any(rgba.reshape(-1, 4)[:, 3] != 255))
    streams = []
    for transforms, main, sub, _ in cands:
        w = Bits()
        w.put(0x2F, 8)
        w.put(width - 1, 14)
        w.put(height - 1, 14)
        w.put(int(alpha_used), 1)
        w.put(0, 3)
        for t in transforms:
            w.put(1, 1)
            if t == "green":
                w.put(2, 2)
            else:
                w.put(0, 2)
                w.put(TILE_BITS - 2, 3)
                sub.write(w, main=False)
                vals, cnts = data_fields(sub.sym, sub.tok, sub.codes)
                w.parts.extend(zip(vals.tolist(), cnts.tolist()))
        w.put(0, 1)
        main.write(w, main=True)
        streams.append((w, main))
    sizes = [w.size + m.data_bits() for w, m in streams]
    best = int(np.argmin(sizes))
    w, main = streams[best]
    vals, cnts = data_fields(main.sym, main.tok, main.codes)
    bits = np.concatenate([w.bits(), bits_of(vals, cnts)])
    assert len(bits) == sizes[best]
    payload = np.packbits(np.concatenate([bits, np.zeros(-len(bits) % 8, np.uint8)]), bitorder="little").tobytes()
    if info is not None:
        info.update(candidate=best, bits=sizes, modes=cands[best][3], pixel_bits=pixel_bits(main.sym, main.tok,
                                                                                             main.codes))
    chunk = len(payload)
    body = b"WEBP" + b"VP8L" + chunk.to_bytes(4, "little") + payload + b"\0" * (chunk & 1)
    return b"RIFF" + len(body).to_bytes(4, "little") + body


# ---------------------------------------------------------------------------------------------------- test images


def _fib_values(count: int, rng) -> np.ndarray:
    """`count` values in 0..255 whose histogram grows like the Fibonacci numbers (deeper than 15 bits unlimited)."""
    fib = [1, 1]
    while sum(fib) < count:
        fib.append(fib[-1] + fib[-2])
    v = np.repeat(np.arange(len(fib)), fib)[:count]
    return rng.permutation(v).astype(np.uint8)


def sog_textures(n: int = 3000):
    """The seven textures tests/sog_oracle.encode makes for a small synth cloud (cheap deterministic fits)."""
    import sog_oracle as so
    from gsx import synth
    np.random.seed(4)
    fit = lambda v: np.quantile(v.reshape(-1), np.linspace(0, 1, 256)).astype(np.float32)  # noqa: E731
    tex, _, _ = so.encode(synth.structured(n, "mixed", 3), 0, codebook_fit=fit)
    return tex


def cases() -> dict:
    """name -> uint8 RGBA [height, width, 4]: the shapes and symbol statistics the encoder has to get right."""
    rng = np.random.default_rng(2026)
    c = {}
    c["1x1"] = rng.integers(0, 256, (1, 1, 4), dtype=np.uint8)
    c["1xN"] = rng.integers(0, 256, (1, 301, 4), dtype=np.uint8)
    c["Nx1"] = rng.integers(0, 256, (301, 1, 4), dtype=np.uint8)
    c["37x53_noise"] = rng.integers(0, 256, (37, 53, 4), dtype=np.uint8)
    c["constant"] = np.full((40, 33, 4), (12, 200, 7, 255), np.uint8)
    c["transparent"] = np.where(rng.integers(0, 2, (29, 31, 1)) == 0, 0, rng.integers(0, 256, (29, 31, 4))).astype(
        np.uint8)
    c["two_symbols"] = np.where(rng.integers(0, 2, (33, 47, 1)) == 1, np.uint8(200), np.uint8(3)).repeat(4, -1)
    c["all_values"] = np.stack([rng.permutation(np.arange(4096) % 256).reshape(64, 64) for _ in range(4)],
                               -1).astype(np.uint8)
    v = _fib_values(331 * 317, rng).astype(np.int64)     # every channel a bijection of v: rare pixels take ~60 bits
    c["fibonacci"] = np.stack([(37 * v + 11) % 256, v, (101 * v + 7) % 256, (53 * v + 3) % 256],
                              -1).astype(np.uint8).reshape(331, 317, 4)
    long_run = np.full((70, 90, 4), 77, np.uint8)
    long_run[0, 0] = (1, 2, 3, 4)
    long_run[69, 89] = (5, 6, 7, 8)
    c["long_run"] = long_run
    rows = np.zeros((20, 7, 4), np.uint8)
    rows[...] = (rng.integers(0, 4, (20, 1, 1)) * 60).astype(np.uint8)
    rows[::3, 5] = 9
    c["runs_across_rows"] = rows
    y, x = np.mgrid[:48, :48]
    c["wins_raw"] = rng.integers(0, 256, (48, 48, 4), dtype=np.uint8)
    c["wins_predictor"] = np.stack([(x * 5) % 256, (y * 7 + rng.integers(0, 2, (48, 48))) % 256,
                                    (x * 3 + y * 11) % 256, np.full((48, 48), 255)], -1).astype(np.uint8)
    g = np.tile(np.arange(64, dtype=np.uint8)[None, :, None], (40, 1, 4))
    g[..., 3] = 255
    c["wins_subtract_green"] = g
    return c


WINNERS = {"wins_raw": 0, "wins_predictor": 1, "wins_subtract_green": 2}

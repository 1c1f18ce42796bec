"""A Python restatement of the device VP8L (RFC 9649) decoder, gsx/webp_decode.py with csrc/gsx_vp8l.cu.

decode(data) -> uint8 [h, w, 4]: what Pillow's Image.open(...).convert('RGBA') gives for a lossless RIFF WEBP file,
or ValueError for a stream the decoder refuses.  The main image is decoded the device's way: tokens (literal, copy,
cache index) from speculative chunks of bits with guessed pixel positions, the chain walked by bits, each piece's
groups checked at its true position, re-decode rounds, a serial decode from the verified frontier after max_rounds,
then the tokens resolved to pixels.  COUNTERS counts the stream features decoded, so tests can show they were hit.
"""
from __future__ import annotations

import numpy as np

CL_ORDER = (17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
PLANE = ((0, 1), (1, 0), (1, 1), (-1, 1), (0, 2), (2, 0), (1, 2), (-1, 2),
         (2, 1), (-2, 1), (2, 2), (-2, 2), (0, 3), (3, 0), (1, 3), (-1, 3),
         (3, 1), (-3, 1), (2, 3), (-2, 3), (3, 2), (-3, 2), (0, 4), (4, 0),
         (1, 4), (-1, 4), (4, 1), (-4, 1), (3, 3), (-3, 3), (2, 4), (-2, 4),
         (4, 2), (-4, 2), (0, 5), (3, 4), (-3, 4), (4, 3), (-4, 3), (5, 0),
         (1, 5), (-1, 5), (5, 1), (-5, 1), (2, 5), (-2, 5), (5, 2), (-5, 2),
         (4, 4), (-4, 4), (3, 5), (-3, 5), (5, 3), (-5, 3), (0, 6), (6, 0),
         (1, 6), (-1, 6), (6, 1), (-6, 1), (2, 6), (-2, 6), (6, 2), (-6, 2),
         (4, 5), (-4, 5), (5, 4), (-5, 4), (3, 6), (-3, 6), (6, 3), (-6, 3),
         (0, 7), (7, 0), (1, 7), (-1, 7), (5, 5), (-5, 5), (7, 1), (-7, 1),
         (4, 6), (-4, 6), (6, 4), (-6, 4), (2, 7), (-2, 7), (7, 2), (-7, 2),
         (3, 7), (-3, 7), (7, 3), (-7, 3), (5, 6), (-5, 6), (6, 5), (-6, 5),
         (8, 0), (4, 7), (-4, 7), (7, 4), (-7, 4), (8, 1), (8, 2), (6, 6),
         (-6, 6), (8, 3), (5, 7), (-5, 7), (7, 5), (-7, 5), (8, 4), (6, 7),
         (-6, 7), (7, 6), (-7, 6), (8, 5), (7, 7), (-7, 7), (8, 6), (8, 7))
PREDICTOR, CROSS_COLOUR, SUBTRACT_GREEN, COLOUR_INDEXING = range(4)
COUNTERS: dict = {}


def _count(key, n=1):
    COUNTERS[key] = COUNTERS.get(key, 0) + n


class Reader:
    """LSB-first bits of `data`; reading past the end is a truncated stream."""

    def __init__(self, data: bytes, pos: int = 0):
        self.data, self.pos, self.nbits = bytes(data), pos, 8 * len(data)

    def peek(self, n: int) -> int:
        b = self.pos >> 3
        return (int.from_bytes(self.data[b:b + 8], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def read(self, n: int) -> int:
        if self.pos + n > self.nbits:
            raise ValueError("VP8L: truncated stream")
        v = self.peek(n)
        self.pos += n
        return v


class Code:
    """A canonical prefix code from its lengths, libwebp's acceptance rule: not all zero, exactly one used symbol (of
    any length 1..15) -> a 0-bit code, else the lengths must fill the code space exactly."""

    def __init__(self, lengths):
        lengths = list(lengths)
        count = [0] * 16
        for ln in lengths:
            count[ln] += 1
        if count[0] == len(lengths):
            raise ValueError("VP8L: an empty prefix code")
        for ln in range(1, 15):
            if count[ln] > (1 << ln):
                raise ValueError("VP8L: an over-subscribed prefix code")
        if sum(count[1:16]) == 1:
            self.single = next(s for s, ln in enumerate(lengths) if ln)
            _count(f"single_len_{lengths[self.single]}")
            return
        self.single = None
        left = 1
        for ln in range(1, 16):
            left = 2 * left - count[ln]
            if left < 0:
                raise ValueError("VP8L: an over-subscribed prefix code")
        if left:
            raise ValueError("VP8L: an incomplete prefix code")
        self.max = max(ln for ln in lengths)
        self.table = np.zeros(1 << self.max, np.int32)
        code = 0
        for ln in range(1, self.max + 1):
            for s, l in enumerate(lengths):
                if l == ln:
                    rev = int(bin(code)[2:].zfill(ln)[::-1], 2)
                    self.table[rev::1 << ln] = s | ln << 16
                    code += 1
            code <<= 1

    def decode(self, br: Reader) -> int:
        if self.single is not None:
            return self.single
        e = int(self.table[br.peek(self.max)])
        br.read(e >> 16)
        return e & 0xFFFF


def read_code(br: Reader, alphabet: int) -> Code:
    if br.read(1):
        _count("simple_code")
        two = br.read(1)
        lengths = [0] * alphabet
        wide = br.read(1)
        _count("simple_code_8bit" if wide else "simple_code_1bit")
        s0 = br.read(8 if wide else 1)
        # a symbol past the alphabet (only the 40-symbol distance alphabet has room for one) gets no length, as in
        # libwebp: the code is built from the other symbol, and Code refuses a simple code with none
        if s0 < alphabet:
            lengths[s0] = 1
        else:
            _count("simple_code_past_alphabet")
        if two:
            s1 = br.read(8)
            if s1 < alphabet:
                lengths[s1] = 1
            else:
                _count("simple_code_past_alphabet")
            _count("simple_code_2")
        else:
            _count("simple_code_1")
        return Code(lengths)
    _count("normal_code")
    cl = [0] * 19
    for i in range(4 + br.read(4)):
        cl[CL_ORDER[i]] = br.read(3)
    clc = Code(cl)
    if br.read(1):
        max_symbol = 2 + br.read(2 + 2 * br.read(3))
        if max_symbol > alphabet:
            raise ValueError("VP8L: max_symbol past the alphabet")
    else:
        max_symbol = alphabet
    lengths, prev, s = [0] * alphabet, 8, 0
    while s < alphabet:
        if max_symbol == 0:
            break
        max_symbol -= 1
        c = clc.decode(br)
        if c < 16:
            lengths[s] = c
            s += 1
            if c:
                prev = c
            continue
        if c == 16 and s == 0:
            _count("repeat_before_first")
        extra, base = ((2, 3), (3, 3), (7, 11))[c - 16]
        rep = br.read(extra) + base
        if s + rep > alphabet:
            raise ValueError("VP8L: a code-length repeat past the alphabet")
        for _ in range(rep):
            lengths[s] = prev if c == 16 else 0
            s += 1
    return Code(lengths)


def prefix_value(br: Reader, sym: int) -> int:
    if sym < 4:
        return sym + 1
    extra = (sym - 2) >> 1
    return ((2 + (sym & 1)) << extra) + br.read(extra) + 1


def plane_distance(code: int, width: int) -> int:
    if code > 120:
        _count("dist_long")
        return code - 120
    _count("dist_plane")
    dx, dy = PLANE[code - 1]
    return max(1, dx + dy * width)


def read_groups(br: Reader, ngroups: int, cache_bits: int) -> list:
    size = (1 << cache_bits) if cache_bits else 0
    return [[read_code(br, a) for a in (280 + size, 256, 256, 256, 40)] for _ in range(ngroups)]


def next_token(br: Reader, g: list):
    """(kind, a, b): ('lit', argb, 1), ('copy', length, distance code), ('cache', index, 1)."""
    s = g[0].decode(br)
    if s < 256:
        r = g[1].decode(br)
        b = g[2].decode(br)
        a = g[3].decode(br)
        return "lit", (a << 24) | (r << 16) | (s << 8) | b, 1
    if s < 280:
        length = prefix_value(br, s - 256)
        d = g[4].decode(br)
        if d >= 40:
            raise ValueError("VP8L: a distance symbol past 39")
        return "copy", length, prefix_value(br, d)
    return "cache", s - 280, 1


def token_pixels(tok) -> int:
    return tok[1] if tok[0] == "copy" else 1


def resolve(tokens: list, width: int, npix: int, cache_bits: int) -> np.ndarray:
    """Tokens to ARGB pixels, every pixel entering the colour cache."""
    out = np.zeros(npix, np.uint32)
    cache = [0] * (1 << cache_bits) if cache_bits else None
    shift = 32 - cache_bits
    i = 0
    for kind, a, b in tokens:
        if kind == "copy":
            d = plane_distance(b, width)
            if d > i:
                raise ValueError("VP8L: a copy from before the first pixel")
            if i + a > npix:
                raise ValueError("VP8L: a copy past the last pixel")
            _count("copy")
            for _ in range(a):
                out[i] = out[i - d]
                i += 1
        else:
            if i >= npix:
                raise ValueError("VP8L: a pixel past the last pixel")
            if kind == "cache":
                _count("cache_hit")
                out[i] = cache[a]
            else:
                out[i] = a
            i += 1
        if cache is not None:
            for k in range(i - token_pixels((kind, a, b)), i):
                v = int(out[k])
                cache[((0x1E35A7BD * v) & 0xFFFFFFFF) >> shift] = v
    if i != npix:
        raise ValueError("VP8L: the image data ends early")
    return out


def sub_image(br: Reader, w: int, h: int) -> np.ndarray:
    """An entropy-coded sub-image: optional colour cache, one group, no meta prefix codes."""
    cache_bits = read_cache_bits(br)
    g = read_groups(br, 1, cache_bits)[0]
    toks, n = [], 0
    while n < w * h:
        t = next_token(br, g)
        toks.append(t)
        n += token_pixels(t)
    return resolve(toks, w, w * h, cache_bits)


def read_cache_bits(br: Reader) -> int:
    if not br.read(1):
        return 0
    bits = br.read(4)
    if not 1 <= bits <= 11:
        raise ValueError(f"VP8L: colour cache bits {bits}")
    _count("cache")
    return bits


def div(a, b):
    return -(-a // (1 << b))


class Header:
    """Everything before the main image's pixel data."""

    def __init__(self, data: bytes):
        br = Reader(data)
        if len(data) < 5 or br.read(8) != 0x2F:
            raise ValueError("VP8L: no 0x2f signature")
        self.width, self.height = br.read(14) + 1, br.read(14) + 1
        self.alpha_hint = br.read(1)
        if br.read(3):
            raise ValueError("VP8L: version is not 0")
        xs = self.width
        self.transforms, seen = [], set()
        while br.read(1):
            t = br.read(2)
            if t in seen:
                raise ValueError("VP8L: a transform used twice")
            seen.add(t)
            _count(("predictor", "cross_colour", "subtract_green", "colour_indexing")[t])
            if t in (PREDICTOR, CROSS_COLOUR):
                bits = br.read(3) + 2
                img = sub_image(br, div(xs, bits), div(self.height, bits))
                self.transforms.append((t, xs, bits, img))
            elif t == SUBTRACT_GREEN:
                self.transforms.append((t, xs, 0, None))
            else:
                n = br.read(8) + 1
                bits = 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3
                pal = sub_image(br, n, 1)
                c = pal.view(np.uint8).reshape(-1, 4).copy()
                c = np.cumsum(c, axis=0, dtype=np.uint32).astype(np.uint8)   # delta-coded, per byte mod 256
                table = np.zeros(256, np.uint32)
                table[:n] = c.reshape(-1).view(np.uint32)
                self.transforms.append((t, xs, bits, table))
                xs = div(xs, bits)
        self.xsize = xs
        self.cache_bits = read_cache_bits(br)
        self.meta_bits, self.entropy = 0, None
        if br.read(1):
            self.meta_bits = br.read(3) + 2
            img = sub_image(br, div(xs, self.meta_bits), div(self.height, self.meta_bits))
            self.entropy = (img >> 8) & 0xFFFF
        self.ngroups = int(self.entropy.max()) + 1 if self.entropy is not None else 1
        if self.ngroups > 1:
            _count("multi_group")
        self.groups = read_groups(br, self.ngroups, self.cache_bits)
        self.main_bit = br.pos

    def group_at(self, p: int) -> int:
        if self.entropy is None:
            return 0
        y, x = divmod(p, self.xsize)
        if y >= self.height:
            return 0
        tx = div(self.xsize, self.meta_bits)
        return int(self.entropy[(y >> self.meta_bits) * tx + (x >> self.meta_bits)])


def run_job(h: Header, data: bytes, start: int, target: int, guess: int, limit: int | None = None):
    """Decode tokens from bit `start` as if at pixel `guess` until a token ends at or past `target` or the pixels
    reach the image's end.  -> dict(start, stop, tokens, rel (each token's first pixel, relative), groups, npix,
    status 'ok' / 'end' / 'error')."""
    br = Reader(data, start)
    npix = h.xsize * h.height
    toks, rel, groups, n = [], [], [], 0
    status = "ok"
    try:
        while guess + n < npix and (limit is None or len(toks) < limit):
            if br.pos >= target:
                break
            g = h.group_at(guess + n)
            t = next_token(br, h.groups[g])
            toks.append(t)
            rel.append(n)
            groups.append(g)
            n += token_pixels(t)
        else:
            status = "end"
    except ValueError:
        status = "error"
    return dict(start=start, stop=br.pos, tokens=toks, rel=rel, groups=groups, npix=n, status=status, guess=guess)


def main_tokens(h: Header, data: bytes, chunk_bits: int, max_rounds: int, stats: dict) -> list:
    """The chunked speculative walk: jobs at chunk starts with positions guessed from the bit fraction; rounds that
    re-decode, at its chain position, every piece that does not stand, and decode from the stop where the chain
    breaks; after max_rounds a serial decode from the verified frontier."""
    npix = h.xsize * h.height
    nbits = 8 * len(data) - h.main_bit
    nchunks = max(1, -(-nbits // chunk_bits))
    stats.update(chunks=nchunks, false_starts=0, group_mismatches=0, moved_refused=0, rounds=0, serial_fallbacks=0)

    def target(s):
        return h.main_bit + ((s - h.main_bit) // chunk_bits + 1) * chunk_bits

    found = {}
    for c in range(nchunks):
        s = h.main_bit + c * chunk_bits
        found[s] = run_job(h, data, s, target(s), (c * npix) // nchunks if c else 0)
    while True:
        chain, p, pos = [], h.main_bit, 0            # the chain by bits, each piece at its chain position
        while p in found:
            x = dict(found[p], pos=pos)
            chain.append(x)
            pos += x["npix"]
            if x["status"] != "ok":
                break
            p = x["stop"]
        ended = bool(chain) and chain[-1]["status"] != "ok"
        # a piece decoded at another position stands when it stopped at its target short of the image's end and
        # read every token with the group of the token's true position; one that ended, failed or reaches the end
        # may have done so by its guess
        moved = [k for k, x in enumerate(chain) if x["guess"] != x["pos"]]
        refused = [k for k in moved if chain[k]["status"] != "ok" or chain[k]["pos"] + chain[k]["npix"] >= npix]
        flagged = [k for k in moved if k not in refused and h.ngroups > 1 and any(
            h.group_at(chain[k]["pos"] + r) != g for r, g in zip(chain[k]["rel"], chain[k]["groups"]))]
        bad = sorted(refused + flagged)
        if not bad and ended:
            break
        first = bad[0] if bad else len(chain)
        fp, fpos = (chain[first]["start"], chain[first]["pos"]) if bad else (p, pos)
        if stats["rounds"] >= max_rounds:
            stats["serial_fallbacks"] += 1
            chain = chain[:first] + [run_job(h, data, fp, 8 * len(data) + 1, fpos)]
            break
        stats["rounds"] += 1
        stats["group_mismatches"] += len(flagged)
        stats["moved_refused"] += len(refused)
        stats["false_starts"] += int(not ended)
        jobs = {chain[k]["start"]: chain[k]["pos"] for k in bad}
        if not ended:
            jobs[p] = pos
        for y in list(found.values()):
            if y["status"] == "ok" and y["stop"] > fp and y["stop"] not in found:
                jobs.setdefault(y["stop"], y["guess"] + y["npix"])
        for s, g in jobs.items():
            found[s] = run_job(h, data, s, target(s), g)
    last = chain[-1]
    if last["status"] == "error":
        raise ValueError("VP8L: invalid main image data")
    return [t for x in chain for t in x["tokens"]]


def predict_modes(L, T, TR, TL, mode):
    """The predictor of `mode` for one pixel (channel arrays int)."""
    def avg(a, b):
        return (a + b) >> 1

    if mode == 0 or mode >= 14:
        return np.array([0, 0, 0, 255])   # B G R A order below is irrelevant: 0xff000000
    if mode == 1:
        return L
    if mode == 2:
        return T
    if mode == 3:
        return TR
    if mode == 4:
        return TL
    if mode == 5:
        return avg(avg(L, TR), T)
    if mode == 6:
        return avg(L, TL)
    if mode == 7:
        return avg(L, T)
    if mode == 8:
        return avg(TL, T)
    if mode == 9:
        return avg(T, TR)
    if mode == 10:
        return avg(avg(L, TL), avg(T, TR))
    if mode == 11:
        pl = np.abs(T - TL).sum()
        pt = np.abs(L - TL).sum()
        return L if pl < pt else T
    if mode == 12:
        return np.clip(L + T - TL, 0, 255)
    a = avg(L, T)
    return np.clip(a + np.trunc((a - TL) / 2).astype(np.int64), 0, 255)


def inverse(h: Header, argb: np.ndarray) -> np.ndarray:
    px = argb
    for t, xs, bits, img in reversed(h.transforms):
        ch = px.view(np.uint8).reshape(-1, 4).astype(np.int64)   # B, G, R, A
        if t == SUBTRACT_GREEN:
            ch[:, 0] = (ch[:, 0] + ch[:, 1]) & 255
            ch[:, 2] = (ch[:, 2] + ch[:, 1]) & 255
            px = ch.astype(np.uint8).reshape(-1).view(np.uint32)
        elif t == CROSS_COLOUR:
            tx = div(xs, bits)
            for i in range(len(px)):
                y, x = divmod(i, xs)
                m = int(img[(y >> bits) * tx + (x >> bits)])
                g2r, g2b, r2b = [np.int8(np.uint8((m >> s) & 255)) for s in (0, 8, 16)]
                g = int(np.int8(np.uint8(ch[i, 1])))
                r = (ch[i, 2] + ((int(g2r) * g) >> 5)) & 255
                b = (ch[i, 0] + ((int(g2b) * g) >> 5) + ((int(r2b) * int(np.int8(np.uint8(r)))) >> 5)) & 255
                ch[i, 2], ch[i, 0] = r, b
            px = ch.astype(np.uint8).reshape(-1).view(np.uint32)
        elif t == PREDICTOR:
            tx = div(xs, bits)
            out = ch.copy()
            for i in range(len(px)):
                y, x = divmod(i, xs)
                if i == 0:
                    p = np.array([0, 0, 0, 255])
                elif y == 0:
                    p = out[i - 1]
                elif x == 0:
                    p = out[i - xs]
                else:
                    mode = (int(img[(y >> bits) * tx + (x >> bits)]) >> 8) & 15
                    _count(f"mode_{mode}")
                    p = predict_modes(out[i - 1], out[i - xs], out[i - xs + 1], out[i - xs - 1], mode)
                out[i] = (ch[i] + p) & 255
            px = out.astype(np.uint8).reshape(-1).view(np.uint32)
        else:
            # the image before this transform was xs wide; the packed one is div(xs, bits)
            n_per, pw = 1 << bits, div(xs, bits)
            packed = px.reshape(-1, pw)
            x = np.arange(xs)
            g = ((packed[:, x >> bits] >> 8) & 255).astype(np.int64)
            idx = (g >> ((x & (n_per - 1)) * (8 >> bits))) & ((1 << (8 >> bits)) - 1)
            px = img[idx].reshape(-1)
    return px


def container(data: bytes):
    """(VP8L payload, whether Pillow opens it with alpha: the VP8L header's alpha hint), or None for what the device
    decoder leaves to Pillow."""
    data = bytes(data)
    if len(data) < 20 or data[:4] != b"RIFF" or data[8:12] != b"WEBP":
        return None
    pos, vp8x_alpha = 12, None
    while pos + 8 <= len(data):
        tag, size = data[pos:pos + 4], int.from_bytes(data[pos + 4:pos + 8], "little")
        body = data[pos + 8:pos + 8 + size]
        if tag == b"VP8X":
            if pos != 12 or size < 10 or (body[0] & 0x02):     # animation
                return None
            vp8x_alpha = bool(body[0] & 0x10)
        elif tag == b"VP8L":
            if len(body) < 5:
                raise ValueError("VP8L: truncated header")
            hint = bool((body[4] >> 4) & 1)
            return body, hint          # Pillow follows the VP8L header's alpha hint, not VP8X's flag
        elif tag in (b"VP8 ", b"ALPH", b"ANIM", b"ANMF") or vp8x_alpha is None:
            return None
        pos += 8 + size + (size & 1)
    return None


def decode(data: bytes, chunk_bits: int = 1 << 12, max_rounds: int = 64, stats: dict | None = None) -> np.ndarray:
    c = container(data)
    if c is None:
        raise ValueError("not a lossless RIFF WEBP file the decoder reads")
    body, alpha = c
    h = Header(body)
    st = {} if stats is None else stats
    toks = main_tokens(h, body, chunk_bits, max_rounds, st)
    argb = resolve(toks, h.xsize, h.xsize * h.height, h.cache_bits)
    px = inverse(h, argb)
    rgba = px.view(np.uint8).reshape(h.height, h.width, 4)[..., [2, 1, 0, 3]].copy()
    if not alpha:
        rgba[..., 3] = 255
    return rgba


# ------------------------------------------------------------------------------------------------ test streams
def _prefix(v: int):
    """(prefix symbol, extra bits, extra value) of a length or distance code v >= 1."""
    d = v - 1
    if d < 4:
        return d, 0, 0
    hb = d.bit_length() - 1
    return 2 * hb + ((d >> (hb - 1)) & 1), hb - 1, d & ((1 << (hb - 1)) - 1)


def riff(body: bytes, vp8x_flags: int | None = None, width: int = 1, height: int = 1) -> bytes:
    """A RIFF WEBP file of the VP8L payload `body`, after a VP8X chunk with `vp8x_flags` when given."""
    def chunk(tag, b):
        return tag + len(b).to_bytes(4, "little") + b + b"\0" * (len(b) & 1)

    out = b""
    if vp8x_flags is not None:
        out += chunk(b"VP8X", bytes([vp8x_flags, 0, 0, 0]) + (width - 1).to_bytes(3, "little")
                     + (height - 1).to_bytes(3, "little"))
    out += chunk(b"VP8L", body)
    return b"RIFF" + (4 + len(out)).to_bytes(4, "little") + b"WEBP" + out


def build(width: int, height: int, tokens: list, cache_bits: int = 0, alpha_hint: int = 1, trailer=None) -> bytes:
    """The VP8L payload of a main image with no transforms, one group and the given tokens ('lit', argb) /
    ('copy', length, distance code) / ('cache', index), its prefix codes built with gsx.webp's Tree.  trailer(w)
    may append raw bits after the header (for malformed streams it replaces the codes and data)."""
    from gsx.webp import BitWriter, Tree
    size = (1 << cache_bits) if cache_bits else 0
    counts = [[0] * a for a in (280 + size, 256, 256, 256, 40)]
    for t in tokens:
        if t[0] == "lit":
            v = t[1]
            counts[0][(v >> 8) & 255] += 1
            counts[1][(v >> 16) & 255] += 1
            counts[2][v & 255] += 1
            counts[3][v >> 24] += 1
        elif t[0] == "copy":
            counts[0][256 + _prefix(t[1])[0]] += 1
            counts[4][_prefix(t[2])[0]] += 1
        else:
            counts[0][280 + t[1]] += 1
    for c in counts:
        if not any(c):
            c[0] = 1
    trees = [Tree(c) for c in counts]
    w = BitWriter()
    w.put(0x2F, 8)
    w.put(width - 1, 14)
    w.put(height - 1, 14)
    w.put(alpha_hint, 1)
    w.put(0, 3)
    w.put(0, 1)                                      # no transform
    if trailer is not None:
        trailer(w)
    else:
        w.put(1 if cache_bits else 0, 1)
        if cache_bits:
            w.put(cache_bits, 4)
        w.put(0, 1)                                  # no meta prefix codes
        for t in trees:
            w.extend(t.desc)

        def sym(k, s):
            used = sum(1 for ln in trees[k].lengths if ln)
            if used > 1:
                w.put(trees[k].codes[s], trees[k].lengths[s])

        for t in tokens:
            if t[0] == "lit":
                v = t[1]
                sym(0, (v >> 8) & 255)
                sym(1, (v >> 16) & 255)
                sym(2, v & 255)
                sym(3, v >> 24)
            elif t[0] == "copy":
                p, nb, x = _prefix(t[1])
                sym(0, 256 + p)
                w.put(x, nb)
                p, nb, x = _prefix(t[2])
                sym(4, p)
                w.put(x, nb)
            else:
                sym(0, 280 + t[1])
    return (w.value | 0).to_bytes((w.size + 7) // 8 + 4, "little")


def pillow_file(rgba: np.ndarray, **kw) -> bytes:
    import io
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(rgba, "RGBA").save(b, "WEBP", lossless=True, **kw)
    return b.getvalue()


def pillow_rgba(data: bytes) -> np.ndarray:
    import io
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGBA"))


def images(seed: int = 0) -> dict:
    """Small RGBA images that steer libwebp to each feature: noise, gradients, half/half (several groups), palettes of
    2, 4, 16 and 200 colours (every bundling width), one row, one column, odd sizes."""
    rng = np.random.default_rng(seed)
    out = {"noise": rng.integers(0, 256, (23, 37, 4), dtype=np.uint8)}
    y, x = np.mgrid[0:40, 0:50]
    out["gradient"] = np.stack([x * 5, y * 6, (x + y) * 2, 255 - x], -1).astype(np.uint8)
    y, x = np.mgrid[0:70, 0:90]
    half = np.stack([x * 3, y, x ^ y, np.full_like(x, 255)], -1).astype(np.uint8)
    half[:, 45:] = rng.integers(0, 256, (70, 45, 4))
    out["half"] = half
    for k in (2, 4, 16, 200):
        pal = rng.integers(0, 256, (k, 4), dtype=np.uint8)
        out[f"palette{k}"] = pal[rng.integers(0, k, (19, 33))]
    out["column"] = rng.integers(0, 256, (17, 1, 4), dtype=np.uint8)
    out["row"] = rng.integers(0, 256, (1, 17, 4), dtype=np.uint8)
    out["odd"] = (rng.integers(0, 4, (67, 131, 4)) * 60).astype(np.uint8)
    return out


def pillow_cases() -> dict:
    """name -> file: the mixed image at methods 0..6 x qualities 0 / 50 / 100, every other image at three settings."""
    ims = images()
    out = {}
    for m in range(7):
        for q in (0, 50, 100):
            out[f"half_m{m}_q{q}"] = pillow_file(ims["half"], method=m, quality=q)
    for name, a in ims.items():
        if name != "half":
            for m, q in ((0, 0), (1, 100), (6, 100)):
                out[f"{name}_m{m}_q{q}"] = pillow_file(a, method=m, quality=q)
    return out


def built_cases() -> dict:
    """name -> file: hand-built streams -- all cache tokens, all copies, distance codes on both sides of 120, and the
    alpha hint / VP8X alpha flag combinations."""
    rng = np.random.default_rng(5)
    out = {}
    lits = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, 16, dtype=np.uint64)]
    toks = list(lits)
    for k in range(200):
        v = lits[k % 16][1]
        toks.append(("cache", ((0x1E35A7BD * v) & 0xFFFFFFFF) >> (32 - 6)))
    out["all_cache"] = riff(build(27, delta_h(216, 27), toks, cache_bits=6))
    toks = [("lit", 0xFF102030)] + [("copy", 37, 121)] * 7 + [("copy", 12, 2)]
    out["all_copies"] = riff(build(16, 17, toks))
    toks = lits + lits[::-1] + [("copy", 20, c) for c in (1, 2, 121, 130, 3, 4, 50, 120)]
    out["plane_codes"] = riff(build(16, delta_h(32 + 160, 16), toks))
    px = [("lit", int(v)) for v in rng.integers(0, 2 ** 32, 12, dtype=np.uint64)]
    for hint in (0, 1):
        out[f"alpha_hint{hint}"] = riff(build(4, 3, px, alpha_hint=hint))
        for flags in (0x00, 0x10):
            out[f"vp8x{flags:02x}_hint{hint}"] = riff(build(4, 3, px, alpha_hint=hint), flags, 4, 3)
    return out


def delta_h(npix: int, width: int) -> int:
    assert npix % width == 0
    return npix // width


def coded(width: int, tokens: list, cache_bits: int = 0, main: bool = False, meta=None):
    """The bits of one entropy-coded image of `width` columns: its cache bits, for the main image the meta prefix
    flag (meta = (bits, entropy image as a list of group indices per tile, tile columns) or None), every group's five
    codes (gsx.webp's Tree) and the tokens, each coded with the group of its first pixel."""
    from gsx.webp import BitWriter, Tree
    w = BitWriter()
    w.put(1 if cache_bits else 0, 1)
    if cache_bits:
        w.put(cache_bits, 4)
    ngroups, group_of = 1, (lambda p: 0)
    if main:
        w.put(1 if meta else 0, 1)
        if meta:
            bits, ent, tx = meta
            w.put(bits - 2, 3)
            w.extend(coded(tx, [("lit", 0xFF000000 | g << 8) for g in ent]))
            ngroups = max(ent) + 1

            def group_of(p):
                y, x = divmod(p, width)
                return ent[(y >> bits) * tx + (x >> bits)]
    size = (1 << cache_bits) if cache_bits else 0
    counts = [[[0] * a for a in (280 + size, 256, 256, 256, 40)] for _ in range(ngroups)]
    pos, coded_toks = 0, []
    for t in tokens:
        c = counts[group_of(pos)]
        coded_toks.append((group_of(pos), t))
        if t[0] == "lit":
            v = t[1]
            c[0][(v >> 8) & 255] += 1
            c[1][(v >> 16) & 255] += 1
            c[2][v & 255] += 1
            c[3][v >> 24] += 1
            pos += 1
        elif t[0] == "copy":
            c[0][256 + _prefix(t[1])[0]] += 1
            c[4][_prefix(t[2])[0]] += 1
            pos += t[1]
        else:
            c[0][280 + t[1]] += 1
            pos += 1
    trees = []
    for g in counts:
        for c in g:
            if not any(c):
                c[0] = 1
        trees.append([Tree(c) for c in g])
        for t in trees[-1]:
            w.extend(t.desc)

    def sym(g, k, s):
        tr = trees[g][k]
        if sum(1 for ln in tr.lengths if ln) > 1:
            w.put(tr.codes[s], tr.lengths[s])

    for g, t in coded_toks:
        if t[0] == "lit":
            v = t[1]
            sym(g, 0, (v >> 8) & 255)
            sym(g, 1, (v >> 16) & 255)
            sym(g, 2, v & 255)
            sym(g, 3, v >> 24)
        elif t[0] == "copy":
            p, nb, x = _prefix(t[1])
            sym(g, 0, 256 + p)
            w.put(x, nb)
            p, nb, x = _prefix(t[2])
            sym(g, 4, p)
            w.put(x, nb)
        else:
            sym(g, 0, 280 + t[1])
    return w


def compose(width: int, height: int, main_tokens: list, transforms=(), cache_bits: int = 0, meta=None,
            alpha_hint: int = 1) -> bytes:
    """A RIFF WEBP file built token by token.  transforms, in reading order: ('predictor' | 'cross', bits, tile
    tokens, tile cache bits), ('green',), ('palette', colours, palette tokens, palette cache bits) -- the palette
    tokens code the delta-coded colour table.  main_tokens are at the width the transforms leave."""
    from gsx.webp import BitWriter
    w = BitWriter()
    w.put(0x2F, 8)
    w.put(width - 1, 14)
    w.put(height - 1, 14)
    w.put(alpha_hint, 1)
    w.put(0, 3)
    xs = width
    for t in transforms:
        w.put(1, 1)
        if t[0] in ("predictor", "cross"):
            w.put(0 if t[0] == "predictor" else 1, 2)
            w.put(t[1] - 2, 3)
            w.extend(coded(div(xs, t[1]), t[2], t[3]))
        elif t[0] == "green":
            w.put(2, 2)
        else:
            n = t[1]
            w.put(3, 2)
            w.put(n - 1, 8)
            w.extend(coded(n, t[2], t[3]))
            xs = div(xs, 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3)
    w.put(0, 1)
    w.extend(coded(xs, main_tokens, cache_bits, main=True, meta=meta))
    return riff(w.value.to_bytes((w.size + 7) // 8 + 4, "little"))


def cache_index(v: int, bits: int) -> int:
    return ((0x1E35A7BD * v) & 0xFFFFFFFF) >> (32 - bits)

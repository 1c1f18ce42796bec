"""Pure-Python model of gsx.deflate.gunzip's chunked DEFLATE decoder (csrc/gsx_inflate.cu), for tests only.

The same stages as the device, one function each:
  find      the first plausible block start in a chunk's span of bits: a dynamic block whose header is valid and
            whose trial decode reaches its end-of-block, or a stored block with LEN = ~NLEN and zero padding
  run       decode from a start until the first block end at or past a target bit (or the final block), into 16-bit
            symbols: a byte, or MARK | w for byte w of the unknown 32 KiB window before the start
  inflate   speculate every chunk, walk the chain (re-decode where a chunk's start is not where the chain stopped;
            re-run a chunk that overflowed its capacity with 8x more), then resolve the markers: tails in chain order,
            heads in any order
  gunzip    members, headers, trailers and zero padding as CPython's gzip.decompress
Errors are the classes gzip.decompress raises: EOFError, gzip.BadGzipFile, zlib.error.  COUNTERS counts the code
lengths, incomplete codes, stored blocks, long lengths and distances and capacity overflows that decodes reached.
"""
from __future__ import annotations

import gzip
import struct
import zlib

MARK = 0x8000
WINDOW = 32768
COUNTERS: dict = {}      # what the decodes since the last clear reached, so tests can show a case hits its path


def _count(key, n=1):
    COUNTERS[key] = COUNTERS.get(key, 0) + n

OK, FINAL, EOF, DATA, OVERFLOW = range(5)

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
         258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class RanOut(Exception):
    pass


class Bad(Exception):
    pass


class Full(Exception):
    pass


class Reader:
    def __init__(self, data: bytes, pos: int):
        self.d, self.n, self.pos = data, 8 * len(data), pos

    def bits(self, k: int) -> int:
        if self.pos + k > self.n:
            raise RanOut
        p = self.pos
        v = (int.from_bytes(self.d[p >> 3:(p + k + 7) >> 3], "little") >> (p & 7)) & ((1 << k) - 1)
        self.pos += k
        return v


class Code:
    """Canonical Huffman code of `lengths` as zlib's inflate_table judges it: over-subscribed, incomplete, empty."""

    def __init__(self, lengths, name: str = ""):
        self.name = name
        self.count = [0] * 16
        for n in lengths:
            self.count[n] += 1
        self.count[0] = 0
        self.syms = [s for n in range(1, 16) for s, m in enumerate(lengths) if m == n]
        self.max = max([n for n in range(1, 16) if self.count[n]], default=0)
        left = 1
        self.over = False
        for n in range(1, 16):
            left = 2 * left - self.count[n]
            if left < 0:
                self.over = True
                break
        self.incomplete = not self.over and left > 0

    def decode(self, r: Reader) -> int:
        code = first = index = 0
        for n in range(1, 16):
            code |= r.bits(1)
            c = self.count[n]
            if code - c < first:
                if self.name:
                    _count(f"{self.name}_len_{n}")
                return self.syms[index + code - first]
            if n >= self.max:
                raise Bad("invalid code")        # zlib reads max(1, longest code) bits of an incomplete code
            index += c
            first = (first + c) << 1
            code <<= 1
        raise Bad("invalid code")


FIXED_LIT = Code([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
FIXED_DIST = Code([5] * 32)


def dynamic_codes(r: Reader):
    """The codes of a dynamic block's header, with zlib's checks in zlib's order."""
    nlen, ndist, ncode = r.bits(5) + 257, r.bits(5) + 1, r.bits(4) + 4
    if nlen > 286 or ndist > 30:
        raise Bad("too many length or distance symbols")
    cl = [0] * 19
    for i in range(ncode):
        cl[CLORDER[i]] = r.bits(3)
    clc = Code(cl)
    if clc.over or (clc.incomplete and clc.max > 0):
        raise Bad("invalid code lengths set")
    if not clc.max:
        _count("cl_empty")
    lens = []
    while len(lens) < nlen + ndist:
        sym = clc.decode(r) if clc.max else (r.bits(1) & 0)   # an empty code-length code reads 1 bit as length 0
        if sym < 16:
            lens.append(sym)
            continue
        if sym == 16:
            copy = 3 + r.bits(2)
            if not lens:
                raise Bad("invalid bit length repeat")
            val = lens[-1]
        else:
            copy, val = (3 + r.bits(3) if sym == 17 else 11 + r.bits(7)), 0
        if len(lens) + copy > nlen + ndist:
            raise Bad("invalid bit length repeat")
        lens += [val] * copy
    if lens[256] == 0:
        raise Bad("invalid code -- missing end-of-block")
    lit, dist = Code(lens[:nlen], "lit"), Code(lens[nlen:], "dist")
    for c in (lit, dist):
        if c.over or (c.incomplete and c.max > 1):      # an empty or one-code set of 1 bit passes
            raise Bad("invalid literal/lengths or distances set")
    if dist.incomplete:
        _count("dist_empty" if dist.max == 0 else "dist_one_code")
    return lit, dist


def block(r: Reader, out, first: bool, cap: int | None) -> bool:
    """Decode one block at r into `out` (None: a trial that keeps no symbols); True when it was the final block."""
    final, kind = r.bits(1), r.bits(2)
    if kind == 3:
        raise Bad("invalid block type")
    if kind == 0:
        r.pos = (r.pos + 7) & ~7
        ln, nl = r.bits(16), r.bits(16)
        if ln != nl ^ 0xFFFF:
            raise Bad("invalid stored block lengths")
        if out is None:
            r.bits(8 * ln) if ln else None
            return bool(final)
        _count(f"stored_len_{ln}" if ln in (0, 65535) else "stored")
        for _ in range(ln):
            if cap is not None and len(out) >= cap:
                _count("overflow_stored")
                raise Full
            out.append(r.bits(8))
        return bool(final)
    lit, dist = (FIXED_LIT, FIXED_DIST) if kind == 1 else dynamic_codes(r)
    made = 0
    while True:
        sym = lit.decode(r)
        if sym < 256:
            if out is not None:
                if cap is not None and len(out) >= cap:
                    _count("overflow_literal")
                    raise Full
                out.append(sym)
            made += 1
            continue
        if sym == 256:
            return bool(final)
        if sym > 285:
            raise Bad("invalid literal/length code")
        length = LBASE[sym - 257] + r.bits(LEXT[sym - 257])
        if length == 258 and out is not None:
            _count("len_285" if sym == 285 else "len_284_31")
        ds = dist.decode(r)
        if ds > 29:
            raise Bad("invalid distance code")
        d = DBASE[ds] + r.bits(DEXT[ds])
        if d == WINDOW and out is not None:
            _count("dist_32768")
        if first and d > (len(out) if out is not None else made):
            raise Bad("invalid distance too far back")
        made += length
        if out is None:
            continue
        if cap is not None and len(out) + length > cap:
            _count("overflow_copy")
            raise Full
        for _ in range(length):
            s = len(out) - d
            out.append(out[s] if s >= 0 else MARK | (WINDOW + s))


def stored_at(body: bytes, b: int) -> bool:
    """A stored block header at bit b: BTYPE 00, zero bits to the byte boundary, LEN = ~NLEN."""
    r = Reader(body, b)
    try:
        r.bits(1)
        if r.bits(2):
            return False
        if r.bits((8 - r.pos % 8) % 8):
            return False
        return r.bits(16) == r.bits(16) ^ 0xFFFF
    except RanOut:
        return False


def plausible(body: bytes, b: int) -> bool:
    """The finder's test of bit offset b: a dynamic block that decodes to its end-of-block, or a stored block whose
    padding bits are zero and whose LEN = ~NLEN -- unless it starts inside a byte and the next byte boundary holds a
    stored header too (the zero bits before a byte-aligned header would pass, reading the header byte and LEN as
    LEN / NLEN)."""
    r = Reader(body, b)
    try:
        r.bits(1)
        kind = r.bits(2)
        if kind == 0:
            return stored_at(body, b) and not (b % 8 and stored_at(body, (b + 7) & ~7))
        if kind != 2:
            return False
        r.pos = b
        block(r, None, False, None)
        return True
    except (RanOut, Bad):
        return False


def find(body: bytes, lo: int, hi: int) -> int:
    """First plausible block start in [lo, hi), or -1."""
    for b in range(lo, min(hi, 8 * len(body))):
        if plausible(body, b):
            return b
    return -1


def run(body: bytes, start: int, target: int, first: bool, cap: int):
    """Decode blocks from `start` until one ends at or past `target`, or the final block ends.
    -> dict(start, stop, syms, status, last_marker)."""
    r, out, status = Reader(body, start), [], OK
    stop = start
    try:
        while True:
            final = block(r, out, first, cap)
            stop = r.pos
            if final:
                status = FINAL
                break
            if stop >= target:
                break
    except RanOut:
        status = EOF
    except Bad:
        status = DATA
    except Full:
        status = OVERFLOW
    last = max((i for i, s in enumerate(out) if s & MARK), default=-1)
    return dict(start=start, stop=stop, syms=out, status=status, last_marker=last)


def inflate(body: bytes, chunk_bytes: int, ratio: int = 4, stats: dict | None = None):
    """The raw DEFLATE stream at the start of `body` -> (its bytes, bit offset where it ends).  zlib.error for a
    malformed stream, EOFError when `body` ends before the final block does."""
    cb = 8 * chunk_bytes
    nchunks = max(1, -(-8 * len(body) // cb))
    cap = ratio * chunk_bytes
    spec = []
    for c in range(nchunks):
        s = 0 if c == 0 else find(body, c * cb, (c + 1) * cb)
        spec.append(run(body, s, (c + 1) * cb, c == 0, cap) if s >= 0 else None)
    st = dict(chunks=nchunks, false_starts=0, redecoded=0, overflow_reruns=0)
    grow = cap
    while any(x is not None and x["status"] == OVERFLOW for x in spec):     # batched re-runs of every overflow
        grow *= 8
        for c, x in enumerate(spec):
            if x is not None and x["status"] == OVERFLOW:
                spec[c] = run(body, x["start"], (c + 1) * cb, c == 0, grow)
                st["overflow_reruns"] += 1
    chain, p = [], 0
    while True:
        c = p // cb
        x = spec[c] if c < nchunks else None
        if x is None or x["start"] != p:
            if x is not None and x["start"] >= 0:
                st["false_starts"] += 1
            st["redecoded"] += 1
            x, g = run(body, p, (c + 1) * cb, p == 0, cap), cap
            while x["status"] == OVERFLOW:
                g *= 8
                st["overflow_reruns"] += 1
                x = run(body, p, (c + 1) * cb, p == 0, g)
        chain.append(x)
        if x["status"] != OK:
            break
        p = x["stop"]
    st["chain"] = [(x["start"], x["stop"]) for x in chain]
    if stats is not None:
        for key, v in st.items():
            stats[key] = stats.get(key, 0) + v if key != "chain" else stats.get(key, []) + v
    if chain[-1]["status"] == DATA:
        raise zlib.error("invalid deflate stream")
    out, far = resolve(chain)
    if far is not None:
        raise zlib.error(f"invalid distance too far back (output byte {far})")
    if chain[-1]["status"] == EOF:
        raise EOFError("Compressed file ended before the end-of-stream marker was reached")
    return bytes(out), chain[-1]["stop"]


def resolve(chain):
    """Write the chain's symbols at their offsets (an exclusive scan of the lengths).  Pass 1 writes the bytes; pass 2
    walks the pieces in order over their last 32 KiB (the next piece's window), from the first to the last marker
    there; pass 3 replaces the markers before that.  -> (bytes, the first output byte whose marker lands before the
    first byte, or None)."""
    offs, total = [], 0
    for x in chain:
        offs.append(total)
        total += len(x["syms"])
    out, far = bytearray(total), None

    def fill(x, off, lo, hi):
        nonlocal far
        for i in range(lo, hi):
            s = x["syms"][i]
            if s & MARK:
                t = off - WINDOW + (s & ~MARK)
                if t < 0:
                    far = off + i if far is None else min(far, off + i)
                else:
                    out[off + i] = out[t]

    for x, off in zip(chain, offs):
        for i, s in enumerate(x["syms"]):
            if not s & MARK:
                out[off + i] = s
    walk = []
    for x, off in zip(chain, offs):
        n, last = len(x["syms"]), x["last_marker"]
        lo = max(0, n - WINDOW)
        walk.append((lo, last + 1) if last >= lo else (n, n))
        fill(x, off, *walk[-1])
    for x, off, (lo, _) in zip(chain, offs, walk):
        fill(x, off, 0, lo)
    return out, far


def header_end(data: bytes, pos: int):
    """CPython's gzip._read_gzip_header at `pos`: None at the end of data, else the offset of the DEFLATE body."""
    if pos >= len(data):
        return None
    if data[pos:pos + 2] != b"\x1f\x8b":
        raise gzip.BadGzipFile(f"Not a gzipped file ({data[pos:pos + 2]!r})")

    def exact(k):
        nonlocal pos
        if len(data) - pos < k:
            raise EOFError("Compressed file ended before the end-of-stream marker was reached")
        pos += k
        return data[pos - k:pos]

    pos += 2
    method, flag = struct.unpack("<BBIxx", exact(8))[:2]
    if method != 8:
        raise gzip.BadGzipFile("Unknown compression method")
    if flag & 4:
        exact(struct.unpack("<H", exact(2))[0])
    for bit in (8, 16):
        if flag & bit:
            z = data.find(b"\x00", pos)
            pos = len(data) if z < 0 else z + 1
    if flag & 2:
        exact(2)
    return pos


def gunzip(data: bytes, chunk_bytes: int, stats: dict | None = None) -> bytes:
    """gzip.decompress(data) through the chunked model."""
    out, pos = [], 0
    while True:
        h = header_end(data, pos)
        if h is None:
            return b"".join(out)
        member, end = inflate(data[h:], chunk_bytes, stats=stats)
        t = h + (end + 7) // 8
        if len(data) - t < 8:
            raise EOFError("Compressed file ended before the end-of-stream marker was reached")
        crc, size = struct.unpack_from("<II", data, t)
        if crc != zlib.crc32(member):
            raise gzip.BadGzipFile("CRC check failed")
        if size != len(member) & 0xFFFFFFFF:
            raise gzip.BadGzipFile("Incorrect length of data produced")
        out.append(member)
        pos = t + 8
        while pos < len(data) and data[pos] == 0:
            pos += 1


# ------------------------------------------------------------------------------------------- the seeded test corpus
def payloads(n: int = 20_000) -> dict:
    """Seeded payloads of about n bytes (the periods of 32 KiB are longer: two periods and 5000 bytes)."""
    import numpy as np
    rng = np.random.default_rng(1952)
    words = [bytes(rng.integers(97, 123, rng.integers(2, 9), dtype=np.uint8)) for _ in range(300)]
    text = b" ".join(words[i] for i in rng.integers(0, len(words), n // 5))[:n]
    rec = np.round(np.cumsum(rng.normal(0, 1, (n // 16, 4)), 0)).astype(np.int32).tobytes()
    period = lambda p: (bytes(rng.integers(0, 256, p, dtype=np.uint8)) * (-(-(2 * p + 5000) // p)))
    return {
        "empty": b"", "one": b"\x7f", "random": bytes(rng.integers(0, 256, n, dtype=np.uint8)), "text": text,
        "records": rec, "zeros": bytes(n), "period3": period(3)[:n], "period7": period(7)[:n],
        "period32768": period(32768), "period32769": period(32769),
        "match258": b"q" + b"a" * 258 + b"b" * 517 + b"c" * 259,
    }


def gz(raw: bytes, flags: int = 0, extra: bytes = b"", name: bytes = b"", comment: bytes = b"") -> bytes:
    """A gzip member around raw DEFLATE bytes (`raw` ends with its 8-byte trailer), with the header flags given."""
    h = struct.pack("<BBBBLBB", 0x1F, 0x8B, 8, flags, 0, 0, 3)
    if flags & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flags & 8:
        h += name + b"\x00"
    if flags & 16:
        h += comment + b"\x00"
    if flags & 2:
        h += b"\xab\xcd"
    return h + raw


def raw_deflate(data: bytes, level=6, wbits=15, mem=8, strategy=0, flushes=()) -> bytes:
    """DEFLATE body + gzip trailer from zlib, flushing with each (offset, mode) of `flushes`."""
    co = zlib.compressobj(level, zlib.DEFLATED, -wbits, mem, strategy)
    out, prev = [], 0
    for off, mode in sorted(flushes):
        out.append(co.compress(data[prev:off]))
        out.append(co.flush(mode))
        prev = off
    out.append(co.compress(data[prev:]) + co.flush())
    return b"".join(out) + struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


class BitWriter:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, val: int, k: int):
        self.v |= (val & ((1 << k) - 1)) << self.n
        self.n += k

    def huff(self, code: int, k: int):     # Huffman codes go MSB first
        self.put(int(f"{code:0{k}b}"[::-1], 2) if k else 0, k)

    def fixed_lit(self, s: int):
        if s < 144:
            self.huff(0x30 + s, 8)
        elif s < 256:
            self.huff(0x190 + s - 144, 9)
        elif s < 280:
            self.huff(s - 256, 7)
        else:
            self.huff(0xC0 + s - 280, 8)

    def align(self):
        self.n = (self.n + 7) & ~7

    def bytes(self) -> bytes:
        return self.v.to_bytes((self.n + 7) // 8, "little")


def _stored(w: BitWriter, data: bytes, final: int, nlen=None):
    w.put(final, 1)
    w.put(0, 2)
    w.align()
    w.put(len(data), 16)
    w.put(len(data) ^ 0xFFFF if nlen is None else nlen, 16)
    for b in data:
        w.put(b, 8)


def _fixed(w: BitWriter, tokens, final=1):
    """tokens: ints (literals / raw lit-len symbols >= 256 without extra bits) or (length, distance) pairs."""
    w.put(final, 1)
    w.put(1, 2)
    for t in tokens:
        if isinstance(t, tuple):
            ln, d = t
            s = max(i for i in range(29) if LBASE[i] <= ln)
            w.fixed_lit(257 + s)
            w.put(ln - LBASE[s], LEXT[s])
            ds = max(i for i in range(30) if DBASE[i] <= d)
            w.huff(ds, 5)
            w.put(d - DBASE[ds], DEXT[ds])
        else:
            w.fixed_lit(t)
    w.fixed_lit(256)


def _trailer(data: bytes) -> bytes:
    return struct.pack("<II", zlib.crc32(data), len(data) & 0xFFFFFFFF)


def _dyn_head(w: BitWriter, final, hlit, hdist, cl4, syms):
    """A dynamic block header with HCLEN 4: code-length lengths cl4 for symbols 16, 17, 18, 0, then the code-length
    symbols `syms` ((symbol, extra value) pairs, coded canonically)."""
    w.put(final, 1)
    w.put(2, 2)
    w.put(hlit, 5)
    w.put(hdist, 5)
    w.put(0, 4)
    for x in cl4:
        w.put(x, 3)
    lens = dict(zip((16, 17, 18, 0), cl4))
    codes, code = {}, 0
    for n in range(1, 8):
        for s in sorted(s for s, m in lens.items() if m == n):
            codes[s] = (code, n)
            code += 1
        code <<= 1
    for s, extra in syms:
        w.huff(*codes[s])
        if s >= 16:
            w.put(extra, {16: 2, 17: 3, 18: 7}[s])


def malformed() -> dict:
    """Hand-built members, each failing one of zlib's checks -> the exception class gzip.decompress raises."""
    cases = {}

    def member(build, data=b"x"):
        w = BitWriter()
        build(w)
        return gz(w.bytes() + _trailer(data))

    cases["block_type_3"] = member(lambda w: (w.put(1, 1), w.put(3, 2)))
    cases["stored_nlen"] = member(lambda w: _stored(w, b"abc", 1, nlen=0x1234), b"abc")
    cases["fixed_lit_286"] = member(lambda w: _fixed(w, [65, 286]))
    cases["fixed_lit_287"] = member(lambda w: _fixed(w, [65, 287]))
    cases["fixed_dist_30"] = member(lambda w: (w.put(1, 1), w.put(1, 2), w.fixed_lit(65), w.fixed_lit(257),
                                               w.huff(30, 5), w.put(0, 8)))
    cases["fixed_dist_31"] = member(lambda w: (w.put(1, 1), w.put(1, 2), w.fixed_lit(65), w.fixed_lit(257),
                                               w.huff(31, 5), w.put(0, 8)))
    cases["too_many_lengths"] = member(lambda w: (w.put(1, 1), w.put(2, 2), w.put(30, 5), w.put(0, 5), w.put(0, 4),
                                                  w.put(0, 12)))
    cases["too_many_distances"] = member(lambda w: (w.put(1, 1), w.put(2, 2), w.put(0, 5), w.put(30, 5),
                                                    w.put(0, 4), w.put(0, 12)))
    cases["cl_oversubscribed"] = member(lambda w: _dyn_head(w, 1, 0, 0, (1, 1, 1, 0), []))
    cases["cl_incomplete"] = member(lambda w: _dyn_head(w, 1, 0, 0, (1, 0, 0, 0), []))
    cases["repeat_first"] = member(lambda w: _dyn_head(w, 1, 0, 0, (1, 0, 0, 1), [(16, 0)]))
    cases["repeat_past_end"] = member(lambda w: _dyn_head(w, 1, 0, 0, (0, 0, 1, 1), [(18, 127), (18, 127)]))
    cases["missing_eob"] = member(lambda w: _dyn_head(w, 1, 0, 0, (0, 0, 1, 1), [(18, 127), (18, 109)]))
    # literal/length lengths: 0..255 at 8 bits, 256 at 8 bits -> over-subscribed (257 codes of 8 bits)
    lit = [8] * 255 + [9, 9]                     # 257 literal/length lengths forming a complete code
    cases["lit_oversubscribed"] = member(lambda w: _dyn_lit(w, [8] * 257, [1]))
    cases["lit_incomplete"] = member(lambda w: _dyn_lit(w, [9] * 200 + [0] * 56 + [9], [1]))
    cases["dist_incomplete"] = member(lambda w: _dyn_lit(w, lit, [2]))
    cases["dist_oversubscribed"] = member(lambda w: _dyn_lit(w, lit, [1, 1, 1]))
    cases["far_chunk0"] = member(lambda w: _fixed(w, [65, 66, (3, 3)]), b"ABABA")
    far_later = b"".join(bytes([i]) * 7 for i in range(256)) * 3
    w = BitWriter()
    _stored(w, far_later, 0)
    _fixed(w, [65, (10, 30000)])
    cases["far_later_chunk"] = gz(w.bytes() + _trailer(far_later + b"A" * 11))
    good = gzip.compress(b"hello, hello, hello world" * 40, 6, mtime=0)
    cases["bad_crc"] = good[:-8] + bytes([good[-8] ^ 1]) + good[-7:]
    cases["bad_isize"] = good[:-4] + bytes([good[-4] ^ 1]) + good[-3:]
    cases["trailer_short"] = good[:-3]
    cases["trailing_garbage"] = good + b"\x00\x00garbage"
    cases["lone_1f"] = good + b"\x1f"
    cases["second_header_short"] = good + good[:6]
    cases["bad_magic"] = b"\x1f\x8c" + good[2:]
    cases["bad_method"] = good[:2] + b"\x07" + good[3:]
    cases["header_only"] = good[:10]
    cases["extra_cut"] = gz(b"", 4, extra=b"0123456789")[:14]
    return cases


def _dyn_lit(w: BitWriter, lit, dist):
    """A final dynamic block with these literal/length and distance code lengths, written with code-length symbols
    0..15 at 4 bits each; no data after the header."""
    lens = list(lit) + list(dist)
    w.put(1, 1)
    w.put(2, 2)
    w.put(len(lit) - 257, 5)
    w.put(len(dist) - 1, 5)
    w.put(15, 4)                  # HCLEN 19
    cl = {s: 4 if s < 16 else 0 for s in range(19)}     # 16 codes of 4 bits: a complete code-length code
    for s in CLORDER:
        w.put(cl[s], 3)
    codes, code = {}, 0
    for n in range(1, 8):
        for s in sorted(s for s in cl if cl[s] == n):
            codes[s] = (code, n)
            code += 1
        code <<= 1
    for x in lens:
        w.huff(*codes[x])
    w.put(0, 16)


def streams(n: int = 20_000, seed: int = 7) -> dict:
    """{name: gzip file} over the payloads: zlib levels, strategies, memLevels, window bits, flushes, multi-member
    files, every header flag, the finder's decoys and gsx's own encoder (tests/deflate_oracle.py's bytes)."""
    import numpy as np
    import deflate_oracle as do
    rng = np.random.default_rng(seed)
    P = payloads(n)
    out = {}
    for name, data in P.items():
        for level in range(10):
            if level in (0, 1, 6, 9) or name in ("text", "records"):
                out[f"{name}_l{level}"] = gz(raw_deflate(data, level))
    for name in ("text", "records", "period7", "zeros"):
        data = P[name]
        for s, sname in ((zlib.Z_FILTERED, "filtered"), (zlib.Z_HUFFMAN_ONLY, "huffman"), (zlib.Z_RLE, "rle"),
                         (zlib.Z_FIXED, "fixed")):
            out[f"{name}_{sname}"] = gz(raw_deflate(data, 6, strategy=s))
        for mem in (1, 9):
            out[f"{name}_mem{mem}"] = gz(raw_deflate(data, 6, mem=mem))
        for wb in range(9, 16):
            out[f"{name}_wbits{wb}"] = gz(raw_deflate(data, 6, wbits=wb))
        for mode, mname in ((zlib.Z_SYNC_FLUSH, "sync"), (zlib.Z_FULL_FLUSH, "full"), (zlib.Z_BLOCK, "block")):
            offs = sorted(int(x) for x in rng.integers(0, max(len(data), 1), 6))
            out[f"{name}_{mname}"] = gz(raw_deflate(data, 6, flushes=[(o, mode) for o in offs]))
        x = np.frombuffer(data, np.uint8)
        out[f"{name}_gsx6"] = do.gzip_file(x, 6, 0, (len(x) // 3,))
        out[f"{name}_gsx0"] = do.gzip_file(x, 0, 0)
    t = P["text"]
    out["multi_member"] = (gzip.compress(t[:7000], 1, mtime=0) + bytes(5) + gzip.compress(b"", 6, mtime=0) +
                           gzip.compress(t[7000:], 9, mtime=0) + bytes(3))
    for flags in range(32):
        out[f"flags{flags}"] = gz(raw_deflate(t[:3000], 6), flags, b"xy" * 3, b"name.spz", b"a comment")
    out["flags_reserved"] = gz(raw_deflate(t[:3000], 6), 0xE0)
    out["decoy_stored_zlib"] = gzip.compress(zlib.compress(t, 6) * 2, 0, mtime=0)
    out["decoy_recompressed"] = gzip.compress(gzip.compress(P["records"], 6), 1, mtime=0)
    out["empty_file"] = b""
    return out


def corrupted(seed: int = 11) -> dict:
    """Truncations at every byte of a small file and seeded bit flips of a larger one."""
    import numpy as np
    small = gzip.compress(b"abracadabra, abracadabra! " * 8, 6, mtime=0)
    out = {f"trunc{i}": small[:i] for i in range(1, len(small))}
    big = bytearray(gzip.compress(payloads()["text"][:8000], 6, mtime=0))
    rng = np.random.default_rng(seed)
    for k, pos in enumerate(rng.integers(10, len(big) - 8, 48)):
        b = bytearray(big)
        b[pos] ^= 1 << int(rng.integers(0, 8))
        out[f"flip{k}_{pos}"] = bytes(b)
    return out


def expect(data: bytes):
    """gzip.decompress(data), or the exception class it raises."""
    try:
        return gzip.decompress(data)
    except (EOFError, gzip.BadGzipFile, zlib.error) as e:
        return type(e)

"""The DEFLATE decoder (csrc/gsx_inflate.cu, gsx/deflate.py's inflate / gunzip), path by path: Huffman codes at every
length (both sides of the 10-bit and 8-bit fast tables, and the slow path at the end of the input), the incomplete
codes zlib accepts, lengths of 258 and distances of 32768, stored blocks at their limits, the finder's skips and
screens, capacity overflows in each kind of output, and the resolve passes over short, long and too-far-back pieces.

Each case has a seeded builder (inflate_model's BitWriter and block writers).  An unmarked CPU test proves through
inflate_model (its COUNTERS, find() and chains) that the case reaches the path it is named after, and that zlib and the
model agree on it: the model restates the kernel, so only zlib, which neither of them wrote, catches a bug they share.
A `gpu` test asserts the device result equals zlib's, byte for byte or by exception class, and, where the chain
matters, that the device's chain of pieces equals the model's."""
import gzip
import re
import zlib

import numpy as np
import pytest

import inflate_model as m
from inflate_model import BitWriter, LBASE, LEXT, DBASE, DEXT, CLORDER

LIT_FAST, DIST_FAST = 10, 8      # kLitFast, kDistFast: the longest codes the fast tables hold
SCREEN_MAX = 29                  # HLIT / HDIST above this fail the finder's 13-bit screen


# ------------------------------------------------------------------------------------------------ block writers
def full(n: int) -> list:
    """Lengths of a complete code over n symbols (as balanced as canonical codes allow)."""
    from gsx.webp import code_lengths
    return code_lengths([1] * n, 15)


def canon(lengths) -> dict:
    codes, code = {}, 0
    for n in range(1, 16):
        for s, ln in enumerate(lengths):
            if ln == n:
                codes[s] = (code, n)
                code += 1
        code <<= 1
    return codes


def lsym(length: int) -> int:
    return max(i for i in range(29) if LBASE[i] <= length)


def dsym(dist: int) -> int:
    return max(i for i in range(30) if DBASE[i] <= dist)


def put_tokens(w: BitWriter, lc: dict, dc: dict, tokens):
    """tokens: a literal int, (length, distance), or ('sym', lit/len symbol, extra, dist symbol, extra) to pick the
    length symbol (and its extra bits) by hand; a code missing from lc / dc is written as the raw bit string given
    by ('bits', value, count)."""
    for t in tokens:
        if isinstance(t, int):
            w.huff(*lc[t])
        elif t[0] == "bits":
            w.put(t[1], t[2])
        elif t[0] == "sym":
            _, s, x, ds, dx = t
            w.huff(*lc[s])
            w.put(x, LEXT[s - 257])
            w.huff(*dc[ds])
            w.put(dx, DEXT[ds])
        else:
            ln, d = t
            s, ds = lsym(ln), dsym(d)
            w.huff(*lc[257 + s])
            w.put(ln - LBASE[s], LEXT[s])
            w.huff(*dc[ds])
            w.put(d - DBASE[ds], DEXT[ds])


def dyn_block(w: BitWriter, lit, dist, tokens, final=1, eob=True):
    """A dynamic block with these literal/length and distance code lengths (code-length symbols 0..15 at 4 bits each,
    no repeats), then `tokens` and the end-of-block."""
    w.put(final, 1)
    w.put(2, 2)
    w.put(len(lit) - 257, 5)
    w.put(len(dist) - 1, 5)
    w.put(15, 4)
    cl = {s: 4 if s < 16 else 0 for s in range(19)}
    for s in CLORDER:
        w.put(cl[s], 3)
    clc = canon([cl[s] for s in range(19)])
    for x in list(lit) + list(dist):
        w.huff(*clc[x])
    lc, dc = canon(lit), canon(dist)
    put_tokens(w, lc, dc, tokens)
    if eob:
        w.huff(*lc[256])


FIXED_LIT = canon([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
FIXED_DIST = canon([5] * 30)


def fixed_block(w: BitWriter, tokens, final=1):
    w.put(final, 1)
    w.put(1, 2)
    put_tokens(w, FIXED_LIT, FIXED_DIST, tokens)
    w.huff(*FIXED_LIT[256])


def stored_block(w: BitWriter, data: bytes, final=1, pad=0, length=None):
    """A stored block; `pad` fills the bits up to the byte boundary (zlib ignores them), `length` overrides LEN."""
    w.put(final, 1)
    w.put(0, 2)
    k = -w.n % 8
    w.put(pad, k)
    ln = len(data) if length is None else length
    w.put(ln, 16)
    w.put(ln ^ 0xFFFF, 16)
    for b in data:
        w.put(b, 8)


def member(w: BitWriter, data: bytes) -> bytes:
    return m.gz(w.bytes() + m._trailer(data))


def rand(seed, n, lo=0, hi=256) -> bytes:
    return bytes(np.random.default_rng(seed).integers(lo, hi, n, dtype=np.uint8))


# ------------------------------------------------------------------------------------------------ the cases
# Each builder returns (gzip file or raw body, chunk_bytes).  RAW cases are bare DEFLATE bodies for deflate.inflate.
def every_length():
    """Complete codes using every length 1..15: literals 65..76 at 1..12 bits, length symbols 257 / 258 at 13 / 14,
    literal 77 and the end-of-block at 15; distance symbols 0..15 at 1..14, 15, 15.  Every code is used."""
    lit = [0] * 259
    for k, s in enumerate(range(65, 77)):
        lit[s] = k + 1
    lit[257], lit[258], lit[77], lit[256] = 13, 14, 15, 15
    dist = [k + 1 for k in range(14)] + [15, 15]
    rng = np.random.default_rng(1)
    toks = [int(v) for v in rng.integers(65, 78, 400)]
    for ds in range(16):       # a length-3 and a length-4 copy at every distance symbol, its extra bits random
        d = DBASE[ds] + int(rng.integers(0, 1 << DEXT[ds]))
        toks += [(3, d), 66, (4, d), 67]
    w = BitWriter()
    dyn_block(w, lit, dist, toks)
    return member(w, zlib.decompressobj(-15).decompress(w.bytes())), 64


def slow_tail():
    """A raw body whose final fixed-Huffman end-of-block (7 bits) ends the input: fewer than 10 bits remain there, so
    need(kLitFast) fails and the slow path decodes it.  9-bit literals make the body end on a byte boundary."""
    toks = [65, 66, (5, 2)]
    while True:
        w = BitWriter()
        fixed_block(w, toks)
        if w.n % 8 == 0:
            return w.bytes(), None
        toks.append(200)


def dist_one_code(bad=False):
    """A distance code of one symbol at 1 bit (incomplete, zlib accepts it); bad: a copy coded with the missing
    pattern '1', which zlib refuses -- the body ends right after it, so reading past the code runs out of input."""
    lit = full(258)
    w = BitWriter()
    toks = [65, 66, (3, 1), 67]
    if bad:
        toks += [("bits", lc_bits(lit, 257), canon(lit)[257][1]), ("bits", 1, 1)]
    dyn_block(w, lit, [1], toks, eob=not bad)
    return w.bytes(), None


def lc_bits(lengths, s) -> int:
    """The LSB-first stream value of symbol s's code."""
    code, n = canon(lengths)[s]
    return int(f"{code:0{n}b}"[::-1], 2)


def dist_empty(copy=False):
    """An all-zero distance code: valid in a literal-only block; a length symbol after it is an error."""
    lit = full(258)
    w = BitWriter()
    toks = [65, 66, 67]
    if copy:
        toks.append(("bits", lc_bits(lit, 257), canon(lit)[257][1]))
        toks.append(("bits", 0, 8))
    dyn_block(w, lit, [0], toks, eob=not copy)
    data = b"ABC"
    return member(w, data), None


def cl_empty():
    """A code-length code with no lengths: every literal/length and distance length reads as 0 from one bit each,
    so the block has no end-of-block."""
    w = BitWriter()
    w.put(1, 1), w.put(2, 2), w.put(0, 5), w.put(0, 5), w.put(0, 4)
    w.put(0, 12)                                       # four code-length lengths of 0
    w.put(0, 258)
    return member(w, b"x"), None


def long_lengths():
    """Length symbol 285 (258, no extra bits) and 284 with extra bits 31 (also 258, which zlib accepts)."""
    w = BitWriter()
    fixed_block(w, [65, ("sym", 285, 0, 0, 0), ("sym", 284, 31, 0, 0), 66])
    return member(w, b"A" * (1 + 2 * 258) + b"B"), 64


def far_32768_from_start():
    """A copy at distance 32768 whose source is the member's first byte (the first chunk knows it)."""
    head = rand(2, 32768)
    w = BitWriter()
    stored_block(w, head, final=0)
    fixed_block(w, [(258, 32768), 65])
    return member(w, head + head[:258] + b"A"), None


def window_pieces():
    """Pieces that start with copies from their window, 64-byte chunks so each block is a piece:
      A  128 copies of (258, 32768): 33024 markers, the last 32768 the next piece's window;
      B  (258, 32768) first: window marker 0, which is A's marker at count - 32768, then 70 literals;
      C  (258, 1) first: 258 copies of the window's last byte, then 70 literals;
      D  (258, 32768) then 33000 literals: its last marker lies before walk_lo, so only the markers pass reads it."""
    head = rand(3, 32768, 1, 256)
    w = BitWriter()
    stored_block(w, head, final=0)
    fixed_block(w, [(258, 32768)] * 128, final=0)
    fixed_block(w, [(258, 32768)] + [65] * 70, final=0)      # more than 64 bytes: each block crosses a chunk end
    fixed_block(w, [(258, 1)] + [66] * 70, final=0)
    lits = [int(v) for v in np.random.default_rng(4).integers(0, 256, 33000)]
    fixed_block(w, [(258, 32768)] + lits, final=1)
    data = zlib.decompressobj(-15).decompress(w.bytes())
    return member(w, data), 64


def stored_edges():
    """Stored blocks of LEN 0 and LEN 65535, and one right after a fixed-Huffman block (its first bytes are still in
    the bit buffer), one at the job's start."""
    big = rand(5, 65535)
    w = BitWriter()
    stored_block(w, b"", final=0)
    stored_block(w, big, final=0)
    fixed_block(w, [65, 66, (7, 2)], final=0)
    stored_block(w, b"0123456789abcdef", final=0)
    stored_block(w, b"", final=1)
    return member(w, b"" + big + b"ABABABABA" + b"0123456789abcdef"), 64


def stored_past_input():
    """A stored block whose LEN runs past the input."""
    w = BitWriter()
    stored_block(w, b"abcdefghij", final=1, length=1000)
    return m.gz(w.bytes()), None


def stored_padding():
    """A stored block whose padding bits are not zero (zlib ignores them) at the first block boundary of a chunk: the
    finder's stored_at refuses it, so the chain re-decodes there."""
    a, b = rand(6, 100), rand(7, 300)
    w = BitWriter()
    stored_block(w, a, final=0)
    fixed_block(w, [65] * 100, final=0)
    stored_block(w, b, final=1, pad=0b10101)
    return member(w, a + b"A" * 100 + b), 64


def fixed_many():
    """200 fixed-Huffman blocks over about 40 64-byte chunks: the finder skips BTYPE 01, so every chunk after the
    first has no start and the walk takes one round per piece."""
    rng = np.random.default_rng(8)
    w, data = BitWriter(), b""
    for k in range(200):
        lits = [int(v) for v in rng.integers(97, 123, 10)]
        fixed_block(w, lits, final=int(k == 199))
        data += bytes(lits)
    return member(w, data), 64


def decoy_header(hlit, hdist, final=1) -> bytes:
    """The first two bytes of a dynamic block header with these HLIT / HDIST fields."""
    v = final | 2 << 1 | hlit << 3 | hdist << 8
    return v.to_bytes(2, "little")


def screen_decoys():
    """Stored payload bytes holding dynamic headers whose HLIT or HDIST is 30 or 31 (the finder's 13-bit screen skips
    them), then a whole valid dynamic block with HLIT = HDIST = 29, which the screen passes to plausible() and which
    becomes the next chunk's (false) start."""
    w = BitWriter()
    dyn_block(w, full(286), full(30), [70, 71, (4, 2)])
    decoy = w.bytes()
    pay = b"\x00" * 80
    for hl, hd in ((30, 0), (31, 5), (3, 30), (0, 31), (31, 31)):
        pay += decoy_header(hl, hd) + b"\x00" * 6
    pay += decoy + b"\x00" * 40
    w = BitWriter()
    stored_block(w, pay, final=0)
    fixed_block(w, [65])
    return member(w, pay + b"A"), 64


def overflow_literal():
    """1-bit literals: the first chunk's 64 bytes hold more literals than its 256-symbol capacity."""
    lit = [0] * 257
    lit[97], lit[256] = 1, 1
    w = BitWriter()
    dyn_block(w, lit, [1], [97] * 1200)
    return member(w, b"a" * 1200), 64


def overflow_copy():
    """A copy of 258 after one literal: the first chunk overflows inside the copy."""
    w = BitWriter()
    fixed_block(w, [97, (258, 1), 98] + [99] * 80)
    return member(w, b"a" * 259 + b"b" + b"c" * 80), 64


def overflow_stored():
    """A fixed block of 250 symbols, then a stored block: the capacity runs out inside the stored bytes."""
    s = rand(9, 40)
    w = BitWriter()
    fixed_block(w, [97, (249, 1)], final=0)
    stored_block(w, s, final=1)
    return member(w, b"a" * 250 + s), 64


def overflow_then_far():
    """The first chunk overflows inside a copy; past that point it holds a copy from before the member's start, which
    its re-run with more room (still the first job) must refuse."""
    w = BitWriter()
    fixed_block(w, [97, (258, 1)] + [98] * 30 + [(3, 1000)] + [99] * 40)
    return member(w, b"a" * 259 + b"b" * 30 + b"???" + b"c" * 40), 64


def resolve_chain():
    """Random data at level 1 with a sync flush every 64 bytes, holding two repeats 32000 bytes back, the second of the
    first: with 64-byte chunks every piece is short, so each window spans hundreds of pieces and the second repeat's
    markers resolve through the first repeat's markers, in chain order."""
    r = rand(10, 33000)
    data = r + r[1000:4000] + rand(12, 29000)
    data += data[33000:36000]
    co = zlib.compressobj(1, zlib.DEFLATED, -15)
    out = []
    for k in range(0, len(data), 64):
        out.append(co.compress(data[k:k + 64]))
        out.append(co.flush(zlib.Z_SYNC_FLUSH))
    out.append(co.flush())
    return m.gz(b"".join(out) + m._trailer(data)), 64


def far_two():
    """Two pieces (not the first), each with a copy reaching before the member's start; the error names the smaller
    output byte."""
    w = BitWriter()
    stored_block(w, rand(11, 100), final=0)
    fixed_block(w, [65] * 80 + [(5, 20000)] + [66] * 10, final=0)
    fixed_block(w, [67] * 90 + [(5, 30000)], final=1)
    return member(w, b"?"), 64


def second_member_far():
    """A second member whose first copy reaches 5 bytes before its own start (the first member's bytes are there)."""
    first = gzip.compress(b"0123456789", 6, mtime=0)
    w = BitWriter()
    fixed_block(w, [(5, 5), 65])
    return first + member(w, b"?"), None


CASES = {
    "every_length": every_length, "slow_tail": slow_tail,
    "dist_one_code": dist_one_code, "dist_one_code_bad": lambda: dist_one_code(True),
    "dist_empty": dist_empty, "dist_empty_copy": lambda: dist_empty(True), "cl_empty": cl_empty,
    "long_lengths": long_lengths, "far_32768_from_start": far_32768_from_start, "window_pieces": window_pieces,
    "stored_edges": stored_edges, "stored_past_input": stored_past_input, "stored_padding": stored_padding,
    "fixed_many": fixed_many, "screen_decoys": screen_decoys,
    "overflow_literal": overflow_literal, "overflow_copy": overflow_copy, "overflow_stored": overflow_stored,
    "overflow_then_far": overflow_then_far, "resolve_chain": resolve_chain, "far_two": far_two,
    "second_member_far": second_member_far,
}
RAW = {"slow_tail", "dist_one_code", "dist_one_code_bad"}
WANT = {"dist_one_code_bad": zlib.error, "dist_empty_copy": zlib.error, "cl_empty": zlib.error,
        "stored_past_input": EOFError, "overflow_then_far": zlib.error, "far_two": zlib.error,
        "second_member_far": zlib.error}
CHAIN = ("every_length", "window_pieces", "stored_edges", "stored_padding", "fixed_many", "screen_decoys",
         "overflow_literal", "overflow_copy", "overflow_stored", "overflow_then_far", "resolve_chain", "far_two")


def zlib_result(name, data):
    """What zlib gives: gzip.decompress for a gzip file; for a raw body, zlib.decompressobj(-15)'s bytes and the
    body's bytes it used (an unfinished stream is EOFError, as gunzip raises)."""
    if name not in RAW:
        return m.expect(data)
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(data)
    except zlib.error:
        return zlib.error
    if not d.eof:
        return EOFError
    return out, len(data) - len(d.unused_data)


def model_result(name, data, cb, stats=None):
    try:
        if name in RAW:
            out, end = m.inflate(data, cb or 1 << 15, stats=stats)
            return out, (end + 7) // 8
        return m.gunzip(data, cb or 1 << 15, stats)
    except (EOFError, gzip.BadGzipFile, zlib.error) as e:
        return type(e)


def test_zlib_and_model_agree():
    for name, build in CASES.items():
        data, cb = build()
        want = zlib_result(name, data)
        assert want == WANT.get(name, want) and (name in WANT) == isinstance(want, type), name
        assert model_result(name, data, cb) == want, name


def reach(name):
    data, cb = CASES[name]()
    m.COUNTERS.clear()
    model_result(name, data, cb)
    return dict(m.COUNTERS)


def test_cases_reach_their_paths():
    c = reach("every_length")
    for n in range(1, 16):
        assert c.get(f"lit_len_{n}", 0) and c.get(f"dist_len_{n}", 0), n
    data, _ = slow_tail()
    assert m.inflate(data, 1 << 15)[1] == 8 * len(data)        # the 7-bit end-of-block ends the input: 7 < LIT_FAST
    assert reach("dist_one_code")["dist_one_code"] and reach("dist_one_code_bad")["dist_one_code"]
    data, _ = dist_one_code(True)
    # the bad code is in the last byte: without it the decode runs out of input first
    assert m.run(data, 0, 1 << 30, True, 1 << 20)["status"] == m.DATA
    assert m.run(data[:-1], 0, 1 << 30, True, 1 << 20)["status"] == m.EOF
    assert reach("dist_empty")["dist_empty"] and reach("dist_empty_copy")["dist_empty"]
    assert reach("cl_empty")["cl_empty"]
    c = reach("long_lengths")
    assert c.get("len_285", 0) and c.get("len_284_31", 0)
    assert reach("far_32768_from_start").get("dist_32768", 0)
    c = reach("stored_edges")
    assert c.get("stored_len_0", 0) and c.get("stored_len_65535", 0) and c.get("stored", 0)
    assert reach("overflow_literal")["overflow_literal"]
    assert reach("overflow_copy")["overflow_copy"]
    assert reach("overflow_stored")["overflow_stored"]
    assert reach("overflow_then_far")["overflow_copy"]


def chain_of(name):
    data, cb = CASES[name]()
    st = {}
    if name in RAW:
        m.inflate(data, cb, stats=st)
    else:
        try:
            m.gunzip(data, cb, st)
        except (EOFError, gzip.BadGzipFile, zlib.error):
            pass
    return data, cb, st


def test_window_pieces_layout():
    """A is one piece of 33024 markers, B starts with marker 0, C with the window's last byte, D's last marker lies
    before its walk_lo; every piece but the stored one holds more than 4096 symbols or starts with a marker."""
    data, cb = window_pieces()
    body = data[10:-8]
    st = {}
    m.inflate(body, cb, stats=st)
    pieces = [m.run(body, s, (s // (8 * cb) + 1) * 8 * cb, s == 0, 1 << 20) for s, _ in st["chain"]]
    assert [len(x["syms"]) for x in pieces] == [32768, 33024, 328, 328, 33258]
    a, b, c, d = pieces[1:]
    assert all(s & m.MARK for s in a["syms"]) and a["syms"][len(a["syms"]) - m.WINDOW] & m.MARK
    assert b["syms"][0] == m.MARK | 0 and c["syms"][0] == m.MARK | (m.WINDOW - 1)
    assert d["last_marker"] == 257 and len(d["syms"]) - m.WINDOW > d["last_marker"]


def test_finder_paths():
    data, cb, st = chain_of("fixed_many")
    body = data[10:-8]
    nchunks = -(-len(body) // cb)
    assert nchunks > 30 and all(m.find(body, 8 * cb * k, 8 * cb * (k + 1)) < 0 for k in range(1, nchunks))
    assert st["redecoded"] == len(st["chain"]) - 1
    data, cb = screen_decoys()
    body = data[10:-8]

    def screened(b):                   # k_inflate_run's 13-bit test: BTYPE 10 with HLIT or HDIST above 29
        v = int.from_bytes(body[b >> 3:(b >> 3) + 3], "little") >> (b & 7)
        return (v >> 1) & 3 == 2 and max((v >> 3) & 31, (v >> 8) & 31) > SCREEN_MAX

    decoys = [8 * (5 + 80 + 8 * k) for k in range(5)]          # after the stored header and 80 zero bytes
    assert all(screened(b) and not m.plausible(body, b) for b in decoys)
    valid = 8 * (5 + 80 + 5 * 8)
    assert not screened(valid) and m.plausible(body, valid)
    assert m.find(body, 8 * cb * (valid // (8 * cb)), valid + 1) == valid
    data, cb = stored_padding()
    body = data[10:-8]
    st = {}
    m.inflate(body, cb, stats=st)
    p = st["chain"][-1][0]             # the padded stored block starts the last piece: the walk re-decodes there
    assert len(st["chain"]) == 3 and (body[p >> 3] >> (p & 7)) & 7 == 1 and not m.stored_at(body, p)
    assert st["redecoded"] >= 1


def test_resolve_chain_is_short_pieces():
    data, cb, st = chain_of("resolve_chain")
    assert len(st["chain"]) > 500
    body = data[10:-8]
    tail = [m.run(body, s, (s // (8 * cb) + 1) * 8 * cb, s == 0, 1 << 20)["syms"] for s, _ in st["chain"][-40:]]
    assert max(len(x) for x in tail) < 1024
    assert sum(1 for x in tail for s in x if s & m.MARK) > 1000    # the second repeat: markers into short pieces


def test_far_two_names_the_first():
    data, _ = far_two()
    with pytest.raises(zlib.error, match=r"output byte (\d+)") as e:
        m.gunzip(data, 64)
    assert int(re.search(r"output byte (\d+)", str(e.value)).group(1)) == 100 + 80


# ------------------------------------------------------------------------------------------------ device
def device_result(name, data, cb, cuda, stats=None):
    from gsx import deflate
    from gsx.hostcopy import to_device, to_host
    try:
        if name in RAW:
            out, used = deflate.inflate(to_device(np.frombuffer(data, np.uint8).copy(), cuda), cb, stats)
            return to_host(out).tobytes(), used
        return to_host(deflate.gunzip(data, cuda, cb, stats)).tobytes()
    except (EOFError, gzip.BadGzipFile, zlib.error) as e:
        if stats is not None:
            stats["error"] = str(e)
        return type(e)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_equals_zlib(name, cuda, gsx_lib):
    data, cb = CASES[name]()
    want = zlib_result(name, data)
    for size in {cb, 64, None}:
        assert device_result(name, data, size, cuda) == want, (name, size)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHAIN)
def test_device_chain_equals_model(name, cuda, gsx_lib):
    data, cb = CASES[name]()
    want, got = {}, {}
    model_result(name, data, cb, want)
    device_result(name, data, cb, cuda, got)
    assert got["chain"] == want["chain"], name
    if name == "fixed_many":
        assert got["rounds"] == len(got["chain"]) - 1
    if name.startswith("overflow"):
        assert got["overflow_reruns"] > 0


@pytest.mark.gpu
def test_device_far_error_names_the_first(cuda, gsx_lib):
    data, cb = far_two()
    st = {}
    assert device_result("far_two", data, cb, cuda, st) is zlib.error
    with pytest.raises(zlib.error) as e:
        m.gunzip(data, cb)
    assert re.search(r"output byte \d+", st["error"]).group() == re.search(r"output byte \d+", str(e.value)).group()

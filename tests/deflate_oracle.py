"""NumPy restatement of gsx.deflate's gzip files (csrc/gsx_deflate.cu + gsx/deflate.py), byte for byte, written from
RFC 1951 (DEFLATE) and RFC 1952 (gzip).  The Huffman rule is webp_oracle's.

  * header: CPython's gzip.compress header for (level, mtime); body: below; trailer: CRC-32, n mod 2^32.
  * level 0: stored blocks of 65535 bytes (the last one shorter, final); an empty input is one empty final block.
  * levels 1..9 and -1: blocks cut at every break offset and every 1 MiB inside each span (one empty block for an
    empty input).  Each block is a dynamic block of the cheaper of two token streams (literals on a tie): (a) every
    byte a literal; (b) a maximal run of r >= 4 equal bytes -> one literal, then copies of 258 at distance 1, then one
    copy of the remainder if it is >= 3, else that many literals.  Code lengths: webp_oracle.huffman_lengths with
    limit 15 (literal/length, distance) and 7 (code-length code).  HLIT and HDIST trimmed to the last used symbol (a
    block without copies sends one zero distance length); the HLIT + HDIST lengths run-length coded as one sequence,
    greedy from the left (16: the previous length 3..6 more times, 17: 3..10 zeros, 18: 11..138 zeros); HCLEN
    trimmed in RFC order, at least 4.  The stream is padded to a byte after the final block.
"""
from __future__ import annotations

import struct
import time
import zlib

import numpy as np

import webp_oracle as wo

BLOCK = 1 << 20
STORED = 65535
MAX_COPY = 258
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LEN_BASE = np.array([3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131,
                     163, 195, 227, 258], np.int64)
LEN_EXTRA = np.array([0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0], np.int64)
RLE_EXTRA = {16: 2, 17: 3, 18: 7}


def header(level: int, mtime: int | None) -> bytes:
    if mtime == 0:   # CPython hands mtime 0 to zlib, whose header has OS 3 and XFL by level and strategy
        return struct.pack("<BBBBLBB", 0x1F, 0x8B, 8, 0, 0, 2 if level == 9 else 4 if level in (0, 1) else 0, 3)
    mtime = int(time.time()) if mtime is None else mtime
    return struct.pack("<BBBBLBB", 0x1F, 0x8B, 8, 0, mtime, 2 if level == 9 else 4 if level == 1 else 0, 255)


def block_starts(n: int, breaks=()) -> list:
    if n == 0:
        return [0]
    cuts = sorted({0, n} | {int(b) for b in breaks if 0 < int(b) < n})
    return [s for a, b in zip(cuts, cuts[1:]) for s in range(a, b, BLOCK)]


def length_symbols(lengths: np.ndarray):
    """(symbol 257..285, extra bit count, extra value) of copy lengths 3..258."""
    i = np.searchsorted(LEN_BASE, lengths, side="right") - 1
    return 257 + i, LEN_EXTRA[i], lengths - LEN_BASE[i]


def tokens(x: np.ndarray, copies: bool):
    """(is_copy, literal byte or copy length) of one block, in stream order."""
    if not copies or len(x) == 0:
        return np.zeros(len(x), bool), x.astype(np.int64)
    starts = np.flatnonzero(np.concatenate([[True], x[1:] != x[:-1]]))
    r = np.diff(np.concatenate([starts, [len(x)]]))
    v = x[starts].astype(np.int64)
    full, rem = (r - 1) // MAX_COPY, (r - 1) % MAX_COPY
    long = r >= 4
    ntok = np.where(long, 1 + full + np.where(rem >= 3, 1, rem), r)
    run = np.repeat(np.arange(len(r)), ntok)
    t = np.arange(ntok.sum()) - np.repeat(np.cumsum(ntok) - ntok, ntok)
    lr, fr, rr = long[run], full[run], rem[run]
    is_copy = lr & (t > 0) & ((t <= fr) | ((t == fr + 1) & (rr >= 3)))
    val = np.where(is_copy, np.where(t <= fr, MAX_COPY, rr), v[run])
    return is_copy, val


def rle(seq) -> list:
    """[(symbol, extra value)] of the code-length sequence, greedy from the left."""
    out, i, n = [], 0, len(seq)
    while i < n:
        v, r = seq[i], 1
        while i + r < n and seq[i + r] == v:
            r += 1
        if v == 0:
            c = min(r, 138) if r >= 11 else r if r >= 3 else 1
            out.append((18, c - 11) if c >= 11 else (17, c - 3) if c >= 3 else (0, 0))
            i += c
        else:
            out.append((v, 0))
            i += 1
            rem = r - 1
            while rem >= 3:
                c = min(rem, 6)
                out.append((16, c - 3))
                i += c
                rem -= c
    return out


class Block:
    """One dynamic block's token stream, codes, header fields and bit count."""

    def __init__(self, x: np.ndarray, copies: bool, final: bool):
        self.is_copy, self.val = tokens(x, copies)
        sym = self.val.copy()
        ext_n = np.zeros(len(sym), np.int64)
        ext_v = np.zeros(len(sym), np.int64)
        if self.is_copy.any():
            s, en, ev = length_symbols(self.val[self.is_copy])
            sym[self.is_copy], ext_n[self.is_copy], ext_v[self.is_copy] = s, en, ev
        lit = np.bincount(sym, minlength=286)
        lit[256] += 1
        dist = np.zeros(30, np.int64)
        dist[0] = int(self.is_copy.sum())
        self.lit_len = wo.huffman_lengths(lit, 15)
        self.dist_len = wo.huffman_lengths(dist, 15)
        hlit = max(257, int(np.flatnonzero(self.lit_len).max()) + 1)
        used_d = np.flatnonzero(self.dist_len)
        hdist = int(used_d.max()) + 1 if len(used_d) else 1
        runs = rle(list(self.lit_len[:hlit]) + list(self.dist_len[:hdist]))
        cl_count = np.bincount([s for s, _ in runs], minlength=19)
        cl_len = wo.huffman_lengths(cl_count, 7)
        cl_code = wo.canonical_codes(cl_len)
        hclen = max([4] + [i + 1 for i, s in enumerate(CL_ORDER) if cl_len[s]])
        f = [(int(final), 1), (2, 2), (hlit - 257, 5), (hdist - 1, 5), (hclen - 4, 4)]
        f += [(int(cl_len[s]), 3) for s in CL_ORDER[:hclen]]
        for s, e in runs:
            f.append((int(cl_code[s]), int(cl_len[s])))
            if s in RLE_EXTRA:
                f.append((e, RLE_EXTRA[s]))
        self.head, self.runs = f, runs
        lc, dc = wo.canonical_codes(self.lit_len), wo.canonical_codes(self.dist_len)
        ll, dl = self.lit_len[sym], int(self.dist_len[0])
        vals = lc[sym] | (ext_v << ll) | np.where(self.is_copy, int(dc[0]) << (ll + ext_n), 0)
        cnts = ll + ext_n + np.where(self.is_copy, dl, 0)
        self.vals = np.concatenate([vals, [lc[256]]]).astype(np.int64)
        self.cnts = np.concatenate([cnts, [self.lit_len[256]]]).astype(np.int64)
        self.bits = sum(c for _, c in f) + int(self.cnts.sum())


def pack(vals: np.ndarray, cnts: np.ndarray) -> np.ndarray:
    """uint64 [words] holding the LSB-first bit string of the fields (each < 2^35) in 32-bit words."""
    vals, cnts = np.asarray(vals, np.uint64), np.asarray(cnts, np.int64)
    total = int(cnts.sum())
    pos = (np.cumsum(cnts) - cnts).astype(np.uint64)
    w, sh = (pos >> np.uint64(5)).astype(np.int64), pos & np.uint64(31)
    lo, hi = vals & np.uint64(0xFFFFFFFF), vals >> np.uint64(32)
    a, b = lo << sh, hi << sh                      # a < 2^63, b < 2^34
    m32 = np.uint64(0xFFFFFFFF)
    idx = np.concatenate([w, w + 1, w + 1, w + 2])
    wt = np.concatenate([a & m32, a >> np.uint64(32), b & m32, b >> np.uint64(32)]).astype(np.float64)
    words = np.bincount(idx, weights=wt, minlength=total // 32 + 3)   # disjoint bits: the sum is the OR
    return words.astype(np.uint64)[:(total + 31) // 32]


def join(parts) -> bytes:
    """The bit strings [(words, bits)] one after the other, padded to a byte."""
    total = sum(b for _, b in parts)
    out = np.zeros(total // 32 + 2, np.uint64)
    at = 0
    for words, bits in parts:
        w0, sh = at >> 5, np.uint64(at & 31)
        shifted = words << sh
        out[w0:w0 + len(words)] += shifted & np.uint64(0xFFFFFFFF)
        out[w0 + 1:w0 + 1 + len(words)] += shifted >> np.uint64(32)
        at += bits
    return out.astype("<u4").tobytes()[:(total + 7) // 8]


def body(x: np.ndarray, level: int, breaks=(), info: dict | None = None) -> bytes:
    if level == 0:
        n = len(x)
        out = []
        nb = max(1, -(-n // STORED))
        for k in range(nb):
            c = x[k * STORED:(k + 1) * STORED]
            out.append(struct.pack("<BHH", int(k == nb - 1), len(c), len(c) ^ 0xFFFF) + c.tobytes())
        return b"".join(out)
    starts = block_starts(len(x), breaks)
    ends = starts[1:] + [len(x)]
    parts, chosen = [], []
    for k, (s, e) in enumerate(zip(starts, ends)):
        final = k == len(starts) - 1
        blk = Block(x[s:e], False, final)
        if (x[s + 1:e] == x[s:e - 1]).any():       # a run of two or more: (b) may differ from (a)
            cand = Block(x[s:e], True, final)
            if cand.is_copy.any() and cand.bits < blk.bits:
                blk = cand
        chosen.append(int(blk.is_copy.any()))
        if info is not None:
            info.setdefault("runs", []).append(blk.runs)
            info.setdefault("lit_len", []).append(blk.lit_len)
        vals = np.concatenate([np.array([v for v, _ in blk.head], np.int64), blk.vals])
        cnts = np.concatenate([np.array([c for _, c in blk.head], np.int64), blk.cnts])
        parts.append((pack(vals, cnts), blk.bits))
    if info is not None:
        info["copies"] = chosen
    return join(parts)


def gzip_file(data, level: int, mtime: int | None = 0, breaks=(), info: dict | None = None) -> bytes:
    """The .gz file gsx.deflate.gzip writes for these bytes."""
    x = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data.reshape(-1).view(np.uint8)
    trailer = struct.pack("<II", zlib.crc32(x), len(x) & 0xFFFFFFFF)
    return header(level, mtime) + body(x, level, breaks, info) + trailer


# ------------------------------------------------------------------------------------------------------- cases


def _fib_bytes(count: int, rng) -> np.ndarray:
    """Byte frequencies along a Fibonacci sequence: the unlimited Huffman code is deeper than 15 bits."""
    fib = [1, 1]
    while len(fib) < 24:
        fib.append(fib[-1] + fib[-2])
    x = np.repeat(np.arange(24, dtype=np.uint8) * 7, fib)
    return rng.permutation(np.resize(x, max(count, len(x))))


def _cl_runs(rng) -> np.ndarray:
    """Literals 0..6, 12, 200, 255: equal lengths for 16, a 3..10 zero run for 17, 11..138 and 138+ for 18."""
    vals = np.array([0] * 40 + [1] * 40 + [2] * 40 + [3] * 40 + [4] * 40 + [5] * 40 + [6] * 40 + [12] * 9 + [200] +
                    [255] * 2, np.uint8)
    return rng.permutation(np.tile(vals, 8))


def cases() -> dict:
    """name -> (bytes as uint8 array, breaks)."""
    rng = np.random.default_rng(1951)
    out = {
        "empty": (np.zeros(0, np.uint8), ()),
        "one_byte": (np.array([7], np.uint8), ()),
        "one_distinct_byte": (np.full(5000, 9, np.uint8), ()),
        "flat_256": (np.tile(np.arange(256, dtype=np.uint8), 64), ()),
        "flat_256_shuffled": (rng.permutation(np.tile(np.arange(256, dtype=np.uint8), 64)), ()),
        "fibonacci": (_fib_bytes(200_000, rng), ()),
        "code_length_runs": (_cl_runs(rng), ()),
        "random_small": (rng.integers(0, 256, 3000, dtype=np.uint8), ()),
    }
    for r in (3, 4, 258, 259, 260, 261, 262, 515, 516):
        x = rng.integers(0, 256, 800, dtype=np.uint8)
        x[100:100 + r] = 0xAB
        x[99], x[100 + r] = 0x11, 0x22
        out[f"run_{r}"] = (x, ())
    x = rng.integers(0, 8, 3 * BLOCK // 2, dtype=np.uint8)
    x[BLOCK - 300:BLOCK + 300] = 5
    out["run_across_1mib"] = (x, ())
    x = rng.integers(0, 4, 40_000, dtype=np.uint8)
    x[9_990:10_020] = 3
    out["run_across_break"] = (x, (10_000, 10_002))
    x = rng.integers(0, 256, 5000, dtype=np.uint8)
    x[1000:4000] = 0
    out["breaks_edges_and_repeats"] = (x, (0, 0, 1000, 1000, 1000, 2500, 5000, 5000))
    out["breaks_every_byte"] = (rng.integers(0, 3, 64, dtype=np.uint8), tuple(range(65)))
    sparse = rng.integers(0, 256, 300_000, dtype=np.uint8)
    sparse[rng.random(300_000) < 0.8] = 128
    out["mostly_runs"] = (sparse, (1000, 150_000))
    return out


STORED_SIZES = (0, 1, 65535, 65536, 131070, 131071)

"""gzip files (RFC 1952) on the GPU: writing a device-resident byte buffer (the DEFLATE body, RFC 1951, and CRC-32
computed on the device), and reading any gzip file back into one.

    blob = gzip(payload, level=6)                  # uint8 CUDA tensor -> bytes of a .gz file
    blob = gzip(payload, 6, mtime=0, breaks=(16, 1024))
    data = gunzip(blob)                            # bytes of any .gz file -> uint8 CUDA tensor, as gzip.decompress

Level 0 writes stored blocks of 65535 bytes.  Levels 1..9 and -1 write the same body (csrc/gsx_deflate.cu): the input
is cut at every break offset and every 1 MiB inside each span; each block is a dynamic-Huffman block of literals, or
of literals plus distance-1 copies of runs of equal bytes when that takes fewer bits.  The level only sets the
header's XFL byte.  The file decompresses with any inflater to the input, but its bytes are gsx's, not zlib's.  Only
the finished file comes back to the host.  tests/deflate_oracle.py restates the encoder in NumPy, byte for byte.

gunzip decodes any DEFLATE stream, zlib's included (csrc/gsx_inflate.cu): each member's body is cut into chunks of
compressed bits that are decoded speculatively in parallel, the host walks the chain of block boundaries and
re-decodes where a guess was wrong, and the window each chunk depends on is resolved on the device.  The result and
the exception class (EOFError, gzip.BadGzipFile, zlib.error) are gzip.decompress's.  tests/inflate_model.py restates
the decoder in Python.
"""
from __future__ import annotations

import gzip as _gzip
import struct
import time
import zlib

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

BLOCK = 1 << 20
STORED_BLOCK = 65535


def header(level: int, mtime: int | None = None) -> bytes:
    """The 10 bytes CPython's gzip.compress(data, level, mtime=mtime) starts with: zlib's header when mtime is 0
    (OS 3; XFL 2 at level 9, 4 at levels 0 and 1, else 0), else CPython's own (OS 255; XFL 2 at level 9, 4 at level 1,
    else 0).  mtime None is the current time."""
    level = _level(level)
    if mtime == 0:
        return struct.pack("<BBBBLBB", 0x1F, 0x8B, 8, 0, 0, 2 if level == 9 else 4 if level in (0, 1) else 0, 3)
    mtime = int(time.time()) if mtime is None else int(mtime)
    if not 0 <= mtime < 1 << 32:
        raise ValueError(f"gzip mtime must be 0..2^32-1, not {mtime}")
    return struct.pack("<BBBBLBB", 0x1F, 0x8B, 8, 0, mtime, 2 if level == 9 else 4 if level == 1 else 0, 255)


def _level(level) -> int:
    if isinstance(level, bool) or not isinstance(level, (int, np.integer)) or not -1 <= int(level) <= 9:
        raise ValueError(f"gzip compression level must be an integer in -1..9, not {level!r}")
    return int(level)


def blocks(n: int, breaks=()) -> np.ndarray:
    """int64 starts of the dynamic blocks of n bytes: a cut at every break offset and every 1 MiB inside each span
    between them.  Breaks are ascending and in 0..n (0, n and repeats add no block); n = 0 gives one empty block."""
    b = [int(x) for x in breaks]
    if any(x < 0 or x > n for x in b) or any(y < x for x, y in zip(b, b[1:])):
        raise ValueError(f"breaks must be ascending offsets in 0..{n}")
    if n == 0:
        return np.zeros(1, np.int64)
    cuts = [0] + [x for x in dict.fromkeys(b) if 0 < x < n] + [n]
    return np.concatenate([np.arange(s, e, BLOCK, dtype=np.int64) for s, e in zip(cuts, cuts[1:])])


def _check(data) -> torch.Tensor:
    if not isinstance(data, torch.Tensor) or not data.is_cuda:
        raise ValueError("gzip needs a CUDA tensor")
    if data.dtype != torch.uint8:
        raise ValueError(f"gzip needs uint8 data, not {data.dtype}")
    return data.contiguous().reshape(-1)


def gzip(data: torch.Tensor, level: int, mtime: int | None = None, breaks=()) -> bytes:
    """The bytes of a .gz file of `data` (uint8 CUDA tensor, read in memory order) at compression `level` (-1..9, else
    ValueError).  The header is CPython's for (level, mtime); the body is stored blocks at level 0, else dynamic blocks
    cut at `breaks` (ascending offsets, see blocks()) and every 1 MiB; the trailer is CRC-32 and the size mod 2^32."""
    level = _level(level)
    data = _check(data)
    head = np.frombuffer(header(level, mtime), np.uint8)
    n, dev = data.numel(), data.device
    from .hostcopy import to_bytes, to_device
    with torch.cuda.device(dev):
        stream = _stream()
        if level == 0:
            starts = None
            ws = torch.empty(lib.gsx_deflate_workspace_bytes(0), dtype=torch.uint8, device=dev)
            body = 5 * max(1, -(-n // STORED_BLOCK)) + n
        else:
            starts = to_device(blocks(n, breaks), dev)
            ws = torch.empty(lib.gsx_deflate_workspace_bytes(len(starts)), dtype=torch.uint8, device=dev)
            counts = torch.zeros(2, dtype=torch.int64, device=dev)   # body bits, blocks emitted off their plan
            check(lib.gsx_deflate_plan(_ptr(data), n, _ptr(starts), len(starts), _ptr(ws), ws.numel(), 80,
                                       _ptr(counts), stream), "gsx_deflate_plan")
            body = (int(counts[0].item()) + 7) // 8
        file_bytes = 10 + body + 8
        words = torch.zeros((file_bytes + 3) // 4, dtype=torch.int32, device=dev)
        out = words.view(torch.uint8)
        out[:10].copy_(to_device(head, dev))
        if level == 0:
            check(lib.gsx_deflate_stored(_ptr(data), n, _ptr(out[10:]), stream), "gsx_deflate_stored")
        else:
            check(lib.gsx_deflate_emit(_ptr(data), n, _ptr(starts), len(starts), _ptr(ws), ws.numel(), _ptr(words),
                                       words.numel(), _ptr(counts[1:]), stream), "gsx_deflate_emit")
        check(lib.gsx_crc32(_ptr(data), n, _ptr(ws), ws.numel(), _ptr(out[10 + body:]), stream), "gsx_crc32")
        blob = to_bytes(out[:file_bytes])
        if level != 0 and int(counts[1].item()):
            raise RuntimeError(f"gsx_deflate_emit: {int(counts[1].item())} blocks differ from their plan")
    return blob


# ----------------------------------------------------------------------------------------------------- reading gzip
WINDOW = 32768
OK, FINAL, EOF, DATA, OVERFLOW, NONE, BAD_JOB = range(7)
FIND, FIRST = 1, 2
RATIO = 4                    # first capacity of a chunk, in symbols per compressed byte


def _chunk_bytes(n: int) -> int:
    """About 8192 chunks of at least 32 KiB: enough threads to fill the GPU, few enough window steps."""
    return int(min(max(n // 8192, 1 << 15), 1 << 22))


def _grow(r: np.ndarray, job: np.ndarray) -> int:
    """A larger capacity for a job that overflowed: its output so far, scaled to the bits it has left, and at least
    twice the old capacity."""
    start, done = r[0], max(r[5] - r[0], 1)
    return int(max(2 * job[4], job[4] * (max(job[2] - start, done) / done) * 1.25 + 1024))


def _decode(body: torch.Tensor, jobs: np.ndarray, st: dict) -> list:
    """Run `jobs` (int64 [m, 6], see gsx_inflate_run) on the device, re-running every job that overflowed its
    capacity with more, all of them in one launch per round.  -> per job (result row, symbol address, workspace); a
    workspace lives as long as a result that points into it."""
    from .hostcopy import to_device, to_host
    jobs = np.array(jobs, np.int64)
    out, todo, dev = [None] * len(jobs), np.arange(len(jobs)), body.device
    while len(todo):
        J = jobs[todo]
        J[:, 3] = np.concatenate([[0], np.cumsum(J[:-1, 4])])
        ws = torch.empty(lib.gsx_inflate_workspace_bytes(int(J[:, 4].sum())), dtype=torch.uint8, device=dev)
        res = torch.empty((len(J), 6), dtype=torch.int64, device=dev)
        check(lib.gsx_inflate_run(_ptr(body), body.numel(), _ptr(to_device(J, dev)), len(J), _ptr(ws), ws.numel(),
                                  _ptr(res), _stream()), "gsx_inflate_run")
        res = to_host(res)
        over = res[:, 4] == OVERFLOW
        for i in np.flatnonzero(~over):
            out[todo[i]] = (res[i], ws.data_ptr() + 2 * int(J[i, 3]), ws)
        for i in np.flatnonzero(over):
            t = todo[i]
            jobs[t, 4] = _grow(res[i], jobs[t])
            jobs[t, 0] = res[i, 0]
            jobs[t, 5] &= FIRST
        todo = todo[over]
        st["overflow_reruns"] += len(todo)
    return out


def inflate(body: torch.Tensor, chunk_bytes: int | None = None, stats: dict | None = None):
    """The raw DEFLATE stream (zlib wbits -15) at the start of `body` (uint8 CUDA tensor) -> (uint8 CUDA tensor of
    its bytes, bytes of `body` it used).  zlib.error for an invalid stream, EOFError when `body` ends first.
    chunk_bytes sets the chunks' size (tests use it to force many chunks); the result does not depend on it.
    stats, when given, gains the counts of chunks, false starts (a chunk whose found start is not where the chain
    reached it), re-decoded jobs, re-decode rounds and overflow re-runs, and the chain's (start, stop) bits."""
    body = _check(body)
    n, dev = body.numel(), body.device
    cb = 8 * int(chunk_bytes or _chunk_bytes(n))
    nchunks = max(1, -(-8 * n // cb))
    cap0 = RATIO * cb // 8
    st = dict(chunks=nchunks, false_starts=0, redecoded=0, rounds=0, overflow_reruns=0)
    with torch.cuda.device(dev):
        c = np.arange(nchunks, dtype=np.int64)
        jobs = np.stack([c * cb, (c + 1) * cb, (c + 1) * cb, c, np.full(nchunks, cap0), np.full(nchunks, FIND)], 1)
        jobs[0, 5] = FIRST
        found = {}                      # start bit -> (result, symbol address, workspace)
        for x in _decode(body, jobs, st):
            if x[0][4] != NONE:
                found[int(x[0][0])] = x
        chain, p = [], 0
        while True:
            if p not in found:
                # One round: decode from p and, in the same launch, from every other stop not yet decoded past p --
                # a chunk after a false start needs its predecessor's stop, which is known only now.
                k = p // cb
                st["false_starts"] += int(k < nchunks and any(s // cb == k for s in found))
                want = sorted({p} | {int(x[0][1]) for x in found.values()
                                     if x[0][4] == OK and x[0][1] > p and int(x[0][1]) not in found})
                q = np.array(want, np.int64)
                jobs = np.stack([q, q, (q // cb + 1) * cb, np.zeros_like(q), np.full(len(q), cap0),
                                 np.where(q == 0, FIRST, 0)], 1)
                for s, x in zip(want, _decode(body, jobs, st)):
                    found[s] = x
                st["redecoded"] += len(want)
                st["rounds"] += 1
            x = found[p]
            if x[0][4] == BAD_JOB:
                raise RuntimeError(f"gsx_inflate_run: job at bit {p} outside the input or workspace")
            chain.append(x)
            if x[0][4] != OK:
                break
            p = int(x[0][1])
        found.clear()
        st["chain"] = [(int(r[0]), int(r[1])) for r, _, _ in chain]
        if stats is not None:
            for key, v in st.items():
                stats[key] = stats.get(key, 0) + v if key != "chain" else stats.get(key, []) + v
        last = chain[-1][0]
        if last[4] == DATA:
            raise zlib.error(f"invalid deflate stream (bit {int(last[5])})")
        counts = np.array([r[2] for r, _, _ in chain], np.int64)
        offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
        lo = np.maximum(counts - WINDOW, 0)
        lastm = np.array([r[3] for r, _, _ in chain], np.int64)
        walk = lastm >= lo
        pieces = np.stack([np.array([q for _, q, _ in chain], np.int64), counts, offs, np.where(walk, lo, counts),
                           np.where(walk, lastm + 1, counts)], 1)
        out = torch.empty(int(counts.sum()), dtype=torch.uint8, device=dev)
        status = torch.full((1,), -1, dtype=torch.int64, device=dev)
        from .hostcopy import to_device
        check(lib.gsx_inflate_resolve(_ptr(to_device(pieces, dev)), len(pieces), _ptr(out), _ptr(status), _stream()),
              "gsx_inflate_resolve")
        far = int(status.item())
        chain.clear()
    if far != -1:
        raise zlib.error(f"invalid distance too far back (output byte {far})")
    if last[4] == EOF:
        raise EOFError("Compressed file ended before the end-of-stream marker was reached")
    return out, (int(last[1]) + 7) // 8


class _File:
    """The bytes of a .gz file: the device copy is decoded, the headers and trailers are read on the host (from the
    caller's bytes, or a few small copies from the device)."""

    def __init__(self, data, device):
        if isinstance(data, torch.Tensor):
            self.dev, self.host = _check(data), None
            self.n = self.dev.numel()
            return
        self.host = memoryview(data).cast("B")
        self.n = len(self.host)
        if device is not None:
            from .hostcopy import to_device
            self.dev = to_device(np.frombuffer(self.host, np.uint8), device)

    def read(self, lo: int, hi: int) -> bytes:
        lo, hi = min(lo, self.n), min(hi, self.n)
        if self.host is not None:
            return bytes(self.host[lo:hi])
        from .hostcopy import to_host
        return to_host(self.dev[lo:hi]).tobytes() if hi > lo else b""

    def find(self, pos: int, zero: bool) -> int:
        """First offset >= pos whose byte is (zero) / is not (not zero) 0, else the file's length."""
        step = 4096
        while pos < self.n:
            b = np.frombuffer(self.read(pos, pos + step), np.uint8)
            hit = np.flatnonzero(b == 0 if zero else b != 0)
            if len(hit):
                return pos + int(hit[0])
            pos, step = pos + len(b), min(step * 4, 1 << 24)
        return self.n


def _eof():
    return EOFError("Compressed file ended before the end-of-stream marker was reached")


def _header_end(f: _File, pos: int):
    """CPython's gzip._read_gzip_header at `pos`: None at the end of the file, else the offset of the DEFLATE body.
    Reserved flag bits are ignored and FHCRC is skipped unchecked, as CPython does."""
    if pos >= f.n:
        return None
    head = f.read(pos, pos + 10)
    if head[:2] != b"\x1f\x8b":
        raise _gzip.BadGzipFile(f"Not a gzipped file ({head[:2]!r})")
    if len(head) < 10:
        raise _eof()
    method, flag = head[2], head[3]
    if method != 8:
        raise _gzip.BadGzipFile("Unknown compression method")
    pos += 10
    if flag & 4:
        xlen = f.read(pos, pos + 2)
        if len(xlen) < 2 or f.n - pos - 2 < struct.unpack("<H", xlen)[0]:
            raise _eof()
        pos += 2 + struct.unpack("<H", xlen)[0]
    for bit in (8, 16):
        if flag & bit:
            pos = min(f.find(pos, True) + 1, f.n)
    if flag & 2:
        if f.n - pos < 2:
            raise _eof()
        pos += 2
    return pos


def first_block_stored(data) -> bool:
    """Whether the first member of the gzip file `data` (bytes-like) starts with a stored block, as zlib's level 0
    writes it; False when its header does not parse.  Stored data is copied, not decoded, and zlib on one host thread
    outpaces gunzip there (DESIGN section 10), so readers choose by this."""
    f = _File(data, None)
    try:
        h = _header_end(f, 0)
    except (EOFError, _gzip.BadGzipFile):
        return False
    return h is not None and h < f.n and (f.host[h] >> 1) & 3 == 0


def gunzip(data, device="cuda", chunk_bytes: int | None = None, stats: dict | None = None) -> torch.Tensor:
    """gzip.decompress(data) on the device: `data` is a bytes-like object (uploaded once) or a uint8 CUDA tensor; the
    result is a uint8 CUDA tensor, or the exception gzip.decompress raises (EOFError, gzip.BadGzipFile, zlib.error).
    Members follow each other with any zero bytes between them.  chunk_bytes sets the decoder's chunk size (tests use
    it to force many chunks); the result does not depend on it.  stats, when given, gains inflate()'s counts summed
    over the members, and their chains.
    """
    f = _File(data, device)
    dev = f.dev.device
    members, pos = [], 0
    with torch.cuda.device(dev):
        ws = None
        while True:
            h = _header_end(f, pos)
            if h is None:
                break
            out, used = inflate(f.dev[h:], chunk_bytes, stats)
            t = h + used
            trailer = f.read(t, t + 8)
            if len(trailer) < 8:
                raise _eof()
            if ws is None:
                ws = torch.empty(lib.gsx_deflate_workspace_bytes(0), dtype=torch.uint8, device=dev)
            mine = torch.empty(8, dtype=torch.uint8, device=dev)
            check(lib.gsx_crc32(_ptr(out), out.numel(), _ptr(ws), ws.numel(), _ptr(mine), _stream()), "gsx_crc32")
            from .hostcopy import to_host
            mine = to_host(mine).tobytes()
            if mine[:4] != trailer[:4]:
                raise _gzip.BadGzipFile("CRC check failed")
            if mine[4:] != trailer[4:]:
                raise _gzip.BadGzipFile("Incorrect length of data produced")
            members.append(out)
            pos = f.find(t + 8, False)
    if not members:
        return torch.empty(0, dtype=torch.uint8, device=dev)
    return members[0] if len(members) == 1 else torch.cat(members)

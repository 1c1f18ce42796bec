"""gzip files (RFC 1952) of a device-resident byte buffer, the DEFLATE body (RFC 1951) and CRC-32 computed on the GPU.

    blob = gzip(payload, level=6)                  # uint8 CUDA tensor -> bytes of a .gz file
    blob = gzip(payload, 6, mtime=0, breaks=(16, 1024))

Level 0 writes stored blocks of 65535 bytes.  Levels 1..9 and -1 write the same body (csrc/gsx_deflate.cu): the input
is cut at every break offset and every 1 MiB inside each span; each block is a dynamic-Huffman block of literals, or
of literals plus distance-1 copies of runs of equal bytes when that takes fewer bits.  The level only sets the
header's XFL byte.  The file decompresses with any inflater to the input, but its bytes are gsx's, not zlib's.  Only
the finished file comes back to the host.  tests/deflate_oracle.py restates the encoder in NumPy, byte for byte.
"""
from __future__ import annotations

import struct
import time

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

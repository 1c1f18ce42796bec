"""Lossless WebP (VP8L, RFC 9649) encoding of a device-resident RGBA image.

    data = encode_lossless(pixels, width, height)   # uint8 CUDA [height * width, 4] -> bytes of a RIFF WEBP file

The device (csrc/gsx_webp.cu) clears RGB where alpha is 0, builds three candidates -- the pixels, predictor residuals
on 16x16 tiles, subtract-green then predictor residuals -- with run copies of the left pixel, and their histograms.
This module copies the histograms back (a few KB), builds length-limited Huffman codes, keeps the candidate with the
fewest bits, and has the device emit the chosen image's bits behind the headers written here.  Only the finished file
comes back to the host.  No colour cache, no meta prefix image, one Huffman group; the bytes are not libwebp's.
tests/webp_oracle.py restates the encoder in NumPy, byte for byte.
"""
from __future__ import annotations

import heapq

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

MAX_SIDE = 16384
TILE_BITS = 4
ALPHABETS = (280, 256, 256, 256, 40)               # green + 24 length codes, red, blue, alpha, distance
OFFSETS = (0, 280, 536, 792, 1048)
TREE_SYMS = 1088
CL_ORDER = (17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
RIFF_BITS = 160                                     # "RIFF" size "WEBP" "VP8L" chunk-size


def _length_extra_bits(code: int) -> int:
    return 0 if code < 4 else (code - 2) >> 1


def code_lengths(counts, limit: int) -> list:
    """Huffman code lengths of `counts`, none above `limit`: repeatedly join the two lightest nodes by (weight, id)
    (leaf id = symbol, the k-th joined node = len(counts) + k); while a length exceeds `limit`, raise every used
    weight to a floor of 1, 2, 4, ...  A lone used symbol gets length 1."""
    used = [s for s, c in enumerate(counts) if c]
    lengths = [0] * len(counts)
    if len(used) == 1:
        lengths[used[0]] = 1
        return lengths
    floor = 1
    while len(used) > 1:
        heap = [(max(int(counts[s]), floor), s, (s,)) for s in used]
        heapq.heapify(heap)
        nid = len(counts)
        depth = {s: 0 for s in used}
        while len(heap) > 1:
            wa, _, la = heapq.heappop(heap)
            wb, _, lb = heapq.heappop(heap)
            for s in la + lb:
                depth[s] += 1
            heapq.heappush(heap, (wa + wb, nid, la + lb))
            nid += 1
        if max(depth.values()) <= limit:
            for s, d in depth.items():
                lengths[s] = d
            return lengths
        floor *= 2
    return lengths


def reversed_codes(lengths) -> list:
    """Canonical codes (shorter first, then by symbol), each bit-reversed for the LSB-first stream."""
    codes = [0] * len(lengths)
    nxt = 0
    for ln in range(1, max(lengths, default=0) + 1):
        for s, l in enumerate(lengths):
            if l == ln:
                codes[s] = int(bin(nxt)[2:].zfill(ln)[::-1], 2)
                nxt += 1
        nxt <<= 1
    return codes


class BitWriter:
    """LSB-first bits held in one Python integer."""

    def __init__(self):
        self.value, self.size = 0, 0

    def put(self, v: int, n: int):
        self.value |= int(v) << self.size
        self.size += n

    def extend(self, other: "BitWriter"):
        self.put(other.value, other.size)


class Tree:
    """One prefix code: its description in the stream and the per-symbol (reversed code, bits) it emits."""

    def __init__(self, counts):
        counts = [int(c) for c in counts]
        used = [s for s, c in enumerate(counts) if c]
        self.desc = BitWriter()
        self.lengths = [0] * len(counts)
        self.codes = [0] * len(counts)
        if len(used) <= 2 and all(s < 256 for s in used):
            self._simple(used or [0])
        else:
            self._normal(counts)

    def _simple(self, syms):
        d = self.desc
        d.put(1, 1)
        d.put(len(syms) - 1, 1)
        wide = syms[0] > 1
        d.put(int(wide), 1)
        d.put(syms[0], 8 if wide else 1)
        if len(syms) == 2:
            d.put(syms[1], 8)
            self.lengths[syms[0]] = self.lengths[syms[1]] = 1
            self.codes[syms[1]] = 1

    def _normal(self, counts):
        d = self.desc
        self.lengths = code_lengths(counts, 15)
        self.codes = reversed_codes(self.lengths)
        cl_counts = [0] * 19
        for ln in self.lengths:
            cl_counts[ln] += 1
        cl_len = code_lengths(cl_counts, 7)
        cl_code = reversed_codes(cl_len)
        ncodes = 4
        for i, s in enumerate(CL_ORDER):
            if cl_len[s]:
                ncodes = max(ncodes, i + 1)
        d.put(0, 1)
        d.put(ncodes - 4, 4)
        for s in CL_ORDER[:ncodes]:
            d.put(cl_len[s], 3)
        d.put(0, 1)                                 # no max_symbol: every symbol of the alphabet is described
        lone = sum(1 for x in cl_len if x) == 1     # a single code-length symbol is read with 0 bits
        for ln in self.lengths:
            d.put(cl_code[ln], 0 if lone else cl_len[ln])

    def data_bits(self, counts) -> int:
        return sum(int(c) * l for c, l in zip(counts, self.lengths))

    def table(self) -> np.ndarray:
        return np.array([c | (l << 16) for c, l in zip(self.codes, self.lengths)], np.uint32)


class Coded:
    """The five trees of one entropy-coded image, from its histogram row."""

    def __init__(self, hist):
        self.parts = [hist[o:o + a] for o, a in zip(OFFSETS, ALPHABETS)]
        self.trees = [Tree(p) for p in self.parts]
        green = self.parts[0]
        self.data_bits = (sum(t.data_bits(p) for t, p in zip(self.trees, self.parts))
                          + sum(int(green[256 + c]) * _length_extra_bits(c) for c in range(24)))

    def write_codes(self, w: BitWriter, main: bool):
        w.put(0, 1)                                 # no colour cache
        if main:
            w.put(0, 1)                             # no meta prefix image
        for t in self.trees:
            w.extend(t.desc)

    def table(self) -> np.ndarray:
        return np.concatenate([t.table() for t in self.trees])


def _check(pixels, width, height):
    if not isinstance(pixels, torch.Tensor) or not pixels.is_cuda:
        raise ValueError("encode_lossless needs a CUDA tensor")
    if pixels.dtype != torch.uint8:
        raise ValueError(f"encode_lossless needs uint8 pixels, not {pixels.dtype}")
    width, height = int(width), int(height)
    if not (1 <= width <= MAX_SIDE and 1 <= height <= MAX_SIDE):
        raise ValueError(f"WebP images are 1..{MAX_SIDE} pixels on a side, not {width} x {height}")
    if tuple(pixels.shape) not in ((width * height, 4), (height, width, 4)):
        raise ValueError(f"pixels of shape {tuple(pixels.shape)} are not a {width} x {height} RGBA image")
    return pixels.contiguous(), width, height


def _patches(w: BitWriter, bit_offset: int) -> np.ndarray:
    """(word index, bits) pairs that OR the writer's bits in at bit_offset."""
    v = w.value << (bit_offset & 31)
    nwords = (w.size + (bit_offset & 31) + 31) // 32
    first = bit_offset >> 5
    return np.array([(first + k, (v >> (32 * k)) & 0xFFFFFFFF) for k in range(nwords)], np.uint32).reshape(-1, 2)


def encode_lossless(pixels: torch.Tensor, width: int, height: int, info: dict | None = None) -> bytes:
    """The bytes of a lossless RIFF WEBP/VP8L file of the RGBA image `pixels` (uint8 CUDA [height * width, 4] or
    [height, width, 4]).  Raises ValueError, before any launch, for a side outside 1..16384, a dtype other than uint8,
    a tensor off the GPU or a shape that does not match.  info, if a dict, receives 'candidate' (0 = no transform,
    1 = predictor, 2 = subtract-green + predictor), 'bits' (the file's VP8L bits per candidate) and 'modes' (the
    chosen candidate's tile modes, uint8 [tiles_y, tiles_x], or None)."""
    pixels, width, height = _check(pixels, width, height)
    dev = pixels.device
    tiles_x, tiles_y = -(-width >> TILE_BITS), -(-height >> TILE_BITS)
    ws = torch.empty(lib.gsx_webp_workspace_bytes(width, height), dtype=torch.uint8, device=dev)
    hist = torch.empty(5 * TREE_SYMS + 1, dtype=torch.int32, device=dev)
    modes = torch.empty(2 * tiles_x * tiles_y, dtype=torch.uint8, device=dev) if info is not None else None
    stream = _stream()
    check(lib.gsx_webp_analyze(_ptr(pixels), width, height, _ptr(ws), ws.numel(), _ptr(hist), _ptr(modes), stream),
          "gsx_webp_analyze")
    h = hist.cpu().numpy().view(np.uint32)
    images = [Coded(h[k * TREE_SYMS:(k + 1) * TREE_SYMS]) for k in range(5)]
    alpha_used = int(h[5 * TREE_SYMS] != 0)

    def headers(cand):
        """(the bits before the sub-image's data, the bits between it and the main data, sub-image or None)."""
        a = BitWriter()
        a.put(0x2F, 8)
        a.put(width - 1, 14)
        a.put(height - 1, 14)
        a.put(alpha_used, 1)
        a.put(0, 3)
        sub = None
        if cand:
            if cand == 2:
                a.put(1, 1)
                a.put(2, 2)                         # subtract-green
            a.put(1, 1)
            a.put(0, 2)                             # predictor
            a.put(TILE_BITS - 2, 3)
            sub = images[cand + 2]
            sub.write_codes(a, main=False)
        b = BitWriter()
        b.put(0, 1)                                 # no further transform
        images[cand].write_codes(b, main=True)
        return a, b, sub

    sizes = []
    for cand in range(3):
        a, b, sub = headers(cand)
        sizes.append(a.size + (sub.data_bits if sub else 0) + b.size + images[cand].data_bits)
    cand = int(np.argmin(sizes))
    a, b, sub = headers(cand)
    vp8l_bits = sizes[cand]
    payload = (vp8l_bits + 7) // 8
    file_bytes = 20 + payload + (payload & 1)
    riff = BitWriter()
    for word in (b"RIFF", (file_bytes - 8).to_bytes(4, "little"), b"WEBP", b"VP8L", payload.to_bytes(4, "little")):
        riff.put(int.from_bytes(word, "little"), 32)
    riff.extend(a)
    sub_at = riff.size
    main_at = sub_at + (sub.data_bits if sub else 0) + b.size
    nwords = (8 * file_bytes + 31) // 32
    words = torch.zeros(nwords, dtype=torch.int32, device=dev)
    totals = torch.zeros(2, dtype=torch.int64, device=dev)
    tables = []
    for k, (img, at) in enumerate(((cand + 2, sub_at), (cand, main_at))):
        if k == 0 and sub is None:
            continue
        table = torch.from_numpy(images[img].table().view(np.int32)).to(dev)
        tables.append(table)
        check(lib.gsx_webp_emit(width, height, img, _ptr(table), at, _ptr(ws), ws.numel(), _ptr(words), nwords,
                                _ptr(totals[k:]), stream), "gsx_webp_emit")
    patches = np.concatenate([_patches(riff, 0), _patches(b, main_at - b.size)])
    patches_t = torch.from_numpy(patches.view(np.int32)).to(dev)
    check(lib.gsx_webp_patch(_ptr(words), nwords, _ptr(patches_t), len(patches), stream), "gsx_webp_patch")
    got = totals.cpu().tolist()
    want = [sub.data_bits if sub else 0, images[cand].data_bits]
    if got != want:
        raise RuntimeError(f"gsx_webp_emit wrote {got} data bits where the histograms give {want}")
    if info is not None:
        m = modes.cpu().numpy().reshape(2, tiles_y, tiles_x)
        info.update(candidate=cand, bits=sizes, modes=m[cand - 1] if cand else None)
    return words.cpu().numpy().view(np.uint8)[:file_bytes].tobytes()

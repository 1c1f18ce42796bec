"""Lossless WebP (VP8L, RFC 9649) decoding on the device.

    rgba = decode_lossless(data)        # bytes of a RIFF WEBP file -> uint8 CUDA [height, width, 4]

The pixels are what Pillow's Image.open(...).convert('RGBA') gives: a file whose VP8L header's alpha hint is 0 reads
with alpha 255 whatever the stream holds (a VP8X header's alpha flag does not matter).  csrc/gsx_vp8l.cu does the work:

- One thread parses the header, transforms, sub-images and prefix codes; a few values come back.
- The main image's bits are cut into chunks and each is decoded speculatively into tokens (a literal, a copy or a
  colour-cache index), at a pixel position guessed from its bit offset; the position only picks the prefix-code group.
- The host walks the chain of pieces by bits: a piece stands when it starts where the previous one stopped and, if
  it was decoded at another position than the chain gives it, every token's group is the one at its true position.
  Each round re-decodes, at the position the chain gives it, every piece that does not stand, and decodes from the
  stop where the chain breaks; after max_rounds the rest is decoded by one job from the verified frontier.
- The tokens become pixels: without a colour cache by pointer jumping over the copies' source pixels, with one by a
  replay in pixel order; then the inverse transforms, the predictor as a wavefront.

tests/vp8l_model.py restates all of it in Python.  Anything the decoder refuses raises ValueError.
"""
from __future__ import annotations

import numpy as np
import torch

from ._abi import lib, check
from ._abi import _ptr, _stream

JOB_OK, JOB_END, JOB_EOF, JOB_OVERFLOW = 0, 1, 2, 4
_HEADER_ERRORS = {1: "truncated stream", 2: "invalid prefix code or sub-image", 3: "invalid header field"}
_SPACE = 4
TOKEN_BYTES = 16
MAX_ROUNDS = 8


def container(data):
    """(offset, length of the VP8L payload, whether Pillow opens the file with alpha) of a RIFF WEBP file whose
    image is one VP8L chunk, alone or after a VP8X chunk; None for anything else (lossy, ALPH, animation), which
    Pillow decodes."""
    mv = memoryview(data).cast("B")
    if len(mv) < 20 or bytes(mv[:4]) != b"RIFF" or bytes(mv[8:12]) != b"WEBP":
        return None
    pos, vp8x_alpha = 12, None
    while pos + 8 <= len(mv):
        tag, size = bytes(mv[pos:pos + 4]), int.from_bytes(mv[pos + 4:pos + 8], "little")
        if tag == b"VP8X":
            if pos != 12 or size < 10 or pos + 9 > len(mv) or mv[pos + 8] & 0x02:
                return None
            vp8x_alpha = bool(mv[pos + 8] & 0x10)
        elif tag == b"VP8L":
            size = min(size, len(mv) - pos - 8)
            if size < 5:
                raise ValueError("VP8L: truncated header")
            hint = bool((mv[pos + 12] >> 4) & 1)
            return pos + 8, size, hint     # Pillow follows the VP8L header's alpha hint, whatever VP8X says
        elif vp8x_alpha is None or tag in (b"VP8 ", b"ALPH", b"ANIM", b"ANMF"):
            return None
        pos += 8 + size + (size & 1)
    return None


class _Header:
    def __init__(self, body: torch.Tensor, head: bytes):
        if len(head) < 5 or head[0] != 0x2F:
            raise ValueError("VP8L: no 0x2f signature")
        bits = int.from_bytes(head[1:5], "little")
        width, height = (bits & 0x3FFF) + 1, ((bits >> 14) & 0x3FFF) + 1
        dev, groups = body.device, 8
        self.lens = torch.empty(2328, dtype=torch.uint8, device=dev)
        info_t = torch.empty(32, dtype=torch.int64, device=dev)
        from .hostcopy import to_host
        while True:
            words = lib.gsx_vp8l_header_words(width, height, groups)
            self.ws = torch.empty(words, dtype=torch.int32, device=dev)
            check(lib.gsx_vp8l_header(_ptr(body), body.numel(), _ptr(self.ws), words, _ptr(self.lens), _ptr(info_t),
                                      _stream()), "gsx_vp8l_header")
            info = [int(v) for v in to_host(info_t)]
            if info[0] != _SPACE:
                break
            per_group = lib.gsx_vp8l_header_words(width, height, 2) - lib.gsx_vp8l_header_words(width, height, 1)
            groups = -(-(info[29] - lib.gsx_vp8l_header_words(width, height, 1)) // per_group) + 1
            if groups > 65536 or lib.gsx_vp8l_header_words(width, height, groups) == 0:
                raise ValueError("VP8L: the prefix-code groups overflow the workspace")
        if info[0]:
            raise ValueError(f"VP8L: {_HEADER_ERRORS.get(info[0], 'invalid stream')} (bit {info[1]})")
        self.width, self.height, self.alpha_hint, self.xsize = info[2], info[3], info[4], info[5]
        self.cache_bits, self.meta_bits, self.groups = info[6], info[7], info[8]
        self.entropy_off, self.codes_off, self.main_bit = info[9], info[10], info[11]
        self.transforms = [tuple(info[13 + 4 * t:17 + 4 * t]) for t in range(info[12])]
        self.npix = self.xsize * self.height

    def codes(self):
        return self.ws[self.codes_off:]

    def entropy(self):
        return self.ws[self.entropy_off:] if self.entropy_off >= 0 else None

    def image_args(self):
        return (_ptr(self.codes()), _ptr(self.entropy()), self.xsize, self.height, self.meta_bits)


def _chunk_bits(nbits: int) -> int:
    """About 8192 chunks of at least 16 Kibit.  Smaller chunks cost more rounds than they save: at 65536 chunks of
    1 Kibit a chunk often ends before its decode falls into step with the true token boundaries, and the host's walk
    over the pieces outweighs the kernels (DESIGN section 10)."""
    return int(max(nbits // 8192, 1 << 14))


def _run(body, h: _Header, jobs: list, st: dict) -> list:
    """jobs: (start, target, guess, capacity) -> per job (start, stop, tokens, pixels, status, guess, token address,
    token tensor); overflowed jobs re-run with 8 times the capacity, at most the image's pixels."""
    from .hostcopy import to_device, to_host
    out, todo = [None] * len(jobs), list(range(len(jobs)))
    jobs = [list(j) for j in jobs]
    dev = body.device
    while todo:
        caps = np.array([jobs[i][3] for i in todo], np.int64)
        offs = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
        J = np.array([[jobs[i][0], jobs[i][1], jobs[i][2], o, c] for i, o, c in zip(todo, offs, caps)], np.int64)
        toks = torch.empty((int(caps.sum()), 4), dtype=torch.int32, device=dev)
        res = torch.empty((len(J), 6), dtype=torch.int64, device=dev)
        check(lib.gsx_vp8l_run(_ptr(body), body.numel(), *h.image_args(), _ptr(to_device(J, dev)), len(J), _ptr(toks),
                               _ptr(res), _stream()), "gsx_vp8l_run")
        res = to_host(res)
        again = []
        for k, i in enumerate(todo):
            r = res[k]
            if r[4] == JOB_OVERFLOW:
                jobs[i][3] = min(8 * jobs[i][3], max(h.npix, 1))
                again.append(i)
                st["overflow_reruns"] += 1
                continue
            out[i] = (int(r[0]), int(r[1]), int(r[2]), int(r[3]), int(r[4]), int(J[k, 2]),
                      toks.data_ptr() + TOKEN_BYTES * int(offs[k]), toks)
        todo = again
    return out


def _main_tokens(body, h: _Header, chunk_bits, max_rounds, st) -> list:
    """The chain of pieces of the main image, each (start, stop, tokens, pixels, status, guess, address, tensor) with
    its true first pixel appended."""
    from .hostcopy import to_device, to_host
    nbits = 8 * body.numel() - h.main_bit
    cb = int(chunk_bits or _chunk_bits(nbits))
    nchunks = max(1, -(-nbits // cb))
    # tokens never outnumber pixels: a chunk's share of the pixels, and an overflow re-run for the chunks with more
    cap = int(min(cb + 64, h.npix // nchunks + 256))
    st.update(chunks=nchunks, false_starts=0, group_mismatches=0, moved_refused=0, rounds=0, serial_fallbacks=0,
              overflow_reruns=0)

    def target(s):
        return h.main_bit + ((s - h.main_bit) // cb + 1) * cb

    starts = [h.main_bit + c * cb for c in range(nchunks)]
    found = dict(zip(starts, _run(body, h, [(s, target(s), c * h.npix // nchunks, cap)
                                            for c, s in enumerate(starts)], st)))
    while True:
        # the chain by bits, each piece at the first pixel the pieces before it give it
        chain, p, pos = [], h.main_bit, 0
        while p in found:
            x = found[p]
            chain.append(x + (pos,))
            pos += x[3]
            if x[4] != JOB_OK:
                break
            p = x[1]
        ended = bool(chain) and chain[-1][4] != JOB_OK
        # A piece decoded at another position stands when it stopped at its target short of the image's end and read
        # every token with the group of its true position; one that ended, failed or reaches the end may have done so
        # by its guess.
        moved = [k for k, x in enumerate(chain) if x[5] != x[8]]
        refused = {k for k in moved if chain[k][4] != JOB_OK or chain[k][8] + chain[k][3] >= h.npix}
        check_k = [k for k in moved if k not in refused]
        flagged = set()
        if h.groups > 1 and check_k:
            pieces = np.array([[chain[k][6], chain[k][2], chain[k][8]] for k in check_k], np.int64)
            flags = torch.zeros(len(check_k), dtype=torch.int32, device=body.device)
            check(lib.gsx_vp8l_check(*h.image_args(), _ptr(to_device(pieces, body.device)), len(check_k),
                                     _ptr(flags), _stream()), "gsx_vp8l_check")
            flagged = {check_k[int(i)] for i in np.flatnonzero(to_host(flags))}
        bad = refused | flagged
        if not bad and ended:
            return chain
        first = min(bad) if bad else len(chain)
        fp, fpos = (chain[first][0], chain[first][8]) if bad else (p, pos)
        if st["rounds"] >= max_rounds:
            st["serial_fallbacks"] += 1
            x = _run(body, h, [(fp, 8 * body.numel() + 1, fpos, max(h.npix - fpos, 1))], st)[0]
            return chain[:first] + [x + (fpos,)]
        st["rounds"] += 1
        st["group_mismatches"] += len(flagged)
        st["moved_refused"] += len(refused)
        st["false_starts"] += int(not ended)
        # re-decode every piece that does not stand at its chain position, the stop where the walk found no piece,
        # and every other stop not decoded yet (a chunk after a false start needs it)
        jobs = {chain[k][0]: chain[k][8] for k in bad}
        if not ended:
            jobs[p] = pos
        for y in list(found.values()):
            if y[4] == JOB_OK and y[1] > fp and y[1] not in found:
                jobs.setdefault(y[1], y[5] + y[3])
        # drop the pieces no chain can use any more (their token buffers go with the last piece that holds them)
        keep = {x[0] for x in chain[:first]}
        found = {s: x for s, x in found.items() if s in keep or s > fp}
        keys = sorted(jobs)
        for s, x in zip(keys, _run(body, h, [(s, target(s), jobs[s], cap) for s in keys], st)):
            found[s] = x


def _check_input(data):
    if isinstance(data, torch.Tensor):
        raise ValueError("decode_lossless reads the file's bytes, not a tensor")
    return memoryview(data).cast("B")


def decode_lossless(data, device="cuda", chunk_bits: int | None = None, max_rounds: int | None = None,
                    stats: dict | None = None, parallel_only: bool = False):
    """The RGBA pixels (uint8 CUDA [height, width, 4]) of the lossless RIFF WEBP file `data` (bytes-like), as
    Pillow's Image.open(...).convert('RGBA') gives them.  ValueError for a file that is not one lossless VP8L image
    (see container()) or that the decoder refuses.  chunk_bits sets the chunk size of the main image's speculative
    decode and max_rounds the re-decode rounds before the serial decode (tests use both to force each path); the
    pixels do not depend on them.  stats, when given, gains the counts of chunks, false starts (rounds whose walk
    broke at a start no piece had), group mismatches (pieces gsx_vp8l_check flagged), moved_refused (pieces decoded at
    another position that ended, failed or reach the image's end, so were re-decoded without a check), rounds,
    serial fallbacks and overflow re-runs, and the stream's features.  parallel_only: return None, after the
    header, for a stream whose main image has more than one prefix-code group or a colour cache -- there the chain
    mostly ends in the serial decode, or the cache replay runs on one thread, and Pillow is faster (DESIGN section
    10)."""
    mv = _check_input(data)
    c = container(mv)
    if c is None:
        raise ValueError("not a lossless RIFF WEBP file (VP8L, alone or after VP8X)")
    at, size, alpha = c
    from .hostcopy import to_device, to_host
    dev = torch.device(device)
    with torch.cuda.device(dev):
        body = to_device(np.frombuffer(mv[at:at + size], np.uint8), dev)
        h = _Header(body, bytes(mv[at:at + 5]))
        if parallel_only and (h.groups > 1 or h.cache_bits):
            return None
        st = {}
        chain = _main_tokens(body, h, chunk_bits, MAX_ROUNDS if max_rounds is None else max_rounds, st)
        last = chain[-1]
        total = sum(x[3] for x in chain)
        if last[4] == JOB_EOF:
            raise ValueError(f"VP8L: truncated main image (bit {last[1]})")
        if total < h.npix:
            raise ValueError("VP8L: the image data ends early")
        if total > h.npix:
            raise ValueError("VP8L: a copy past the last pixel")
        pieces = np.array([[x[6], x[2], x[8]] for x in chain if x[2]], np.int64)
        out = torch.empty(h.npix, dtype=torch.int32, device=dev)
        src = torch.empty(h.npix, dtype=torch.int32, device=dev)
        err = torch.zeros(1, dtype=torch.int32, device=dev)
        check(lib.gsx_vp8l_resolve(_ptr(to_device(pieces, dev)), len(pieces), h.xsize, h.npix, h.cache_bits,
                                   _ptr(out), _ptr(src), _ptr(err), _stream()), "gsx_vp8l_resolve")
        scratch = torch.empty(h.height // 32 + 2, dtype=torch.int32, device=dev)
        cur = out
        for kind, xs, bits, off in reversed(h.transforms):
            sub = h.ws[off:] if kind != 2 else None
            nxt = torch.empty(xs * h.height, dtype=torch.int32, device=dev) if kind == 3 else cur
            check(lib.gsx_vp8l_inverse(kind, _ptr(cur), _ptr(nxt), _ptr(sub), xs, h.height, bits, _ptr(scratch),
                                       _stream()), "gsx_vp8l_inverse")
            cur = nxt
        rgba = torch.empty((h.height, h.width, 4), dtype=torch.uint8, device=dev)
        check(lib.gsx_vp8l_rgba(_ptr(cur), _ptr(rgba), h.width * h.height, int(alpha), _stream()), "gsx_vp8l_rgba")
        e = int(to_host(err)[0])
        chain.clear()
    if e & 1:
        raise ValueError("VP8L: a copy from before the first pixel")
    if e & 2:
        raise ValueError("VP8L: a copy past the last pixel")
    if stats is not None:
        for k, v in st.items():
            stats[k] = stats.get(k, 0) + v
        stats.update(width=h.width, height=h.height, transforms=[t[0] for t in h.transforms],
                     cache_bits=h.cache_bits, groups=h.groups, meta_bits=h.meta_bits)
    return rgba

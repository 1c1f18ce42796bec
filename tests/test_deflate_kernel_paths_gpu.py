"""The DEFLATE and CRC-32 kernels (csrc/gsx_deflate.cu), path by path: every use of huffman(), both sides of the
candidate choice, runs against the 4 KiB tiles and the blocks, the densest tile, the block-count edges of
k_deflate_bases, the grid-stride loops of k_deflate_stored and k_crc_chunks, and misaligned CRC inputs.

Each case has a seeded builder.  An unmarked CPU test proves through deflate_oracle (its `info=`, `Block`, `tokens`)
or a NumPy restatement of the kernel's dispatch that the case reaches the branch it is named after, and decodes every
oracle file it builds with gzip and raw zlib: the oracle restates the kernel, so only an inflater neither of them
wrote catches a bug they share.  A `gpu` test asserts the device file equals the oracle's byte for byte (and
inflates), or, where the oracle cannot afford the size, that the device CRC equals zlib's."""
import gzip
import zlib

import numpy as np
import pytest

import deflate_oracle as do
import webp_oracle as wo

TILE = 4096                   # kTile: bytes per k_deflate_plan / k_deflate_emit tile
THREADS = 512                 # kThreads: k_deflate_bases spreads the blocks over one CTA of these
TILE_BITS = (TILE * 15 // 32 + 4) * 32   # kTileWords * 32: the bits of the shared ob[] tile buffer
CRC_CHUNK, CRC_PARTS = 4096, 1024
STORED_GRID_PER_SM = 16
H100_SMS = (114, 132)         # H100 PCIe, H100 SXM


def inflates(f: bytes, x: np.ndarray):
    assert gzip.decompress(f) == x.tobytes()
    d = zlib.decompressobj(-15)
    assert d.decompress(f[10:-8]) == x.tobytes() and d.eof and d.unused_data == b""


def oracle_file(x, breaks=(), info=None, level=6):
    f = do.gzip_file(x, level, 0, breaks, info)
    inflates(f, x)
    return f


def device_gzip(x, cuda, breaks=(), level=6):
    import torch
    from gsx import deflate
    return deflate.gzip(torch.from_numpy(np.ascontiguousarray(x)).to(cuda), level, mtime=0, breaks=breaks)


def check_device(x, cuda, breaks=(), level=6):
    want = do.gzip_file(x, level, 0, breaks)
    got = device_gzip(x, cuda, breaks, level)
    if got != want:
        diff = next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), min(len(got), len(want)))
        raise AssertionError(f"device file ({len(got)} B) differs from the oracle's ({len(want)} B) at byte {diff}")
    inflates(got, x)


def spread(values: np.ndarray) -> np.ndarray:
    """The bytes rearranged so that no two neighbours are equal (the most frequent value at most half of them): the
    values grouped by count, most frequent first, dealt to the even positions, then the odd ones."""
    v, c = np.unique(values, return_counts=True)
    order = np.argsort(-c, kind="stable")
    grouped = np.repeat(v[order], c[order])
    out = np.empty_like(grouped)
    half = (len(grouped) + 1) // 2
    out[0::2], out[1::2] = grouped[:half], grouped[half:]
    assert not (out[1:] == out[:-1]).any()
    return out


def lit_counts(x: np.ndarray) -> np.ndarray:
    c = np.bincount(x, minlength=286)
    c[256] += 1
    return c


def floor_doublings(counts, limit: int) -> int:
    """How often huffman() doubles its weight floor before the code fits `limit` bits."""
    counts = np.asarray(counts, np.int64)
    floor, k = 1, 0
    while wo.huffman_lengths(np.where(counts > 0, np.maximum(counts, floor), 0), 64).max() > limit:
        floor, k = floor * 2, k + 1
    return k


def cl_counts(runs) -> np.ndarray:
    return np.bincount([s for s, _ in runs], minlength=19)


def token_starts(blk) -> np.ndarray:
    """The byte offset in its block of each of a Block's tokens (the end-of-block code excluded)."""
    width = np.where(blk.is_copy, blk.val, 1)
    return np.cumsum(width) - width


def tile_bits(x: np.ndarray, copies: bool) -> np.ndarray:
    """The bits k_deflate_emit assembles per tile of one block: every token counts in the tile of its first byte."""
    blk = do.Block(x, copies, True)
    tiles = token_starts(blk) // TILE
    return np.bincount(tiles, weights=blk.cnts[:-1], minlength=-(-len(x) // TILE)).astype(np.int64)


def e_cache_uses(x: np.ndarray, b0: int, b1: int) -> list:
    """k_deflate_emit's e_cache, restated: for every tile of [b0, b1) whose last run goes on past it, ('scan', end)
    when the run's end is searched (run_end_after) or ('reuse', end) when the end found for an earlier tile is taken
    again."""
    e_cache, out = b0, []
    for t0 in range(b0, b1, TILE):
        last = min(t0 + TILE, b1) - 1
        if last + 1 < b1 and x[last + 1] == x[last]:
            if e_cache <= last:
                other = np.flatnonzero(x[last + 1:b1] != x[last])
                e_cache = last + 1 + int(other[0]) if len(other) else b1
                out.append(("scan", e_cache))
            else:
                out.append(("reuse", e_cache))
    return out


def noise(rng, n, avoid=()):
    """n random bytes, none in `avoid` and no two neighbours equal."""
    pool = np.setdiff1d(np.arange(256), np.asarray(avoid, np.int64)).astype(np.uint8)
    return pool[np.cumsum(rng.integers(1, len(pool), n)) % len(pool)]


# ------------------------------------------------------------------------------------------------ huffman()
def lit_floor_case():
    """Byte counts 1, 1, 2, 4, ..., 2^18 over 20 values, no two neighbours equal: the literal code needs a 19-bit
    leaf unlimited, so the floor doubles several times before it fits 15 bits."""
    rng = np.random.default_rng(15)
    vals = rng.choice(256, 20, replace=False).astype(np.uint8)
    counts = [1] + [1 << k for k in range(19)]
    return spread(np.repeat(vals, counts))


def cl_depth_case():
    """32767 bytes of dyadic counts (value s occurs 2^(15 - l_s) times, l_s a random complete code with the
    end-of-block at 15 bits), no two neighbours equal: the code lengths run-length coded take a code-length code
    8 bits deep unlimited, so huffman() at limit 7 has to raise its floor."""
    rng = np.random.default_rng(1)
    leaves, k = [0], rng.integers(20, 250)
    while len(leaves) < k:
        i = rng.integers(len(leaves))
        if leaves[i] < 15:
            d = leaves.pop(i)
            leaves += [d + 1, d + 1]
    leaves.sort()
    while leaves[-1] < 15:
        d = leaves.pop()
        leaves += [d + 1, d + 1]
    leaves.remove(15)                                    # the end-of-block's leaf: its count is 1
    vals = rng.choice(256, len(leaves), replace=False).astype(np.uint8)
    return spread(np.repeat(vals, [1 << (15 - d) for d in leaves]))


def test_lit_code_floor_doubles_at_least_twice():
    x = lit_floor_case()
    assert wo.huffman_lengths(lit_counts(x), 64).max() > 15 and floor_doublings(lit_counts(x), 15) >= 2
    info = {}
    oracle_file(x, info=info)
    assert info["copies"] == [0] and info["lit_len"][0].max() == 15


def test_lone_symbols_take_length_one():
    info = {}
    oracle_file(np.zeros(0, np.uint8), info=info)        # the empty block: the end-of-block code alone
    assert np.flatnonzero(info["lit_len"][0]).tolist() == [256] and info["lit_len"][0][256] == 1
    blk = do.Block(np.full(1000, 3, np.uint8), True, True)   # a copies block: distance code 0 alone
    assert blk.dist_len.tolist() == [1] + [0] * 29


def test_code_length_code_deeper_than_7_unlimited():
    x = cl_depth_case()
    assert len(x) == 32767 and not (x[1:] == x[:-1]).any()
    info = {}
    oracle_file(x, info=info)
    assert info["copies"] == [0]
    cl = cl_counts(info["runs"][0])
    assert wo.huffman_lengths(cl, 64).max() > 7 and floor_doublings(cl, 7) >= 1
    assert wo.huffman_lengths(cl, 7).max() <= 7


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lit_floor", "cl_depth", "empty", "one_run"])
def test_huffman_uses_match_oracle(name, cuda, gsx_lib):
    x = {"lit_floor": lit_floor_case, "cl_depth": cl_depth_case, "empty": lambda: np.zeros(0, np.uint8),
         "one_run": lambda: np.full(1000, 3, np.uint8)}[name]()
    check_device(x, cuda)


# ------------------------------------------------------------------------------------------------ candidate choice
def small_runs(seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 9, 24)
    return np.repeat(rng.integers(0, 3, 24).astype(np.uint8), lens)[:rng.integers(30, 90)]


CANDIDATE_SEEDS = {"tie": 23, "copies_by_one_bit": 210}   # found by a search over small_runs(seed)


def runs_of_2_3_case():
    rng = np.random.default_rng(23)
    vals = spread(rng.integers(0, 5, 2000).astype(np.uint8))
    return np.repeat(vals, rng.integers(1, 4, len(vals)))


def candidate_case(name):
    return runs_of_2_3_case() if name == "runs_of_2_3" else small_runs(CANDIDATE_SEEDS[name])


def test_candidates_tie_and_differ_by_one_bit():
    for name, (want_diff, want_copies) in {"tie": (0, 0), "copies_by_one_bit": (1, 1)}.items():
        x = candidate_case(name)
        lit, cp = do.Block(x, False, True), do.Block(x, True, True)
        assert cp.is_copy.any() and lit.bits - cp.bits == want_diff, name
        info = {}
        oracle_file(x, info=info)
        assert info["copies"] == [want_copies], name


def test_runs_of_2_3_never_build_copies():
    x = runs_of_2_3_case()
    starts = np.flatnonzero(np.concatenate([[True], x[1:] != x[:-1]]))
    r = np.diff(np.concatenate([starts, [len(x)]]))
    assert set(r.tolist()) == {1, 2, 3}
    assert not do.tokens(x, True)[0].any()               # no copy token: the kernel's ncopies stays 0
    info = {}
    oracle_file(x, info=info)
    assert info["copies"] == [0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tie", "copies_by_one_bit", "runs_of_2_3"])
def test_candidate_choice_matches_oracle(name, cuda, gsx_lib):
    check_device(candidate_case(name), cuda)


# ------------------------------------------------------------------------------------------------ runs, tiles, blocks
RUN = 0xAB


def run_edges_case():
    """A run ending on the last byte of tile 0, one starting on the first byte of tile 2."""
    rng = np.random.default_rng(4096)
    x = noise(rng, 4 * TILE, (RUN,))
    x[TILE - 300:TILE] = RUN
    x[2 * TILE:2 * TILE + 300] = RUN
    return x


def run_tiles_case():
    """Runs over 3, 5 and 9 tiles in one block: the middle tiles reuse the run end found for the first."""
    rng = np.random.default_rng(3)
    x = noise(rng, 20 * TILE, (RUN,))
    for first, k in ((1, 3), (5, 5), (11, 9)):
        x[first * TILE + 1000:(first + k - 1) * TILE + 100] = RUN
    return x


def copy_heads_case():
    """Runs of 1 + 2 * 258 + j bytes, j = 0..3, each placed so that its second (last full) copy's head is a tile's
    last byte: the copy and the j remainder bytes (literals, or a copy of 3) fall in the next tile."""
    rng = np.random.default_rng(258)
    x = noise(rng, 6 * TILE, (RUN,))
    for j in range(4):
        s = (j + 1) * TILE + TILE - 1 - (1 + 258)
        x[s:s + 1 + 2 * 258 + j] = RUN
    return x


BLOCK_END = 3 * TILE + 123


def run_to_block_end_case():
    """A run over three tiles ending on the block's last byte, the next block starting with ten more of that byte."""
    rng = np.random.default_rng(1951)
    x = noise(rng, 6 * TILE, (RUN,))
    x[BLOCK_END - 5000:BLOCK_END + 10] = RUN
    return x, (BLOCK_END,)


RUN_CASES = {"run_edges": lambda: (run_edges_case(), ()), "run_tiles": lambda: (run_tiles_case(), ()),
             "copy_heads": lambda: (copy_heads_case(), ()), "run_to_block_end": run_to_block_end_case,
             "one_mib_run": lambda: (np.full(do.BLOCK, 0x5A, np.uint8), ())}


def runs_of(x):
    starts = np.flatnonzero(np.concatenate([[True], x[1:] != x[:-1]]))
    return starts, np.diff(np.concatenate([starts, [len(x)]]))


def test_runs_on_tile_edges():
    x = run_edges_case()
    s, r = runs_of(x)
    long = r >= 4
    assert (s[long] + r[long]).tolist() == [TILE, 2 * TILE + 300] and s[long].tolist() == [TILE - 300, 2 * TILE]
    info = {}
    oracle_file(x, info=info)
    assert info["copies"] == [1]


def test_runs_over_3_5_9_tiles_reuse_e_cache():
    x = run_tiles_case()
    info = {}
    oracle_file(x, info=info)
    assert info["copies"] == [1]
    ends = [(first + k - 1) * TILE + 100 for first, k in ((1, 3), (5, 5), (11, 9))]
    want = [("scan", ends[0]), ("reuse", ends[0])] + [("scan", ends[1])] + [("reuse", ends[1])] * 3
    assert e_cache_uses(x, 0, len(x)) == want + [("scan", ends[2])] + [("reuse", ends[2])] * 7


def test_copy_heads_on_a_tiles_last_byte():
    x = copy_heads_case()
    blk = do.Block(x, True, True)
    at = token_starts(blk)
    heads = at[blk.is_copy & (blk.val == 258)]
    assert ((heads + 1) % TILE == 0).sum() == 4
    for j in range(4):
        head = (j + 2) * TILE - 1
        k = int(np.flatnonzero(at == head)[0])
        assert blk.is_copy[k] and blk.val[k] == 258
        tail = blk.val[k + 1:k + 1 + (1 if j == 3 else j)]
        if j == 3:
            assert blk.is_copy[k + 1] and tail.tolist() == [3]
        else:
            assert not blk.is_copy[k + 1:k + 1 + j].any() and (tail == RUN).all()
            assert at[k + 1 + j] == head + 258 + j and x[head + 258 + j] != RUN
        assert at[k + 1] // TILE == (j + 2)
    info = {}
    oracle_file(x, info=info)
    assert info["copies"] == [1]


def test_run_ends_on_block_end_and_next_block_repeats_its_byte():
    x, breaks = run_to_block_end_case()
    assert x[BLOCK_END - 1] == x[BLOCK_END] == RUN and x[BLOCK_END - 5001] != RUN
    assert e_cache_uses(x, 0, BLOCK_END) == [("scan", BLOCK_END), ("reuse", BLOCK_END)]   # stops at the block end
    info = {}
    oracle_file(x, breaks, info=info)
    assert info["copies"] == [1, 1]


def test_one_mib_block_is_one_run():
    x = np.full(do.BLOCK, 0x5A, np.uint8)
    assert do.block_starts(len(x)) == [0]
    blk = do.Block(x, True, True)
    assert not blk.is_copy[0] and blk.is_copy[1:].all() and blk.val[1:].sum() == len(x) - 1
    assert e_cache_uses(x, 0, len(x)) == [("scan", len(x))] + [("reuse", len(x))] * (len(x) // TILE - 2)
    inflates(oracle_file(x), x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(RUN_CASES))
def test_runs_match_oracle(name, cuda, gsx_lib):
    x, breaks = RUN_CASES[name]()
    check_device(x, cuda, breaks)


# ------------------------------------------------------------------------------------------------ densest tile
DENSE_TILE = 100


def densest_tile_case():
    """1 MiB: bytes 128..255 32 times each, shuffled, filling tile 100; the rest bytes 0..15 at probabilities 2^-(v+1)
    (the remainder on 0): every byte of tile 100 takes a 15-bit literal."""
    rng = np.random.default_rng(61568)
    p = 0.5 ** np.arange(1, 17)
    p[0] += 1 - p.sum()
    x = rng.choice(16, do.BLOCK, p=p).astype(np.uint8)
    x[DENSE_TILE * TILE:(DENSE_TILE + 1) * TILE] = rng.permutation(np.repeat(np.arange(128, 256), 32))
    return x


def test_densest_tile_fills_most_of_the_tile_buffer():
    x = densest_tile_case()
    info = {}
    oracle_file(x, info=info)
    bits = tile_bits(x, bool(info["copies"][0]))
    assert bits.argmax() == DENSE_TILE and bits[DENSE_TILE] > 14 * TILE
    assert bits.max() + 31 <= TILE_BITS                 # the kernel's bound, with the tile's first bit offset


@pytest.mark.gpu
def test_densest_tile_matches_oracle(cuda, gsx_lib):
    check_device(densest_tile_case(), cuda)


# ------------------------------------------------------------------------------------------------ block counts
BLOCK_COUNTS = (511, 512, 513, 1024, 1025)


def block_count_case(nb):
    rng = np.random.default_rng(nb)
    n = 6 * nb + 5
    x = rng.integers(0, 3, n).astype(np.uint8)
    x[rng.random(n) < 0.3] = 2                            # some runs of 4 or more: some blocks take copies
    return x, tuple(i * n // nb for i in range(1, nb))


def test_block_counts_reach_every_bases_split():
    seen_per, empty = set(), {}
    for nb in BLOCK_COUNTS:
        x, breaks = block_count_case(nb)
        assert len(do.block_starts(len(x), breaks)) == nb
        per = -(-nb // THREADS)                           # k_deflate_bases: blocks per thread
        lo = np.minimum(nb, np.arange(THREADS) * per)
        empty[nb] = int((np.minimum(nb, lo + per) == lo).sum())
        seen_per.add(per)
    assert seen_per == {1, 2, 3}
    assert empty == {511: 1, 512: 0, 513: 255, 1024: 0, 1025: 170}
    x, breaks = block_count_case(513)
    starts = do.block_starts(len(x), breaks)
    assert any(do.tokens(x[a:b], True)[0].any() for a, b in zip(starts, starts[1:]))   # some build copies
    oracle_file(x, breaks)


@pytest.mark.gpu
@pytest.mark.parametrize("nb", BLOCK_COUNTS)
def test_block_counts_match_oracle(nb, cuda, gsx_lib):
    x, breaks = block_count_case(nb)
    check_device(x, cuda, breaks)


# ------------------------------------------------------------------------------------------------ stored blocks
def stored_sizes(sms):
    """n = 16 * SMs * 65535 + d: d = -1 fills the grid short of one block, d = +1 sends one CTA round again."""
    g = STORED_GRID_PER_SM * sms
    return {d: g * do.STORED + d for d in (-1, 1)}


@pytest.mark.parametrize("sms", H100_SMS)
def test_stored_sizes_straddle_the_grid(sms):
    grid = STORED_GRID_PER_SM * sms
    for d, n in stored_sizes(sms).items():
        nb = -(-n // do.STORED)
        assert (nb > grid) == (d > 0) and nb >= grid
    x = np.random.default_rng(0).integers(0, 256, 2 * do.STORED + 1, dtype=np.uint8)
    inflates(do.gzip_file(x, 0, 0), x)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [-1, 1])
def test_stored_grid_stride_matches_oracle(d, cuda, gsx_lib):
    import torch
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    n = stored_sizes(sms)[d]
    x = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8)
    got = device_gzip(x, cuda, level=0)
    want = do.header(0, 0) + do.body(x, 0)
    assert got[:-8] == want, "stored body differs from the oracle's"
    assert got[-8:] == zlib.crc32(x).to_bytes(4, "little") + n.to_bytes(4, "little")
    assert gzip.decompress(got) == x.tobytes()


# ------------------------------------------------------------------------------------------------ CRC-32
CRC_OFFSETS = tuple(range(17))                            # 0 and 16: the 16-byte loads; 1..15: the byte loop only
CRC_LENGTHS = (1, 15, 16, 17, 31, 33, 4095, 4096, 4097, 8192 + 15, 3 * 4096 + 1, 65536 + 7)
CRC_BIG = (1 << 30) + (1 << 26) + 12345


def test_crc_shapes_reach_every_path():
    assert {n % 16 for n in CRC_LENGTHS} >= {0, 1, 15} and {n % CRC_CHUNK for n in CRC_LENGTHS} >= {0, 1, 4095}
    assert {o % 16 for o in CRC_OFFSETS} == set(range(16))
    nchunks = -(-CRC_BIG // CRC_CHUNK)
    parts = max(1, min(-(-nchunks // 256), CRC_PARTS))
    assert parts == CRC_PARTS and nchunks > parts * 256     # every thread's chunk loop goes round again


def device_crc(t, gsx_lib):
    import torch
    from gsx._abi import _ptr, _stream, check
    ws = torch.empty(gsx_lib.gsx_deflate_workspace_bytes(0), dtype=torch.uint8, device=t.device)
    trailer = torch.zeros(8, dtype=torch.uint8, device=t.device)
    check(gsx_lib.gsx_crc32(_ptr(t), t.numel(), _ptr(ws), ws.numel(), _ptr(trailer), _stream()), "gsx_crc32")
    return bytes(trailer.cpu().numpy())


@pytest.mark.gpu
def test_crc_misaligned_equals_zlib(cuda, gsx_lib):
    import torch
    rng = np.random.default_rng(16)
    x = rng.integers(0, 256, max(CRC_LENGTHS) + 32, dtype=np.uint8)
    t = torch.from_numpy(x).to(cuda)
    assert t.data_ptr() % 256 == 0
    for o in CRC_OFFSETS:
        for n in CRC_LENGTHS:
            got = device_crc(t[o:o + n], gsx_lib)
            assert got == zlib.crc32(x[o:o + n]).to_bytes(4, "little") + n.to_bytes(4, "little"), (o, n)


def big_chunk(lo, hi, dev):
    import torch
    i = torch.arange(lo, hi, dtype=torch.int64, device=dev)
    return ((((i * 2654435761) & 0xFFFFFFFF) >> 13) & 255).to(torch.uint8)


@pytest.mark.gpu
def test_crc_past_1024_parts_equals_zlib(cuda, gsx_lib):
    import torch
    step = 1 << 26
    x = torch.empty(CRC_BIG, dtype=torch.uint8, device=cuda)
    for lo in range(0, CRC_BIG, step):
        x[lo:min(CRC_BIG, lo + step)] = big_chunk(lo, min(CRC_BIG, lo + step), cuda)
    got = device_crc(x, gsx_lib)
    crc = 0
    for lo in range(0, CRC_BIG, step):
        crc = zlib.crc32(x[lo:lo + step].cpu().numpy(), crc)
    del x
    torch.cuda.empty_cache()
    assert got == crc.to_bytes(4, "little") + (CRC_BIG & 0xFFFFFFFF).to_bytes(4, "little")

"""The SOR k-NN kernels path by path: every K form, each bucket walk, the numeric edges of the contract, the range and
strided entry points and the visit counters, each on a cloud built to reach that path at the shipped constants.

Every case is a geometry builder (a plain function returning float32 xyz) and two kinds of test:
  * an unmarked CPU test asserting the geometry's PRECONDITION with the oracle's own grid (cell size, int64 bucket
    table, probe hashes) -- the path the case is meant to reach.  If a builder drifts off its path, this fails
    without a GPU;
  * a `gpu` test asserting the kernel's output bit-equal to the oracle in both hash modes, the STATS instantiation
    equal to the plain one, its counters equal to the oracle's, and the mask equal to `oracle.threshold_mask`.

Query-kernel constants these cases are built around (csrc/gsx_sor.cu): K <= 16 batched epilogue with row stride 17,
K <= 32 stride 33, K > 32 two registers per lane and the shuffle epilogue, K clamped to 50; kMergeThreshold = 9;
kSmallBucket = 64 (plain scan up to it); a longer bucket spanning fewer than kFlatSupers = 8 supers of 1024 sorted
points walks its chunk boxes directly, a longer one walks super -> chunk; the own-chunk seed when the centre probe
reaches the query's own big bucket; self-skip d2 > 1e-12; the 1e10 sentinel and the < 0.9e10 validity test.

Not covered: clouds whose grid index exceeds int32.  There CUDA's saturating float -> int conversion and the oracle's
x86 conversion disagree, and what the reference itself does is not pinned.
"""
import functools

import numpy as np
import pytest

import oracle
from oracle.sor import sor_hash_table

MODES = ("i32wrap", "i64")
P1, P2, P3 = 73856093, 19349663, 83492791
SMALL_BUCKET, FLAT_SUPERS = 64, 8
PATTERN = np.uint32(0x7FC0BEEF)          # a NaN that no kernel writes: marks rows a query range must not touch
SWEEP_KS = list(range(1, 51)) + [51, 64, 1000]


# ------------------------------------------------------------------------------------------------ geometry builders
def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    a.setflags(write=False)
    return a


def _corners(lo, hi):
    return np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float64)


@functools.lru_cache(None)
def mixed_cloud():
    """~20 k points of the synthetic mixed cloud; n is odd, so the last batch of 16 queries is partial."""
    from gsx import synth
    return _f32(synth.xyz(20_011, "mixed"))


@functools.lru_cache(None)
def long_bucket():
    """12 000 points spread uniformly over most of one cell (cell 277.3, set by corners at +-1000): one bucket of
    12 000 points, walked super -> chunk.  The spread keeps the Morton-ordered chunks and supers spatially tight, so
    both box levels really prune."""
    rng = np.random.default_rng(3)
    return _f32(np.r_[rng.uniform(-130.0, 70.0, (12_000, 3)), _corners((-1000.0,) * 3, (1000.0,) * 3)])


@functools.lru_cache(None)
def flat_bucket():
    """3 000 points inside one cell (cell 440.0): one long bucket spanning at most 4 supers -> the flat chunk walk."""
    rng = np.random.default_rng(4)
    return _f32(np.r_[rng.uniform(-80.0, 280.0, (3_000, 3)), _corners((-1000.0,) * 3, (1000.0,) * 3)])


EDGE_N, EDGE_CELLS = 4_000, {64: (1, 1, 1), 65: (3, 3, 2)}


@functools.lru_cache(None)
def edge_buckets():
    """A [0,1]^3 background (cell 0.2) that leaves two cells empty, filled with exactly 64 and 65 points: the
    kSmallBucket edge (a plain scan of 64, a box walk of 65 with the own-chunk seed)."""
    rng = np.random.default_rng(5)
    cell = 0.2
    pts = [np.zeros((1, 3)), np.ones((1, 3))]
    for size, c in EDGE_CELLS.items():
        lo = np.array(c) * cell
        pts.append(rng.uniform(lo + 0.1 * cell, lo + 0.9 * cell, (size, 3)))
    need = EDGE_N - sum(len(p) for p in pts)
    bg = rng.uniform(0.0, 1.0, (3 * need, 3))
    gi = np.floor(bg / cell).astype(np.int64)
    keep = np.ones(len(bg), bool)
    for c in EDGE_CELLS.values():
        keep &= ~np.all(np.abs(gi - np.array(c)) <= 0, axis=1)
    pts.append(bg[keep][:need])
    return _f32(np.concatenate(pts))


@functools.lru_cache(None)
def wrapped_centre():
    """A 12 000-point blob at x = 19 000, corners x in {-1000, 20000}, y, z = +-1000: cell 607.2 and grid cell
    (32, 1, 1).  The int64 table puts the blob in bucket 4736; the i32-wrapped centre probe lands in 10848, so under
    i32wrap the query's own big bucket is not reached and the own-chunk seed must be skipped."""
    rng = np.random.default_rng(6)
    blob = rng.normal(0.0, 1e-3, (12_000, 3)) + np.array([19_000.0, 0.0, 0.0])
    return _f32(np.r_[blob, _corners((-1000.0, -1000.0, -1000.0), (20_000.0, 1000.0, 1000.0))])


@functools.lru_cache(None)
def self_skip_twins():
    """2 000 points in [0.25, 1) and a twin of each, 1..20 ulp away along one, two or three axes: twin d2 from
    ~1e-14 to ~1e-11, straddling the self-skip threshold 1e-12."""
    rng = np.random.default_rng(7)
    base = rng.uniform(0.25, 1.0, (2_000, 3)).astype(np.float32)
    steps = rng.integers(1, 21, (2_000, 1)).astype(np.uint32)
    axes = rng.integers(0, 2, (2_000, 3)).astype(bool)
    axes[~axes.any(axis=1), 0] = True
    twin = (base.view(np.uint32) + np.where(axes, steps, 0).astype(np.uint32)).view(np.float32)
    return _f32(np.r_[base, twin])


@functools.lru_cache(None)
def sentinel_band():
    """Around the 1e10 sentinel: a 3x3x3 lattice of spacing 0.95e10, whose axis neighbours lie in [0.9e10, 1e10)
    (inserted into the list, not counted by the mean) and whose diagonals lie past 1e10 (never inserted), plus 64
    points uniform in [0, 1e10)^3 and 12 among the lattice, nearer than 0.9e10 to something (counted).  The grid is
    one or two cells wide, so every point probes every occupied cell."""
    rng = np.random.default_rng(8)
    lattice = np.stack(np.meshgrid(*[np.arange(3)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.95e10
    return _f32(np.r_[lattice, rng.uniform(0.0, 1.9e10, (12, 3)), rng.uniform(0.0, 1e10, (64, 3))])


@functools.lru_cache(None)
def isolated_points():
    """A dense blob of 4 000 points at the centre of [0, 1000]^3 (cell 200) and the 8 corners, two or more cells
    away from it: most corners probe nothing but themselves, and their mean must be 0."""
    rng = np.random.default_rng(9)
    return _f32(np.r_[rng.uniform(499.0, 501.0, (4_000, 3)), _corners((0.0,) * 3, (1000.0,) * 3)])


FACES_N = 3_000


@functools.lru_cache(None)
def cell_faces():
    """[0,1]^3 with coordinates snapped onto cell faces: (x - bmin) / cell is an integer, or one ulp below one."""
    rng = np.random.default_rng(10)
    pts = rng.uniform(0.0, 1.0, (FACES_N, 3)).astype(np.float32)
    pts[0], pts[1] = 0.0, 1.0                                       # fixes bmin = 0, the bbox and so the cell
    _, cell = oracle.sor_cell_size(pts)
    c = np.float32(cell)
    m = rng.integers(1, int(1.0 / cell), pts.shape).astype(np.float32)
    on = m * c                                                      # float32 product: m*cell rounded
    below = np.nextafter(on, np.float32(0.0))
    pick = rng.integers(0, 3, pts.shape)
    pick[:2] = 2
    pts = np.where(pick == 0, on, np.where(pick == 1, below, pts))
    return _f32(pts)


@functools.lru_cache(None)
def signed_zero():
    """Negative coordinates, exact 0.0 and -0.0 (also as twins of each other: d2 = 0, skipped as self)."""
    rng = np.random.default_rng(11)
    pts = rng.normal(0.0, 1.0, (3_000, 3)).astype(np.float32)
    z = rng.integers(0, 4, pts.shape)
    pts = np.where(z == 0, np.float32(-0.0), np.where(z == 1, np.float32(0.0), pts))
    twins = pts[:300].copy()
    twins[twins == 0] = -twins[twins == 0]                           # flip the sign of every zero
    return _f32(np.r_[pts, twins])


def small_cloud(n):
    return _f32(np.random.default_rng(1000 + n).normal(0.0, 1.0, (n, 3)))


def crafted_pairwise_rows():
    """Rows of exact distances on the x axis (d = |dx| exactly in float64) whose NumPy mean depends on the pairwise
    order: at k = 8 the 8-accumulator tree gives 0x3e000000 and a serial sum one ulp more; k = 9 adds the remainder
    after the block, k = 16 a second pass of the block.  Each row sits at its own z, 1000 apart; its query is the
    point at x = 0."""
    rows = {
        8: [2.0 ** -62] * 4 + [2.0 ** -54] * 2 + [2.0 ** -24, 1.0],
        9: [2.0 ** -61, 2.0 ** -58, 2.0 ** -58, 3 * 2.0 ** -55, 3 * 2.0 ** -53, 3 * 2.0 ** -52, 9 * 2.0 ** -24, 1.0, 8.0],
        16: [2.0 ** -62] * 8 + [2.0 ** -54] * 4 + [2.0 ** -24] * 2 + [1.0, 1.0],
    }
    pts = []
    for i, (k, d) in enumerate(rows.items()):
        z = 1000.0 * i
        pts.append([0.0, 0.0, z])
        pts.extend([x, 0.0, z] for x in d)
    return _f32(pts), rows


# ------------------------------------------------------------------------------------------------ oracle-side helpers
def _grid(xyz):
    """The oracle's grid: bmin, cell, int32 grid index per point, and the int64 bucket table."""
    lo, cell = oracle.sor_cell_size(xyz)
    gi = np.floor((xyz - lo) / np.float32(cell)).astype(np.int32).astype(np.int64)
    order, start, count = sor_hash_table(xyz, lo, cell)
    return lo, cell, gi, order, start, count


def _wrap32(v):
    return ((v + 2 ** 31) % 2 ** 32) - 2 ** 31


def _probe_hashes(gi, n, mode):
    """[m, 27] bucket of every probe, in the reference's loop order (dx outer, dz inner); probe 13 is the centre."""
    off = np.array([(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)], np.int64)
    g = gi[:, None, :] + off[None]
    prods = [g[..., 0] * P1, g[..., 1] * P2, g[..., 2] * P3]
    if mode == "i32wrap":
        prods = [_wrap32(p) for p in prods]
    return (prods[0] ^ prods[1] ^ prods[2]) % n


def _table_bucket(gi, n):
    return _probe_hashes(gi, n, "i64")[:, 13]


def _walk_form(start, count):
    """Which walk k_sor_knn takes over a bucket of `count` points starting at sorted position `start`."""
    if count <= SMALL_BUCKET:
        return "plain"
    fc, lc = start >> 5, (start + count - 1) >> 5
    return "flat" if (lc >> 5) - (fc >> 5) < FLAT_SUPERS else "super"


def _candidates(xyz, mode, rows):
    """Restatement of the oracle's candidate multiset for the given rows: float32 distances of every point of every
    probed bucket (a bucket reached by two probes counts twice) that passes the self-skip d2 > 1e-12."""
    lo, cell, gi, order, start, count = _grid(xyz)
    spos = xyz[order]
    out = []
    for r, hs in zip(rows, _probe_hashes(gi[rows], len(xyz), mode)):
        idx = np.concatenate([np.arange(start[h], start[h] + count[h]) for h in hs if start[h] != -1])
        a = xyz[r] - spos[idx]
        d2 = (a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2]
        out.append(np.sort(np.sqrt(d2[d2 > np.float32(1e-12)])))
    return out


def _list_for(cands, k):
    """The oracle's list for K = min(k, 50): the K smallest inserted (< 1e10) distances."""
    return cands[cands < np.float32(1e10)][:min(k, 50)]


def _emulated_mean(cands, k):
    s, valid = np.float32(0.0), 0
    for v in _list_for(cands, k):
        if v < np.float32(0.9e10):
            s = np.float32(s + v)
            valid += 1
    return np.float32(s / np.float32(valid)) if valid else np.float32(0.0)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _assert_bits(got, want, what):
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert bad.size == 0, f"{what}: {bad.size} rows differ, first {bad[:5]}: got {got[bad[:5]]} want {want[bad[:5]]}"


# ------------------------------------------------------------------------------------------------ GPU helpers
def _check_sor(xyz, ks, mode, cuda, sigma=1.0):
    """Bit-equality of mean_dists (plain and STATS), of sor_filter's means and mask, and of the counters."""
    import torch
    from gsx import sor
    n = len(xyz)
    x = torch.from_numpy(np.array(xyz)).to(cuda)
    grid = sor.build_grid(x)
    _, cell = oracle.sor_cell_size(xyz)
    assert grid.cell == np.float32(cell)          # the oracle's kernel, like the reference's, takes the cell as float32
    _, visits = oracle.sor_taichi_mean_dists(xyz, 1, mode, want_visits=True)
    got = {}
    for k in ks:
        want = oracle.sor_taichi_mean_dists(xyz, k, mode)
        plain = sor.mean_dists(grid, k, mode).cpu().numpy()
        _assert_bits(plain, want, f"mean_dists k={k} {mode}")
        counted, st = sor.mean_dists(grid, k, mode, want_stats=True)
        _assert_bits(counted.cpu().numpy(), plain, f"mean_dists(want_stats) k={k} {mode}")
        assert st["queries"] == n, (k, mode, st)
        assert st["visits"] == int(visits.sum()), (k, mode, st, int(visits.sum()))
        mask, means = sor.sor_filter(x, k, sigma, hash_mode=mode, return_means=True)
        _assert_bits(means.cpu().numpy(), want, f"sor_filter k={k} {mode}")
        assert np.array_equal(mask.cpu().numpy(), oracle.threshold_mask(want, sigma)), (k, mode)
        got[k] = plain
    return got


def _sorted_rows(grid):
    """Original row of every hash-sorted position (the w lane of the grid's float4 positions)."""
    import torch
    from gsx._abi import lib
    off = lib.gsx_sor_spos_offset(grid.n)
    spos = grid.ws[off: off + grid.n * 16].view(torch.int32).view(grid.n, 4)
    return spos[:, 3].cpu().numpy().astype(np.int64)


def _prefilled(n, cuda):
    import torch
    return torch.from_numpy(np.full(n, PATTERN, np.uint32).view(np.float32)).to(cuda)


# ================================================================================================ K sweep
def test_k_sweep_geometries_reach_every_walk(gsx_lib):
    for build, forms in ((mixed_cloud, {"plain", "flat"}), (long_bucket, {"plain", "super"})):
        xyz = build()
        _, _, _, _, start, count = _grid(xyz)
        occ = np.flatnonzero(count)
        assert {_walk_form(start[h], count[h]) for h in occ} >= forms, build.__name__


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geometry", ["mixed_cloud", "long_bucket"])
def test_k_sweep(geometry, mode, cuda, gsx_lib):
    """Every k in 1..50 (all three template forms, both sides of 16/17 and 32/33) and k > 50, which must give the
    k = 50 bits."""
    xyz = globals()[geometry]()
    got = _check_sor(xyz, SWEEP_KS, mode, cuda)
    for k in (51, 64, 1000):
        _assert_bits(got[k], got[50], f"k={k} vs k=50 {mode}")


# ================================================================================================ small n
def test_small_n_probes_alias():
    """With hash mod n this small, two of a query's 27 probes often reach the same bucket (scanned twice)."""
    for mode in MODES:
        aliased = 0
        for n in range(1, 81):
            xyz = small_cloud(n)
            _, _, gi, _, start, _ = _grid(xyz)
            hs = _probe_hashes(gi, n, mode)
            occ = np.where(start[hs] != -1, hs, -1)
            aliased += sum(len(set(r[r >= 0])) < (r >= 0).sum() for r in occ)
        assert aliased > 500, (mode, aliased)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_small_n_exhaustive(mode, cuda, gsx_lib):
    for n in range(1, 81):
        _check_sor(small_cloud(n), (1, 2, 8, 9, 16, 17, 32, 33, 50), mode, cuda)


# ================================================================================================ bucket walks
def test_edge_buckets_precondition():
    xyz = edge_buckets()
    assert len(xyz) == EDGE_N
    lo, cell, gi, _, start, count = _grid(xyz)
    assert abs(cell - 0.2) < 1e-6 and not lo.any()
    for size, c in EDGE_CELLS.items():
        h = _table_bucket(np.array([c], np.int64), EDGE_N)[0]
        assert count[h] == size, (size, count[h])
        assert _walk_form(start[h], count[h]) == ("plain" if size <= SMALL_BUCKET else "flat")


def test_long_bucket_preconditions():
    for build, size, form in ((flat_bucket, 3_000, "flat"), (long_bucket, 12_000, "super")):
        xyz = build()
        _, _, gi, _, start, count = _grid(xyz)
        blob = gi[:size]
        assert (blob == blob[0]).all(), build.__name__                 # the blob fills one cell ...
        h = _table_bucket(blob[:1], len(xyz))[0]
        assert count[h] == size and _walk_form(start[h], count[h]) == form, (build.__name__, count[h])   # ... one bucket
        for mode in MODES:                                             # whose centre probe reaches it: own-chunk seed
            assert _probe_hashes(blob[:1], len(xyz), mode)[0, 13] == h
        assert form != "super" or count[h] >= 9 * 1024               # super walk from wherever the bucket starts


def test_wrapped_centre_precondition():
    xyz = wrapped_centre()
    n = len(xyz)
    _, cell, gi, _, start, count = _grid(xyz)
    assert abs(cell - 607.2) < 0.1
    blob = gi[:12_000]
    assert (blob == np.array([32, 1, 1])).all()
    h = _table_bucket(blob[:1], n)[0]
    assert h == 4736 and count[h] == 12_000 and _walk_form(start[h], count[h]) == "super"
    assert _probe_hashes(blob[:1], n, "i64")[0, 13] == h
    wrapped = _probe_hashes(blob[:1], n, "i32wrap")[0]
    assert wrapped[13] == 10848 and h not in wrapped                 # i32wrap never reaches the own bucket
    a = oracle.sor_taichi_mean_dists(xyz, 16, "i32wrap")[:12_000]
    b = oracle.sor_taichi_mean_dists(xyz, 16, "i64")[:12_000]
    assert (a != b).all()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geometry", ["edge_buckets", "flat_bucket", "long_bucket", "wrapped_centre"])
def test_bucket_walks(geometry, mode, cuda, gsx_lib):
    _check_sor(globals()[geometry](), (1, 8, 9, 16, 17, 32, 33, 50), mode, cuda)


# ================================================================================================ numeric edges
def test_self_skip_twins_straddle_threshold():
    xyz = self_skip_twins()
    a = xyz[:2_000] - xyz[2_000:]
    d2 = (a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2]
    eps = np.float32(1e-12)
    assert (d2 > 0).all()
    assert ((d2 <= eps).sum() > 300) and ((d2 > eps).sum() > 300), (d2.min(), d2.max())
    _, _, gi, _, _, _ = _grid(xyz)
    assert (gi[:2_000] == gi[2_000:]).all(axis=1).mean() > 0.95       # twins share a cell: always probed


def test_sentinel_band_precondition():
    xyz = sentinel_band()
    rows = np.arange(len(xyz))
    band = np.float32(0.9e10), np.float32(1e10)
    for mode in MODES:
        cands = _candidates(xyz, mode, rows)
        want = oracle.sor_taichi_mean_dists(xyz, 50, mode)
        assert np.array_equal(_bits([_emulated_mean(c, 50) for c in cands]), _bits(want))    # the restatement holds
        for k in (8, 16, 17, 32, 33, 50):                              # every epilogue: band entries in some lists
            hit = sum(((_list_for(c, k) >= band[0]) & (_list_for(c, k) < band[1])).any() for c in cands)
            assert hit >= 1, (mode, k)
        far = sum((c >= band[1]).any() for c in cands)                 # and distances past the sentinel, never inserted
        assert far >= 1


def test_isolated_points_precondition():
    xyz = isolated_points()
    rows = np.arange(len(xyz) - 8, len(xyz))
    for mode in MODES:
        cands = _candidates(xyz, mode, rows)
        lonely = [r for r, c in zip(rows, cands) if len(c) == 0]
        assert len(lonely) >= 4, (mode, lonely)
        assert (oracle.sor_taichi_mean_dists(xyz, 16, mode)[lonely] == 0).all()


def test_cell_faces_precondition():
    xyz = cell_faces()
    lo, cell, gi, _, _, _ = _grid(xyz)
    assert not lo.any() and len(xyz) == FACES_N
    q = (xyz - lo) / np.float32(cell)
    integer = (q == np.floor(q)) & (q > 0)
    just_below = np.nextafter(q, np.float32(np.inf)) == np.ceil(q)
    assert integer.sum() > 1000 and just_below.sum() > 1000, (integer.sum(), just_below.sum())


def test_signed_zero_precondition():
    xyz = signed_zero()
    neg_zero = (xyz == 0) & np.signbit(xyz)
    pos_zero = (xyz == 0) & ~np.signbit(xyz)
    assert neg_zero.sum() > 1000 and pos_zero.sum() > 1000 and (xyz < 0).sum() > 1000
    assert (oracle.sor_cell_size(xyz)[0] < 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geometry,ks", [
    ("self_skip_twins", (1, 2, 8, 16, 17, 33)),
    ("sentinel_band", tuple(range(1, 51)) + (64,)),
    ("isolated_points", (1, 16, 17, 33, 50)),
    ("cell_faces", (1, 9, 16, 17, 32, 33, 50)),
    ("signed_zero", (1, 9, 16, 17, 32, 33, 50)),
])
def test_numeric_edges(geometry, ks, mode, cuda, gsx_lib):
    got = _check_sor(globals()[geometry](), ks, mode, cuda)
    if geometry == "isolated_points":
        assert all((got[k] == 0).sum() >= 4 for k in ks)


# ================================================================================================ range / strided
@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geometry", ["mixed_cloud", "long_bucket"])
def test_query_range_writes_exactly_its_rows(geometry, mode, cuda, gsx_lib):
    """Unaligned cuts: batches starting at 5, 20, 37 straddle two 32-position cell-bit words."""
    from gsx import sor
    import torch
    xyz = globals()[geometry]()
    n = len(xyz)
    grid = sor.build_grid(torch.from_numpy(np.array(xyz)).to(cuda))
    rows = _sorted_rows(grid)
    assert np.array_equal(np.sort(rows), np.arange(n))
    _, visits = oracle.sor_taichi_mean_dists(xyz, 1, mode, want_visits=True)
    cuts = [0, 5, 20, 37, 37, 1000, n - 1, n]                          # (37, 37) is an empty range
    for k in (1, 16, 17, 33, 50):
        full = sor.mean_dists(grid, k, mode).cpu().numpy()
        _assert_bits(full, oracle.sor_taichi_mean_dists(xyz, k, mode), f"full k={k}")
        union = np.full(n, PATTERN, np.uint32)
        for qb, qe in zip(cuts, cuts[1:]):
            out, st = sor.mean_dists(grid, k, mode, out=_prefilled(n, cuda), want_stats=True, q_range=(qb, qe))
            got = _bits(out.cpu().numpy())
            own = np.zeros(n, bool)
            own[rows[qb:qe]] = True
            assert np.array_equal(got[own], _bits(full)[own]), (k, qb, qe)
            assert (got[~own] == PATTERN).all(), (k, qb, qe, np.flatnonzero(got[~own] != PATTERN)[:5])
            assert st["queries"] == qe - qb and st["visits"] == int(visits[rows[qb:qe]].sum()), (k, qb, qe, st)
            union[own] = got[own]
        assert np.array_equal(union, _bits(full)), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_strided_queries_partition_the_batches(mode, cuda, gsx_lib):
    from gsx import sor
    import torch
    xyz = mixed_cloud()
    n = len(xyz)
    assert n % 16
    grid = sor.build_grid(torch.from_numpy(np.array(xyz)).to(cuda))
    rows = _sorted_rows(grid)
    batch = np.arange(n) // 16
    _, visits = oracle.sor_taichi_mean_dists(xyz, 1, mode, want_visits=True)
    for k in (8, 17, 50):
        full = _bits(sor.mean_dists(grid, k, mode).cpu().numpy())
        for stride in range(1, 6):
            union = np.full(n, PATTERN, np.uint32)
            for phase in range(stride):
                out, st = sor.mean_dists_strided(grid, k, mode, _prefilled(n, cuda), stride, phase, want_stats=True)
                got = _bits(out.cpu().numpy())
                own = np.zeros(n, bool)
                own[rows[batch % stride == phase]] = True
                assert np.array_equal(got[own], full[own]), (k, stride, phase)
                assert (got[~own] == PATTERN).all(), (k, stride, phase)
                assert st["queries"] == own.sum() and st["visits"] == int(visits[own].sum()), (k, stride, phase, st)
                union[own] = got[own]
            assert np.array_equal(union, full), (k, stride)


# ================================================================================================ cKDTree semantics
def test_crafted_rows_depend_on_numpy_order():
    """The crafted rows are where a different summation order than NumPy's pairwise one changes the float32 mean."""
    _, rows = crafted_pairwise_rows()
    for k, d in rows.items():
        d = np.array(d)
        serial = np.float32(functools.reduce(lambda s, v: s + v, d, 0.0) / k)
        numpy_mean = np.float32(np.mean(d[None, :], axis=1)[0])
        assert serial != numpy_mean, k


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0.0, 1e5])
def test_ckdtree_every_k(offset, cuda, gsx_lib):
    """k = 1..63: KK = k + 1 crosses the register split at 32/33 and the mean's k < 8 / 8-block / remainder forms."""
    import torch
    from gsx import sor
    xyz = _f32(np.array(mixed_cloud()) + np.float32(offset))
    x = torch.from_numpy(np.array(xyz)).to(cuda)
    for k in range(1, 64):
        want = oracle.sor_ckdtree_mean_dists(xyz, k)
        _assert_bits(sor.ckdtree_mean_dists(x, k).cpu().numpy(), want, f"ckdtree k={k} offset={offset}")


@pytest.mark.gpu
def test_ckdtree_crafted_pairwise_rows(cuda, gsx_lib):
    import torch
    from gsx import GsxError, sor
    xyz, rows = crafted_pairwise_rows()
    x = torch.from_numpy(np.array(xyz)).to(cuda)
    for k in range(1, 64):
        want = oracle.sor_ckdtree_mean_dists(xyz, k)
        _assert_bits(sor.ckdtree_mean_dists(x, k).cpu().numpy(), want, f"crafted k={k}")
    for bad in (0, 64):
        with pytest.raises(GsxError):
            sor.ckdtree_mean_dists(x, bad)

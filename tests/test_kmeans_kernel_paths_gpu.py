"""The K-Means kernels path by path: every assign form and centroid block, both update forms, tile and problem edges,
ties, sentinels and subnormal rows, each on data built to reach that path at the shipped constants.

Every case is a builder (a plain function returning float32 X, the row offsets and an init [nprob, K, D]) and two
kinds of test:
  * an unmarked CPU test restating the dispatch of `kmeans_lloyd` / `launch_tc_n` (kernel, points per thread and tile
    rows, wgmma column blocks NB, sorted or label-scan update, shared-memory opt-in) and asserting that the case
    reaches the branch it is meant for, plus any property of the data the case relies on (summation order, exact and
    near ties, the subnormal flush argument), checked with NumPy;
  * a `gpu` test running each applicable assign mode through `gsx.kmeans` and asserting labels, counts and centroids
    bit-equal to `oracle.kmeans_lloyd`, per problem; the tensor-core mode also checks its `want_stats` counters.

Constants these cases are built around (csrc/gsx_kmeans.cu, csrc/gsx_kmeans_tc.cu): strict assign 128 threads x P
points (P = 4 for D <= 4, 2 for D in {9, 24, 45}; any other D runs the generic one-point-per-thread kernel), centroids
staged 64 at a time and scored in pairs (an odd tail pairs with a zero row); the tensor-core kernel takes 128-row
tiles, D in {9, 24, 45} and K <= 256, in NB = 1, 2 or 4 blocks of 64 columns whose padding columns get the bias -3e38,
and bulk-copies a tile only when X is 16-byte aligned and the rounded copy stays inside X; the update partitions
1 024-row sub-tiles by label for K <= 2047 (per-warp counters of 8 (K+1) ints, opted in above 48 KiB) and scans labels
per cluster above that; `k_km_accum` adds 32-row batches, then a ragged tail; strict '<', lowest index on ties, 1e20
"no label" sentinel, empty clusters collapse to 0.
"""
import functools

import numpy as np
import pytest

import oracle

F32 = np.float32
TC_KP = {9: 16, 24: 32, 45: 48}          # D -> padded K of the wgmma operands (D + 3 bias columns, multiple of 8)
FIXED_D = (1, 2, 3, 4, 9, 24, 45)         # instantiations of k_kmeans_assign
THREADS, CENT_TILE, TC_ROWS, TC_MAX_K, SUB_TILE, MAX_SORT_K = 128, 64, 128, 256, 1024, 2047
FLT_MIN = 2.0 ** -126


# ------------------------------------------------------------------------------------------------ dispatch, restated
def tc_supported(K, D):
    return D in TC_KP and 1 <= K <= TC_MAX_K


def dispatch(mode, K, D):
    """What `kmeans_lloyd` launches for one Lloyd iteration."""
    if mode == "tensor" or (mode == "auto" and tc_supported(K, D)):
        kernel, P, tile = "tc", None, TC_ROWS
        nb = 1 if K <= 64 else 2 if K <= 128 else 4
    elif D in FIXED_D:
        P = 4 if D <= 4 else 2
        kernel, tile, nb = "strict", THREADS * P, None
    else:
        kernel, P, tile, nb = "generic", 1, THREADS, None
    sorted_update = K <= MAX_SORT_K
    return dict(kernel=kernel, P=P, tile=tile, nb=nb, update="sorted" if sorted_update else "scan",
                optin=sorted_update and 8 * (K + 1) * 4 > 48 * 1024)


def modes_for(K, D):
    return ("strict", "auto") + (("tensor",) if tc_supported(K, D) else ())


def tc_bulk_tiles(n_floats_before, offs, D, x_aligned=True):
    """`geo()` of the tensor-core kernel: for every 128-row tile, whether it is bulk-copied."""
    x_floats = n_floats_before + int(offs[-1]) * D
    out = []
    for p in range(len(offs) - 1):
        for r0 in range(int(offs[p]), int(offs[p + 1]), TC_ROWS):
            rows = min(TC_ROWS, int(offs[p + 1]) - r0)
            ob = (n_floats_before + r0 * D) * 4
            pre = ob & 15
            nbytes = (pre + rows * D * 4 + 15) & ~15
            out.append(x_aligned and (ob - pre) + nbytes <= x_floats * 4)
    return out


# ------------------------------------------------------------------------------------------------ numeric helpers
def _f32(a):
    a = np.ascontiguousarray(a, dtype=F32)
    a.setflags(write=False)
    return a


def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _strict_dist(X, C):
    """The contract's distance in float32: ((0 + d0^2) + d1^2) + ..., no fma."""
    acc = np.zeros((len(X), len(C)), F32)
    for d in range(X.shape[1]):
        df = X[:, None, d] - C[None, :, d]
        acc = acc + df * df
    return acc


def _tf32(a, rounding):
    u = np.ascontiguousarray(a, dtype=F32).view(np.uint32).astype(np.uint64)
    if rounding == "rne":
        u = u + 0xFFF + ((u >> 13) & 1)
    return (u & 0xFFFFE000).astype(np.uint32).view(F32)


def _tf32_scores(X, C, rounding):
    """Float64 score x.c - ||c||^2/2 with both operands converted to TF32 and the bias the kernel builds."""
    cn = (C.astype(np.float64) ** 2).sum(1).astype(F32)
    bias = (F32(-0.5) * cn).astype(np.float64)
    return _tf32(X, rounding).astype(np.float64) @ _tf32(C, rounding).astype(np.float64).T + bias[None]


def _spread(rng, shape, lo=-6, hi=0):
    """Random signs times magnitudes spread over the binades 2^lo .. 2^hi: float32 sums depend on their order."""
    return rng.choice([-1.0, 1.0], shape) * 2.0 ** rng.uniform(lo, hi, shape)


def _offs(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def _init_from_rows(X, offs, K, rng, replace=False):
    return np.stack([X[offs[p]:offs[p + 1]][rng.choice(offs[p + 1] - offs[p], K, replace=replace)]
                     for p in range(len(offs) - 1)])


def _case(X, offs, init):
    X, init = _f32(X), _f32(init)
    offs = np.asarray(offs, np.int64)
    assert init.ndim == 3 and init.shape[0] == len(offs) - 1 and init.shape[2] == X.shape[1]
    assert (np.diff(offs) > init.shape[1]).all(), "every problem needs more rows than K (the oracle passes k >= n through)"
    return X, offs, init


# ------------------------------------------------------------------------------------------------ builders
@functools.lru_cache(None)
def clustered(n, D, K, seed, nprob=1):
    """Prototype blobs with per-row noise over several binades; init = K distinct rows of each problem."""
    rng = np.random.default_rng(seed)
    proto = rng.normal(0.0, 1.0, (max(2 * K, 16), D))
    X = proto[rng.integers(0, len(proto), n * nprob)] + 0.05 * _spread(rng, (n * nprob, D))
    offs = _offs([n] * nprob)
    return _case(X, offs, _init_from_rows(X.astype(F32), offs, K, rng))


@functools.lru_cache(None)
def far_centroids(n, D, K, seed):
    """Points near the origin, every centroid at distance >= 10: every real tensor-core score is negative, and the
    origin (a zero row) is nearer to every point than any centroid is."""
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 0.1, (n, D))
    dirs = rng.normal(0.0, 1.0, (K, D))
    init = dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * rng.uniform(10.0, 12.0, (K, 1))
    return _case(X, [0, n], init[None])


def _far_holds(X, init):
    X64, C64 = X.astype(np.float64), init[0].astype(np.float64)
    scores = X64 @ C64.T - 0.5 * (C64 ** 2).sum(1)[None]
    origin = (X64 ** 2).sum(1)
    return scores.max() < 0 and (origin[:, None] < _strict_dist(X, init[0])).all()


CLUSTER_SIZES = (0, 1, 31, 32, 33, 64, 65, 1024, 1025)


@functools.lru_cache(None)
def cluster_sizes(D):
    """Exactly CLUSTER_SIZES rows in the clusters 0..8, shuffled, each cluster 1e4 apart along dim 0; the init is the
    cluster centres, so every Lloyd iteration keeps these members.  Noise over 2^-4 .. 2^6 makes the sums order-bound."""
    rng = np.random.default_rng(40 + D)
    K = len(CLUSTER_SIZES)
    centres = np.zeros((K, D))
    centres[:, 0] = 1e4 * (np.arange(K) + 1)
    lab = np.repeat(np.arange(K), CLUSTER_SIZES)
    rng.shuffle(lab)
    X = centres[lab] + _spread(rng, (len(lab), D), -4, 6)
    return _case(X, [0, len(X)], centres[None])


@functools.lru_cache(None)
def one_cluster(D):
    """200 000 rows, K = 1: every row joins cluster 0 (196 sub-tiles, 6 250 full batches)."""
    rng = np.random.default_rng(50 + D)
    X = 3.0 + _spread(rng, (200_000, D), -8, 4)
    return _case(X, [0, len(X)], X[:1][None])


EDGE_K = 17
EDGE_ROWS = (EDGE_K + 1, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 2049)


@functools.lru_cache(None)
def problem_edges(D):
    """One batched launch whose problems have rows around every tile size (128, 256, 512, the 1 024-row sub-tile)."""
    rng = np.random.default_rng(60 + D)
    offs = _offs(EDGE_ROWS)
    proto = rng.normal(0.0, 1.0, (64, D))
    X = (proto[rng.integers(0, 64, offs[-1])] + 0.1 * _spread(rng, (offs[-1], D))).astype(F32)
    return _case(X, offs, _init_from_rows(X, offs, EDGE_K, rng))


# the shapes the SOG writer asks for: (name, rows per problem, K, D, iterations)
PRODUCT = {
    "n10k_k911": ([1112] * 8 + [1104], 911, 45, 10),
    "n3k_k1024": ([1500] * 2, 1024, 45, 2),
    "c64_k64_d45": ([1000] * 64, 64, 45, 2),
    "c64_k256_d45": ([1000] * 64, 256, 45, 2),
    "c64_k64_d9": ([1000] * 64, 64, 9, 2),
    "c64_k256_d9": ([1000] * 64, 256, 9, 2),
    "crossing_64x2000": ([2000] * 64, 64, 45, 2),
}


@functools.lru_cache(None)
def product_shape(name):
    sizes, K, D, _ = PRODUCT[name]
    rng = np.random.default_rng(140 + sorted(PRODUCT).index(name))
    offs = _offs(sizes)
    proto = rng.normal(0.0, 0.15, (1024, D))
    noisy = rng.random((offs[-1], 1)) < 0.6                                # the other rows repeat a prototype exactly
    X = (proto[rng.integers(0, 1024, offs[-1])] + 0.03 * rng.normal(0.0, 1.0, (offs[-1], D)) * noisy).astype(F32)
    return _case(X, offs, _init_from_rows(X, offs, K, rng))


@functools.lru_cache(None)
def lattice_ties(D):
    """64 centroids on a spacing-4 grid in dims 0, 1; points on grid nodes, edge midpoints and cell centres (1, 2 and 4
    exactly equidistant centroids) with the same small integers in the other dims: every distance and every TF32
    score is exact, so the ties are exact."""
    rng = np.random.default_rng(70 + D)
    C = np.zeros((64, D))
    C[:, 0], C[:, 1] = 4 * (np.arange(64) // 8), 4 * (np.arange(64) % 8)
    base = rng.integers(0, 64, 3000)
    step = np.array([[0, 0], [2, 0], [0, 2], [2, 2], [2, 2]])[rng.integers(0, 5, 3000)]
    X = np.zeros((3000, D))
    X[:, :2] = C[base, :2] + step
    X[:, 2:] = rng.integers(-1, 2, (3000, D - 2)) if D > 2 else 0
    return _case(X, [0, 3000], C[None])


DUP_PAIRS = ((0, 2), (5, 7), (13, 15), (22, 24), (30, 32), (41, 43), (61, 63))


@functools.lru_cache(None)
def duplicate_centroids(D):
    """Clustered data, K = 64, centroid c + 2 a copy of centroid c: the tie falls in another lane of the quad."""
    X, offs, init = clustered(4000, D, 64, 80 + D)
    init = init.copy()
    for a, b in DUP_PAIRS:
        init[0, b] = init[0, a]
    return _case(X, offs, init)


@functools.lru_cache(None)
def collapse_ties(D):
    """40 distinct rows (5 of them near the origin) repeated 15 times; K = 64 drawn with replacement from the 35 far
    rows.  After the first update most clusters are empty and collapse to 0, and the near-origin rows then tie
    between all those zero centroids."""
    rng = np.random.default_rng(90 + D)
    far = rng.normal(0.0, 1.0, (35, D)) + 3.0
    near = rng.normal(0.0, 0.01, (5, D))
    distinct = np.r_[far, near]
    X = distinct[rng.permutation(np.repeat(np.arange(40), 15))]
    return _case(X, [0, len(X)], far[rng.integers(0, 35, 64)][None])


@functools.lru_cache(None)
def near_ties(D):
    """Crafted rows: 16 centroid pairs 1e-3 apart and rows near them, kept (seeded search) only where the strict
    winner scores below the best TF32 score under both truncation and round-to-nearest, by more than the float32
    accumulation error -- a zero margin would drop the true answer."""
    rng = np.random.default_rng(100 + D)
    base = rng.normal(0.0, 1.0, (16, D))
    C = np.empty((32, D))
    C[0::2], C[1::2] = base, base + rng.normal(0.0, 1e-3, (16, D))
    C = C.astype(F32)
    kept = []
    while sum(map(len, kept)) < 600:
        cand = (base[rng.integers(0, 16, 4096)] + rng.normal(0.0, 0.02, (4096, D))).astype(F32)
        win = _strict_dist(cand, C).argmin(1)
        ok = np.ones(len(cand), bool)
        for rounding in ("trunc", "rne"):
            s = _tf32_scores(cand, C, rounding)
            tol = 8 * D * 2.0 ** -24 * (np.abs(cand).astype(np.float64) @ np.abs(C).astype(np.float64).T).max(1)
            ok &= s.max(1) - s[np.arange(len(cand)), win] > tol
        kept.append(cand[ok])
    X = np.concatenate(kept)[:600]
    fill = (base[rng.integers(0, 16, 1400)] + rng.normal(0.0, 0.05, (1400, D))).astype(F32)
    X = np.r_[X, fill][rng.permutation(2000)]
    return _case(X, [0, 2000], C[None])


@functools.lru_cache(None)
def sentinels(D, K):
    """Rows whose strict distance is >= 1e20 (2e10 and 1e11 offsets), NaN or inf against every centroid: label -1,
    left out of counts and sums."""
    rng = np.random.default_rng(110 + D + K)
    n = max(3000, 2 * K + 500)
    X = rng.normal(0.0, 1.0, (n, D))
    bad = rng.choice(n, 80, replace=False)
    X[bad[:20], 0] = 2e10
    X[bad[20:40]] = rng.choice([-1e11, 1e11], (20, D))
    X[bad[40:60], rng.integers(0, D, 20)] = np.nan
    X[bad[60:], 0] = -np.inf
    good = np.setdiff1d(np.arange(n), bad)
    init = X[rng.choice(good, K, replace=False)]
    return _case(X, [0, n], init[None])


@functools.lru_cache(None)
def inf_centroid(D):
    X, offs, init = clustered(3000, D, 32, 120 + D)
    init = init.copy()
    init[0, 3, 0] = np.inf
    return _case(X, offs, init)


SUB = 2.0 ** -63


@functools.lru_cache(None)
def subnormal_rows(D):
    """300 rows x_k = 2^-63 and 84 zero rows; centroid A = 0, centroid B with c_k = 2^-63 (1 - 2^-10).  Every product
    x_k c_k is just below FLT_MIN: a tensor core that flushed them would score B at -||c||^2/2 instead of +||c||^2/2."""
    rng = np.random.default_rng(130 + D)
    X = np.r_[np.full((300, D), SUB), np.zeros((84, D))][rng.permutation(384)]
    init = np.stack([np.zeros(D), np.full(D, SUB * (1 - 2.0 ** -10))])
    return _case(X, [0, 384], init[None])


def _tc_threshold(x, C, flushed):
    """The tensor-core epilogue's candidate threshold smax - marg for one row, in float32 as the kernel evaluates it,
    with the scores exact or with every subnormal product flushed to zero."""
    D = len(x)
    u = 5.9604645e-8
    kGs, kEpsIn, kEpsAcc = F32(2 * (D + 3) * u * 1.02), F32(1.953125e-3 * 1.01), F32(3.0517578e-5)
    x64, C64 = x.astype(np.float64), C.astype(np.float64)
    prod = x64[None] * C64
    if flushed:
        prod = np.where(np.abs(prod) < FLT_MIN, 0.0, prod)
    scores = prod.sum(1) - 0.5 * (C64 ** 2).sum(1)
    smax = F32(scores.max())
    xnu = F32(F32((x64 ** 2).sum()) * F32(1.0001))
    xnorm = F32(np.sqrt(xnu) * F32(1.0001))
    Cm = F32(np.sqrt(F32((C64 ** 2).sum(1).max())) * F32(1.0001))
    eta = F32((kEpsIn * xnorm * Cm + kEpsAcc * (xnorm * Cm + Cm * Cm)) * F32(1.5) + F32(1e-37))
    e_ub = max(F32(xnu - F32(2) * smax + F32(2) * eta), F32(0))
    marg = F32(F32(2) * eta + kGs * e_ub)
    return scores, F32(smax - marg)


# ------------------------------------------------------------------------------------------------ GPU runner
@functools.lru_cache(None)
def _oracle(builder, args, iters):
    X, offs, init = builder(*args)
    return [oracle.kmeans_lloyd(X[offs[p]:offs[p + 1]], init.shape[1], iters, init=init[p]) for p in range(len(offs) - 1)]


def _check(builder, args, iters, cuda, modes=None, Xd=None, stats=None):
    """Run every mode on the GPU and compare with the oracle per problem.  `stats` maps a check name to a predicate
    over the tensor-core counters.  Returns the tensor-core counters (or None)."""
    import torch
    from gsx import kmeans as gk
    X, offs, init = builder(*args)
    K, D = init.shape[1], X.shape[1]
    want = _oracle(builder, args, iters)
    Xd = torch.from_numpy(np.array(X)).to(cuda) if Xd is None else Xd
    initd = torch.from_numpy(np.array(init)).to(cuda)
    tc_stats = None
    for mode in modes or modes_for(K, D):
        tc = mode == "tensor"
        out = gk.kmeans_lloyd_batched(Xd, offs, K, iters, initd, assign=mode, want_stats=tc)
        Cc, L, cnt = (t.cpu().numpy() for t in out[:3])
        for p, (Co, Lo, cnto) in enumerate(want):
            what = f"{builder.__name__}{args} iters={iters} mode={mode} problem={p}"
            lab = L[offs[p]:offs[p + 1]]
            bad = np.flatnonzero(lab != Lo)
            assert not len(bad), f"{what}: {len(bad)} labels differ, first rows {bad[:5]}: {lab[bad[:5]]} vs {Lo[bad[:5]]}"
            assert np.array_equal(cnt[p], cnto), f"{what}: counts differ"
            assert np.array_equal(_bits(Cc[p]), _bits(Co)), f"{what}: centroid bits differ"
        if tc:
            tc_stats = out[3]
            for name, pred in (stats or {"full_scans == 0": lambda s: s["full_scans"] == 0}).items():
                assert pred(tc_stats), f"{builder.__name__}{args}: tensor stats {tc_stats} fail {name}"
    return tc_stats


FULL_SCANS = {"full_scans > 0": lambda s: s["full_scans"] > 0}
TIES = {"multi_candidate_points > 0": lambda s: s["multi_candidate_points"] > 0,
        "full_scans == 0": lambda s: s["full_scans"] == 0}


# ================================================================================================ tensor K sweep
TC_KS = (1, 2, 31, 32, 33, 63, 64, 65, 96, 127, 128, 129, 160, 192, 193, 255, 256)


def tc_clustered(D, K):
    return clustered(20_000, D, K, 1000 * D + K)


def tc_far(D, K):
    return far_centroids(20_000, D, K, 2000 * D + K)


def test_tc_sweep_reaches_every_column_block():
    seen = set()
    for D in TC_KP:
        for K in TC_KS:
            d = dispatch("tensor", K, D)
            assert d["kernel"] == "tc" and dispatch("auto", K, D)["kernel"] == "tc"
            seen.add((d["nb"], d["nb"] * 64 > K))                       # (NB, has padding columns)
            assert TC_KP[D] >= D + 3 and TC_KP[D] % 8 == 0
    assert seen == {(1, True), (1, False), (2, True), (2, False), (4, True), (4, False)}


@pytest.mark.parametrize("D", sorted(TC_KP))
def test_far_geometry_scores_are_all_negative(D):
    for K in TC_KS:
        X, _, init = tc_far(D, K)
        assert _far_holds(X, init), (D, K)


@pytest.mark.gpu
@pytest.mark.parametrize("geometry", ["tc_clustered", "tc_far"])
@pytest.mark.parametrize("D", sorted(TC_KP))
def test_tc_k_sweep(D, geometry, cuda, gsx_lib):
    for K in TC_KS:
        _check(globals()[geometry], (D, K), 2, cuda)


# ================================================================================================ strict sweep
SWEEP_D = (1, 2, 3, 4, 9, 24, 45, 5, 7, 46, 64, 65, 100)
SWEEP_K = (1, 2, 3, 63, 64, 65, 127, 257)


def test_strict_fma_sweep_dispatch():
    kernels = {}
    for D in SWEEP_D:
        for K in SWEEP_K:
            s = dispatch("strict", K, D)
            kernels.setdefault(s["kernel"], set()).add(D)
            if D <= 4:
                assert s["kernel"] == "strict" and s["P"] == 4 and s["tile"] == 512
            elif D in TC_KP:
                assert s["kernel"] == "strict" and s["P"] == 2 and s["tile"] == 256
            else:
                assert s["kernel"] == "generic" and s["P"] == 1 and s["tile"] == 128
    assert kernels == {"strict": {1, 2, 3, 4, 9, 24, 45}, "generic": {5, 7, 46, 64, 65, 100}}
    assert max(kernels["generic"]) > 64                                  # a second 64-dim strip in the update
    assert {K % CENT_TILE for K in SWEEP_K if K % 2} >= {1, 3, 63}       # odd tails: pair with a zero row


@pytest.mark.parametrize("D", SWEEP_D)
def test_far_geometry_for_odd_k(D):
    for K in SWEEP_K:
        if K % 2:
            X, _, init = far_centroids(3001, D, K, 3000 * D + K)
            assert _far_holds(X, init), (D, K)


@pytest.mark.gpu
@pytest.mark.parametrize("D", SWEEP_D)
def test_strict_fma_sweep(D, cuda, gsx_lib):
    for K in SWEEP_K:
        _check(clustered, (3001, D, K, 4000 * D + K), 2, cuda, modes=("strict", "auto"))
        if K % 2:
            _check(far_centroids, (3001, D, K, 3000 * D + K), 1, cuda, modes=("strict", "auto"))


# ================================================================================================ update forms
UPDATE_KS = (255, 256, 511, 512, 1535, 1536, 2047, 2048)


def test_update_forms_dispatch():
    got = {K: (dispatch("strict", K, 3)["update"], dispatch("strict", K, 3)["optin"]) for K in UPDATE_KS}
    assert got == {255: ("sorted", False), 256: ("sorted", False), 511: ("sorted", False), 512: ("sorted", False),
                   1535: ("sorted", False), 1536: ("sorted", True), 2047: ("sorted", True), 2048: ("scan", False)}
    assert [(K + 1 + 255) // 256 for K in UPDATE_KS] == [1, 2, 2, 3, 6, 7, 8, 9]   # k_km_offsets strips: carries


@pytest.mark.gpu
@pytest.mark.parametrize("K", UPDATE_KS)
def test_update_forms(K, cuda, gsx_lib):
    _check(clustered, (20_000, 3, K, 5000 + K), 2, cuda, modes=("strict", "auto"))


# ================================================================================================ cluster sizes
def _serial(rows):
    s = np.zeros(rows.shape[1], F32)
    for r in rows:
        s = s + r
    return s


def _batch_reversed(rows):
    s = np.zeros(rows.shape[1], F32)
    full = len(rows) // 32 * 32
    for b in range(0, full, 32):
        for r in rows[b:b + 32][::-1]:
            s = s + r
    for r in rows[full:]:
        s = s + r
    return s


def _warp_reversed(idx):
    """Member order if the scatter ranked a lane after the higher lanes of its 32-row window."""
    return np.concatenate([w[::-1] for w in np.split(idx, np.flatnonzero(np.diff(idx // 32)) + 1)])


def test_cluster_sizes_are_exact_and_order_sensitive(gsx_lib):
    X, _, init = cluster_sizes(45)
    _, L, cnt = _oracle(cluster_sizes, (45,), 2)[0]
    assert tuple(cnt) == CLUSTER_SIZES and (L >= 0).all()
    assert {s % 32 for s in CLUSTER_SIZES} == {0, 1, 31}                  # batches only, and ragged tails of 1, 31
    for c, size in enumerate(CLUSTER_SIZES):
        if size < 31:
            continue
        idx = np.flatnonzero(L == c)
        rows = X[idx]
        inv = F32(1) / F32(size)
        mean = _serial(rows) * inv
        others = {"reversed": _serial(rows[::-1]), "pairwise": np.ascontiguousarray(rows.T).sum(axis=1, dtype=F32)}
        if size >= 32:
            others.update(batch_reversed=_batch_reversed(rows), warp_reversed=_serial(X[_warp_reversed(idx)]))
        for name, other in others.items():
            assert (_bits(mean) != _bits(other * inv)).any(), (c, size, name)
    X1, _, _ = one_cluster(3)
    assert (_bits(_serial(X1)) != _bits(np.ascontiguousarray(X1.T).sum(axis=1, dtype=F32))).any()


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 45, 100])
def test_cluster_sizes(D, cuda, gsx_lib):
    _check(cluster_sizes, (D,), 2, cuda)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 45])
def test_one_cluster_of_200k_rows(D, cuda, gsx_lib):
    _check(one_cluster, (D,), 2, cuda)


# ================================================================================================ problem edges
def test_problem_edges_straddle_every_tile():
    tiles = {dispatch("strict", EDGE_K, 3)["tile"], dispatch("strict", EDGE_K, 45)["tile"],
             dispatch("tensor", EDGE_K, 45)["tile"], dispatch("strict", EDGE_K, 7)["tile"], SUB_TILE}
    assert tiles == {512, 256, 128, 1024}
    assert dispatch("strict", EDGE_K, 3)["P"] == 4 and dispatch("strict", EDGE_K, 45)["P"] == 2
    assert dispatch("strict", EDGE_K, 7)["kernel"] == "generic"
    for t in tiles:
        assert {t - 1, t, t + 1} <= set(EDGE_ROWS), t
    assert len(EDGE_ROWS) <= 64 and min(EDGE_ROWS) == EDGE_K + 1 and max(EDGE_ROWS) > 2 * SUB_TILE


def test_tc_ctas_cross_problems():
    sizes = PRODUCT["crossing_64x2000"][0]
    tile0 = np.concatenate([[0], np.cumsum([(s + 127) // 128 for s in sizes])])
    total = int(tile0[-1])
    for grid in (132, 264):                                              # one or two resident CTAs per H100 SM
        crossing = 0
        for b in range(grid):
            t0, t1 = total * b // grid, total * (b + 1) // grid
            crossing += np.searchsorted(tile0, t0, "right") != np.searchsorted(tile0, t1 - 1, "right")
        assert crossing > 10, grid


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 45, 7])
def test_problem_edges(D, cuda, gsx_lib):
    _check(problem_edges, (D,), 2, cuda)


# ================================================================================================ product shapes
def test_product_shapes_collapse_and_tie(gsx_lib):
    X, offs, init = product_shape("n10k_k911")
    assert len(offs) == 10 and offs[-1] == 10_000 and (np.diff(offs)[:-1] == 1112).all() and offs[-1] - offs[-2] == 1104
    C9 = _oracle(product_shape, ("n10k_k911",), 9)
    assert all(((C == 0).all(1)).sum() >= 2 for C, _, _ in C9)           # several empty clusters collapsed to 0 ...
    assert all((cnt == 1).sum() >= 50 for _, _, cnt in C9)               # ... next to many singletons
    assert dispatch("auto", 911, 45)["kernel"] == "strict" and dispatch("auto", 1024, 45)["update"] == "sorted"
    assert dispatch("auto", 256, 9)["nb"] == 4 and dispatch("auto", 64, 45)["nb"] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PRODUCT))
def test_product_shapes(name, cuda, gsx_lib):
    _check(product_shape, (name,), PRODUCT[name][3], cuda)


# ================================================================================================ alignment
ALIGN_N = 1001


def test_alignment_reaches_the_non_bulk_load():
    for D in TC_KP:
        bulk = tc_bulk_tiles(0, [0, ALIGN_N], D)
        if D == 24:                                                      # 96-byte rows: every tile is aligned
            assert (ALIGN_N * D * 4) % 16 == 0 and all(bulk)
        else:                                                            # only the last tile falls back
            assert (ALIGN_N * D * 4) % 16 and all(bulk[:-1]) and not bulk[-1], D
        assert not any(tc_bulk_tiles(1, [0, ALIGN_N], D, x_aligned=False))


@pytest.mark.gpu
@pytest.mark.parametrize("D", sorted(TC_KP))
def test_alignment(D, cuda, gsx_lib):
    import torch
    args = (ALIGN_N, D, 32, 6000 + D)
    X, _, _ = clustered(*args)
    _check(clustered, args, 2, cuda)                                     # aligned X, ragged end of the buffer
    buf = torch.zeros(X.size + 1, dtype=torch.float32, device=cuda)
    buf[1:] = torch.from_numpy(np.array(X)).reshape(-1).to(cuda)
    view = buf[1:].view(ALIGN_N, D)
    assert view.is_contiguous() and view.data_ptr() % 16 == 4
    _check(clustered, args, 2, cuda, Xd=view)                            # X at storage offset 1 float


# ================================================================================================ ties and collapse
def _tie_rows(X, C):
    d = _strict_dist(X, C)
    return d == d.min(1, keepdims=True)


def test_lattice_ties_are_exact():
    for D in (3, 9, 45):
        X, _, init = lattice_ties(D)
        tie = _tie_rows(X, init[0])
        assert (tie.sum(1) == 2).sum() > 500 and (tie.sum(1) == 4).sum() > 500, D
        lanes = [{(c % 64 % 8) // 2 for c in np.flatnonzero(r)} for r in tie[tie.sum(1) > 1][:200]]
        assert any(len(s) > 1 for s in lanes)                            # ties across quad lanes ...
        assert any(len(s) == 1 for s in lanes)                           # ... and inside one thread
        for rounding in ("trunc", "rne"):                                # the TF32 scores tie exactly too
            s = _tf32_scores(X, init[0], rounding)
            assert ((s == s.max(1, keepdims=True)) == tie).all()


def test_duplicate_centroids_tie_across_quad_lanes():
    for D in (3, 9, 45):
        X, _, init = duplicate_centroids(D)
        win = _strict_dist(X, init[0]).argmin(1)
        for a, b in DUP_PAIRS:
            assert (a % 8) // 2 != (b % 8) // 2 and (init[0, a] == init[0, b]).all()
            assert (win == a).sum() >= 5, (D, a)                          # the lower copy wins real rows


def test_collapse_ties_between_zero_centroids(gsx_lib):
    for D in (3, 9, 45):
        X, _, init = collapse_ties(D)
        C1, _, cnt1 = _oracle(collapse_ties, (D,), 1)[0]
        zero = (C1 == 0).all(1)
        assert zero.sum() >= 10 and (cnt1[zero] == 0).all()
        tie = _tie_rows(X, C1)
        assert (tie[:, zero].sum(1) >= 2).sum() >= 75, D                 # every near-origin row ties between zeros


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 9, 45])
@pytest.mark.parametrize("case,iters", [("lattice_ties", 2), ("duplicate_centroids", 2), ("collapse_ties", 4)])
def test_ties(case, iters, D, cuda, gsx_lib):
    _check(globals()[case], (D,), iters, cuda, stats=TIES)


# ================================================================================================ near ties
@pytest.mark.parametrize("D", sorted(TC_KP))
def test_near_ties_need_the_margin(D):
    X, _, init = near_ties(D)
    C = init[0]
    win = _strict_dist(X, C).argmin(1)
    for rounding in ("trunc", "rne"):
        s = _tf32_scores(X, C, rounding)
        assert (s[np.arange(len(X)), win] < s.max(1)).sum() >= 600, rounding


@pytest.mark.gpu
@pytest.mark.parametrize("D", sorted(TC_KP))
def test_near_ties(D, cuda, gsx_lib):
    _check(near_ties, (D,), 1, cuda, stats=TIES)
    _check(near_ties, (D,), 3, cuda)


# ================================================================================================ sentinels
SENTINEL_CASES = [(3, 32), (3, 2048), (45, 32)]


def test_sentinel_rows_get_no_label(gsx_lib):
    for D, K in SENTINEL_CASES:
        X, _, init = sentinels(D, K)
        bad = ~np.isfinite(X).all(1) | (np.abs(X) >= 1e10).any(1)
        _, L, cnt = _oracle(sentinels, (D, K), 2)[0]
        assert bad.sum() == 80 and (L[bad] == -1).all() and (L[~bad] >= 0).all()
        assert cnt.sum() == len(X) - 80
        assert dispatch("strict", K, D)["update"] == ("scan" if K > MAX_SORT_K else "sorted")


@pytest.mark.gpu
@pytest.mark.parametrize("D,K", SENTINEL_CASES)
def test_sentinels(D, K, cuda, gsx_lib):
    _check(sentinels, (D, K), 2, cuda, stats=FULL_SCANS)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 45])
def test_inf_centroid(D, cuda, gsx_lib):
    C1, _, cnt1 = _oracle(inf_centroid, (D,), 1)[0]
    assert cnt1[3] == 0 and (C1[3] == 0).all()                          # the inf centroid wins nothing, then collapses
    _check(inf_centroid, (D,), 2, cuda, stats=FULL_SCANS)


# ================================================================================================ subnormal rows
@pytest.mark.parametrize("D", sorted(TC_KP))
def test_subnormal_flush_argument(D, gsx_lib):
    X, _, init = subnormal_rows(D)
    C = init[0]
    x = X[(X != 0).any(1)][0]
    assert (x.astype(np.float64)[None] * C[1].astype(np.float64) < FLT_MIN).all()      # every product subnormal
    assert (x.astype(np.float64) ** 2 >= FLT_MIN).all() and (C[1] ** 2 > 0).all()
    dist = _strict_dist(x[None], C)[0]
    assert dist[1] < dist[0] and dist[1] > 0                              # the contract picks B
    _, L, _ = _oracle(subnormal_rows, (D,), 1)[0]
    assert (L == np.where((X != 0).any(1), 1, 0)).all()
    exact, thr = _tc_threshold(x, C, flushed=False)
    flushed, thr_f = _tc_threshold(x, C, flushed=True)
    assert exact[1] > 0 and exact[1] >= thr and flushed[1] < 0 == flushed[0]
    if D == 45:
        assert thr > exact[0]                                             # exact scores: B is the only candidate
        assert flushed[1] < thr_f                                         # a flush would drop B and answer A
    else:                                                                 # the 1e-37 slack keeps both candidates,
        assert thr <= exact[0] and flushed[1] >= thr_f                    # flushed or not: the strict scan decides


@pytest.mark.gpu
@pytest.mark.parametrize("D", sorted(TC_KP))
def test_subnormal_rows(D, cuda, gsx_lib):
    """On an H100 the wgmma TF32 product keeps subnormal x_k c_k: B scores +||c||^2/2, not the flushed -||c||^2/2."""
    import torch
    from gsx import kmeans as gk
    X, _, init = subnormal_rows(D)
    S = gk.tc_debug_scores(torch.from_numpy(np.array(X)).to(cuda), torch.from_numpy(np.array(init[0])).to(cuda))
    S = S.cpu().numpy()[:, :2]
    assert (S[:, 0] == 0).all() and np.array_equal(S[:, 1] > 0, (X[:128] != 0).any(1)), S[:4]
    _check(subnormal_rows, (D,), 1, cuda)
    _check(subnormal_rows, (D,), 2, cuda)


# ================================================================================================ API edges
def test_only_auto_strict_tensor_are_assign_modes(gsx_lib):
    """AUTO (0), STRICT (1) and TENSOR (3) are the assign modes; any other value is GSX_ERR_ARG (-2), checked before
    the shape, the workspace or the device."""
    import ctypes as C
    off = (C.c_int64 * 2)(0, 1000)
    for mode in (-1, 2, 4, 5):
        assert gsx_lib.gsx_kmeans_lloyd_device(None, off, 1, 32, 45, 1, None, None, None, None, 0, mode, None,
                                               None) == -2, mode


@pytest.mark.gpu
def test_max_iter_zero_returns_init(cuda, gsx_lib):
    import torch
    from gsx import kmeans as gk
    X, offs, init = clustered(1000, 45, 32, 7000)
    for mode in modes_for(32, 45):
        Cc, L, cnt = gk.kmeans_lloyd_batched(torch.from_numpy(np.array(X)).to(cuda), offs, 32, 0,
                                             torch.from_numpy(np.array(init)).to(cuda), assign=mode)
        assert np.array_equal(_bits(Cc.cpu().numpy()), _bits(init)) and not cnt.any(), mode


@pytest.mark.gpu
@pytest.mark.parametrize("K,D", [(257, 45), (32, 10)])
def test_tensor_rejects_unsupported_shapes(K, D, cuda, gsx_lib):
    import torch
    from gsx import GsxError, kmeans as gk
    X, _, init = clustered(1000, D, K, 7100 + D)
    with pytest.raises(GsxError):
        gk.kmeans_lloyd(torch.from_numpy(np.array(X)).to(cuda), K, 1, torch.from_numpy(np.array(init[0])).to(cuda),
                        assign="tensor")

"""GPU: the wgmma (tensor-core) K-Means assign -- score GEMM in registers, candidate margin, strict re-evaluation.
Labels / counts / centroids bit-identical to the oracle and to the strict CUDA-core kernel at the C3 chunk size
(SURVEY 8(d): one full 781 250 x 45 chunk vs the oracle, all-chunk run-to-run determinism), on SH-like shapes and on
adversarial near-tie inputs that exercise the candidate margin and its fallbacks."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _tf32(a):
    return (a.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


# every (D, NB) instantiation of k_km_assign_tc: NB = 1, 2, 4 column blocks for K <= 64, 128, 256
@pytest.mark.parametrize("D,K", [(45, 256), (45, 50), (24, 100), (9, 16), (45, 128), (24, 33), (24, 256), (9, 65),
                                 (9, 193)])
def test_tc_scores_are_the_gemm(D, K, cuda, gsx_lib):
    """The accumulator holds x.c - ||c||^2/2 (layout / descriptor check) within the input-conversion error the
    margin assumes: kind::tf32, 2^-10 per operand."""
    import torch
    from gsx import kmeans as gk
    rng = np.random.default_rng(D * 1000 + K)
    X = rng.normal(0, 0.15, (128, D)).astype(np.float32)
    C = rng.normal(0, 0.15, (K, D)).astype(np.float32)
    S = gk.tc_debug_scores(torch.from_numpy(X).to(cuda), torch.from_numpy(C).to(cuda)).cpu().numpy()[:, :K]
    exact = X.astype(np.float64) @ C.astype(np.float64).T - 0.5 * (C.astype(np.float64) ** 2).sum(1)[None]
    bound = 2.0 ** -9 * (np.linalg.norm(X, axis=1)[:, None] * np.linalg.norm(C, axis=1)[None] + 0.5 * (C ** 2).sum(1)[None]) + 1e-7
    assert np.all(np.abs(S - exact) <= bound), float(np.abs(S - exact).max())


def test_tc_full_c3_chunk_matches_oracle(cuda, gsx_lib):
    """One full SOG chunk of the 50 M-splat config: 781 250 x 45, K=256, injected init, 2 Lloyd iterations."""
    import torch
    import oracle
    from gsx import kmeans as gk
    n, D, K = 781_250, 45, 256
    rng = np.random.default_rng(7)
    proto = rng.normal(0, 0.15, (1024, D)).astype(np.float32)
    X = (proto[rng.integers(0, 1024, n)] + rng.normal(0, 0.03, (n, D))).astype(np.float32)
    init = X[rng.choice(n, K, replace=False)].copy()
    Co, Lo, cnto = oracle.kmeans_lloyd(X, K, 2, init=init)
    Xd, initd = torch.from_numpy(X).to(cuda), torch.from_numpy(init).to(cuda)
    Cc, L, cnt, st = gk.kmeans_lloyd_batched(Xd, [0, n], K, 2, initd.reshape(1, K, D), assign="tensor", want_stats=True)
    assert np.array_equal(L.cpu().numpy(), Lo)
    assert np.array_equal(cnt[0].cpu().numpy(), cnto)
    assert np.allclose(Cc[0].cpu().numpy(), Co, rtol=1e-5, atol=0)
    assert np.array_equal(Cc[0].cpu().numpy().view(np.uint32), Co.view(np.uint32))
    assert st["full_scans"] == 0 and st["strict_evals"] < 2 * 2 * n  # the margin leaves ~1 candidate per point


def test_tc_all_chunks_deterministic_and_equal_to_strict(cuda, gsx_lib):
    """16 chunks x 200 000 rows in one launch: run-to-run determinism and tensor == strict, bit for bit."""
    import torch
    from gsx import kmeans as gk
    nprob, rows, D, K = 16, 200_000, 45, 256
    g = torch.Generator(device=cuda).manual_seed(5)
    proto = torch.randn(1024, D, device=cuda, generator=g) * 0.15
    X = proto[torch.randint(0, 1024, (nprob * rows,), device=cuda, generator=g)] + \
        0.03 * torch.randn(nprob * rows, D, device=cuda, generator=g)
    offs = [p * rows for p in range(nprob + 1)]
    init = torch.stack([X[offs[p]:offs[p] + K] for p in range(nprob)])
    tc = gk.kmeans_lloyd_batched(X, offs, K, 3, init, assign="tensor")
    again = gk.kmeans_lloyd_batched(X, offs, K, 3, init, assign="tensor")
    strict = gk.kmeans_lloyd_batched(X, offs, K, 3, init, assign="strict")
    for a, b in zip(tc, again):
        assert torch.equal(a, b)
    assert torch.equal(tc[1], strict[1])
    assert torch.equal(tc[0].view(torch.int32), strict[0].view(torch.int32))
    assert torch.equal(tc[2], strict[2])


def test_tc_ragged_rows_and_unaligned_chunks(cuda, gsx_lib):
    """Chunk starts that are not 16-byte aligned, partial last tiles, K not a multiple of 32, tiny problems."""
    import torch
    import oracle
    from gsx import kmeans as gk, synth
    X = np.ascontiguousarray(synth.attributes(40_000)["f_rest"])
    offs = [0, 47, 176, 7_001, 16_002, 16_131, 40_000]   # K=45 < rows everywhere (k >= N is the dispatcher's passthrough)
    K = 45
    rng = np.random.default_rng(3)
    nprob = len(offs) - 1
    init = np.stack([X[offs[p]:offs[p + 1]][rng.choice(offs[p + 1] - offs[p], K, replace=True)] for p in range(nprob)])
    Cc, L, cnt = gk.kmeans_lloyd_batched(torch.from_numpy(X).to(cuda), offs, K, 3, torch.from_numpy(init).to(cuda),
                                         assign="tensor")
    for p in range(nprob):
        Co, Lo, cnto = oracle.kmeans_lloyd(X[offs[p]:offs[p + 1]], K, 3, init=init[p])
        assert np.array_equal(L[offs[p]:offs[p + 1]].cpu().numpy(), Lo), p
        assert np.array_equal(Cc[p].cpu().numpy().view(np.uint32), Co.view(np.uint32)), p


def test_tc_nan_inf_inputs_follow_the_contract(cuda, gsx_lib):
    import torch
    import oracle
    from gsx import kmeans as gk
    rng = np.random.default_rng(11)
    X = rng.normal(0, 0.15, (3000, 45)).astype(np.float32)
    X[5, 3] = np.nan
    X[77, 0] = np.inf
    X[100] *= np.float32(1e19)
    init = X[rng.choice(3000, 32, replace=False)].copy()
    init[0] = X[200]
    Co, Lo, cnto = oracle.kmeans_lloyd(X, 32, 1, init=init)
    Cc, L, cnt = gk.kmeans_lloyd(torch.from_numpy(X).to(cuda), 32, 1, torch.from_numpy(init).to(cuda), assign="tensor")
    assert np.array_equal(L.cpu().numpy(), Lo)


def _check_oracle(X, k, it, cuda, mode, seed=1234):
    import torch
    import oracle
    from gsx import kmeans as gk
    np.random.seed(seed)
    init = oracle.kmeans_reference_init(X, k)
    Co, Lo, cnto = oracle.kmeans_lloyd(X, k, it, init=init)
    C, L, cnt = gk.kmeans_lloyd(torch.from_numpy(X).to(cuda), k, it, torch.from_numpy(init).to(cuda), assign=mode)
    assert np.array_equal(L.cpu().numpy(), Lo)
    assert np.array_equal(cnt.cpu().numpy(), cnto)
    assert np.array_equal(C.cpu().numpy().view(np.uint32), Co.view(np.uint32))


# K = 300 is beyond the tensor-core path: "auto" runs the strict kernel there
@pytest.mark.parametrize("n,d,k,it,mode", [(100_000, 45, 256, 3, "tensor"), (20_000, 45, 64, 5, "tensor"),
                                           (10_000, 24, 100, 3, "tensor"), (10_000, 9, 16, 10, "tensor"),
                                           (4_000, 45, 300, 2, "auto")])
def test_tc_matches_oracle(n, d, k, it, mode, cuda, gsx_lib):
    from gsx import synth
    X = np.ascontiguousarray(synth.attributes(n)["f_rest"][:, :d])
    _check_oracle(X, k, it, cuda, mode)


def _adversarial(case):
    rng = np.random.default_rng(0)
    base = rng.normal(0, 0.15, (3000, 45)).astype(np.float32)
    Xg = rng.integers(-2, 3, (5000, 9)).astype(np.float32)
    return {
        # many exactly duplicated rows: the init draws duplicate centroids, so rows tie exactly between them
        "duplicate_rows": (np.repeat(base[:150], 20, axis=0), 64, 3, 3),
        # large common offset: heavy cancellation in ||x||^2 - 2 x.c + ||c||^2
        "offset_100": (base + np.float32(100.0), 50, 3, 1234),
        # lattice: exact distance ties between different centroids (lowest index must win)
        "lattice_ties": (Xg, 40, 4, 1234),
        # distances around the 1e20 start value (label -1 rows are skipped by the update)
        "sentinel_1e20": (base * np.float32(3e10), 32, 2, 1234),
    }[case]


@pytest.mark.parametrize("case", ["duplicate_rows", "offset_100", "lattice_ties", "sentinel_1e20"])
def test_tc_adversarial(case, cuda, gsx_lib):
    X, k, it, seed = _adversarial(case)
    _check_oracle(np.ascontiguousarray(X), k, it, cuda, "tensor", seed=seed)

"""GPU: the wgmma (tensor-core) K-Means assign -- score GEMM in registers, candidate margin, strict re-evaluation.
Labels / counts / centroids bit-identical to the oracle and to the strict CUDA-core kernel at the C3 chunk size
(SURVEY 8(d): one full 781 250 x 45 chunk vs the oracle, all-chunk run-to-run determinism)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _tf32(a):
    return (a.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


@pytest.mark.parametrize("variant,rel", [(0, 2.0 ** -9), (2, 2.0 ** -15)])
@pytest.mark.parametrize("D,K", [(45, 256), (45, 50), (24, 100), (9, 16)])
def test_tc_scores_are_the_gemm(D, K, variant, rel, cuda, gsx_lib):
    """The accumulator holds x.c - ||c||^2/2 (layout / descriptor check) within the input-conversion error the
    margin assumes: variant 0 = kind::tf32 (2^-10 per operand), variant 2 = split-bf16, three kind::f16 products."""
    import torch
    from gsx import kmeans as gk
    rng = np.random.default_rng(D * 1000 + K)
    X = rng.normal(0, 0.15, (128, D)).astype(np.float32)
    C = rng.normal(0, 0.15, (K, D)).astype(np.float32)
    if variant == 2 and not gk.tensor_bf16_built():
        pytest.skip("split-bf16 variant is not part of this library")
    S = gk.tc_debug_scores(torch.from_numpy(X).to(cuda), torch.from_numpy(C).to(cuda), variant).cpu().numpy()[:, :K]
    exact = X.astype(np.float64) @ C.astype(np.float64).T - 0.5 * (C.astype(np.float64) ** 2).sum(1)[None]
    bound = rel * (np.linalg.norm(X, axis=1)[:, None] * np.linalg.norm(C, axis=1)[None] + 0.5 * (C ** 2).sum(1)[None]) + 1e-7
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


def test_tc_bf16_variant_margin_is_tight(cuda, gsx_lib):
    """Split-bf16 scores: the 100x tighter margin leaves < 2 % of the points with more than one candidate."""
    import torch
    from gsx import kmeans as gk
    if not gk.tensor_bf16_built():
        pytest.skip("split-bf16 variant is not part of this library")
    n, D, K = 400_000, 45, 256
    g = torch.Generator(device=cuda).manual_seed(9)
    proto = torch.randn(1024, D, device=cuda, generator=g) * 0.15
    X = proto[torch.randint(0, 1024, (n,), device=cuda, generator=g)] + 0.03 * torch.randn(n, D, device=cuda, generator=g)
    init = X[:K].clone().reshape(1, K, D)
    a = gk.kmeans_lloyd_batched(X, [0, n], K, 2, init, assign="tensor_bf16", want_stats=True)
    b = gk.kmeans_lloyd_batched(X, [0, n], K, 2, init, assign="tensor", want_stats=True)
    assert torch.equal(a[1], b[1]) and torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
    assert a[3]["full_scans"] == 0 and a[3]["multi_candidate_points"] < 0.02 * 2 * n
    assert a[3]["multi_candidate_points"] < b[3]["multi_candidate_points"]


def test_tc_all_chunks_deterministic_and_equal_to_strict(cuda, gsx_lib):
    """16 chunks x 200 000 rows in one launch: run-to-run determinism and tensor == strict == fma, bit for bit."""
    import torch
    from gsx import kmeans as gk
    nprob, rows, D, K = 16, 200_000, 45, 256
    g = torch.Generator(device=cuda).manual_seed(5)
    proto = torch.randn(1024, D, device=cuda, generator=g) * 0.15
    X = proto[torch.randint(0, 1024, (nprob * rows,), device=cuda, generator=g)] + \
        0.03 * torch.randn(nprob * rows, D, device=cuda, generator=g)
    offs = [p * rows for p in range(nprob + 1)]
    init = torch.stack([X[offs[p]:offs[p] + K] for p in range(nprob)])
    others = ("strict", "fma", "tensor_bf16") if gk.tensor_bf16_built() else ("strict", "fma")
    runs = {m: gk.kmeans_lloyd_batched(X, offs, K, 3, init, assign=m) for m in ("tensor",) + others}
    again = gk.kmeans_lloyd_batched(X, offs, K, 3, init, assign="tensor")
    for a, b in zip(runs["tensor"], again):
        assert torch.equal(a, b)
    for m in others:
        assert torch.equal(runs["tensor"][1], runs[m][1])
        assert torch.equal(runs["tensor"][0].view(torch.int32), runs[m][0].view(torch.int32))
        assert torch.equal(runs["tensor"][2], runs[m][2])


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

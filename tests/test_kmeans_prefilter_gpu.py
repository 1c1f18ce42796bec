"""GPU: K-Means with the exact pre-filters (fma scores on the FP32 pipes, or wgmma TF32 scores) is
bit-identical to the oracle (labels, counts, centroids), including adversarial near-tie inputs and the fallbacks."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["fma", "tensor", "tensor_bf16"])
def mode(request, gsx_lib):
    return request.param


def _check(X, k, it, cuda, mode, seed=1234):
    import torch
    import oracle
    from gsx import kmeans as gk
    np.random.seed(seed)
    init = oracle.kmeans_reference_init(X, k)
    Co, Lo, cnto = oracle.kmeans_lloyd(X, k, it, init=init)
    if mode.startswith("tensor") and not gk.tensor_core_supported(k, X.shape[1]):
        pytest.skip("shape not supported by the tensor-core path")
    if mode == "tensor_bf16" and not gk.tensor_bf16_built():
        pytest.skip("split-bf16 variant is not part of this library")
    C, L, cnt = gk.kmeans_lloyd(torch.from_numpy(X).to(cuda), k, it, torch.from_numpy(init).to(cuda), assign=mode)
    assert np.array_equal(L.cpu().numpy(), Lo)
    assert np.array_equal(cnt.cpu().numpy(), cnto)
    assert np.array_equal(C.cpu().numpy().view(np.uint32), Co.view(np.uint32))


@pytest.mark.parametrize("n,d,k,it", [(100_000, 45, 256, 3), (20_000, 45, 64, 5), (10_000, 24, 100, 3),
                                      (10_000, 9, 16, 10), (4_000, 45, 300, 2)])
def test_prefilter_matches_oracle(n, d, k, it, cuda, mode):
    from gsx import synth
    X = np.ascontiguousarray(synth.attributes(n)["f_rest"][:, :d])
    _check(X, k, it, cuda, mode)


def test_prefilter_adversarial(cuda, mode):
    rng = np.random.default_rng(0)
    base = rng.normal(0, 0.15, (3000, 45)).astype(np.float32)
    # many exactly duplicated rows -> the init draws duplicate centroids: > 8 exact ties -> overflow fallback
    X = np.ascontiguousarray(np.repeat(base[:150], 20, axis=0))
    _check(X, 64, 3, cuda, mode, seed=3)
    # large common offset: heavy cancellation in ||x||^2 - 2 x.c + ||c||^2
    _check(np.ascontiguousarray(base + np.float32(100.0)), 50, 3, cuda, mode)
    # lattice: exact distance ties between different centroids (lowest index must win)
    Xg = rng.integers(-2, 3, (5000, 9)).astype(np.float32)
    _check(Xg, 40, 4, cuda, mode)
    # distances around the 1e20 start value (label -1 rows are skipped by the update)
    _check(np.ascontiguousarray(base * np.float32(3e10)), 32, 2, cuda, mode)

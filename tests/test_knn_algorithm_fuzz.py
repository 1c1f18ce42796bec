"""CPU: the query kernel's ALGORITHM (tests/knn_emulator.py, small fan-outs) equals the brute-force oracle bit for bit
on adversarial clouds -- exactness of the pruning rules independent of the CUDA implementation."""
import numpy as np
import pytest

import oracle
from knn_emulator import emulate


def _clouds():
    rng = np.random.default_rng(42)
    yield "uniform", rng.uniform(-1, 1, (700, 3))
    yield "lattice_ties", np.stack(np.meshgrid(*[np.arange(8)] * 3), -1).reshape(-1, 3) * 0.25   # exact distance ties
    yield "dense_blob+halo", np.r_[rng.normal(0, 0.01, (500, 3)), rng.uniform(-2, 2, (150, 3))]   # big buckets
    yield "duplicates", np.repeat(rng.normal(size=(100, 3)), 5, axis=0)
    yield "planar", np.c_[rng.uniform(-1, 1, (500, 2)), np.zeros(500)]
    yield "two_scales", np.r_[rng.normal(0, 1e-3, (300, 3)), rng.normal(5, 1.0, (300, 3))]
    yield "wide_grid_wraps", rng.uniform(0, 1, (1500, 3)) * np.array([400.0, 3.0, 3.0])       # gx >= 30: i32 wrap differs


@pytest.mark.parametrize("mode", ["i32wrap", "i64"])
@pytest.mark.parametrize("k", [1, 16])
def test_emulated_algorithm_is_exact(mode, k):
    for name, pts in _clouds():
        xyz = pts.astype(np.float32)
        want = oracle.sor_taichi_mean_dists(xyz, k, mode)
        for chunk, fan, small in ((4, 4, 6), (3, 5, 0)):
            got, st = emulate(xyz, k, mode, chunk=chunk, fan=fan, small_bucket=small)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, mode, k, chunk, fan, small)


def test_pruning_actually_prunes():
    rng = np.random.default_rng(1)
    xyz = np.r_[rng.normal(0, 0.01, (1000, 3)), rng.uniform(-2, 2, (200, 3))].astype(np.float32)
    got, st = emulate(xyz, 8, "i64", chunk=4, fan=4, small_bucket=6)
    assert st["scanned"] < 0.5 * st["visits"], st       # a large part of the reference's visits is skipped ...
    assert np.array_equal(got, oracle.sor_taichi_mean_dists(xyz, 8, "i64"))   # ... without changing a bit


@pytest.mark.parametrize("flat,group", [(2, 3), (8, 4), (1000, 5)])
def test_flat_walk_of_long_buckets_is_exact(flat, group):
    """kFlatSupers (shipped: 8): a long bucket spanning fewer supers than that tests its chunk boxes directly,
    `group` at a time, in bucket order instead of nearest-super-first -- a different visiting ORDER, the same rule
    (a chunk is skipped only while its lower bound is >= the current tau), hence the same bits."""
    for name, pts in _clouds():
        if name not in ("dense_blob+halo", "two_scales", "duplicates", "lattice_ties"):
            continue
        xyz = pts.astype(np.float32)
        for k in (3, 16):
            want = oracle.sor_taichi_mean_dists(xyz, k, "i32wrap")
            got, st = emulate(xyz, k, "i32wrap", chunk=4, fan=4, small_bucket=6, flat_supers=flat, group=group)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, k, flat, group)

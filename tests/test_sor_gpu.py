"""GPU parity: SOR (Taichi semantics) through the C ABI vs the CPU oracle -- bit-exact.

Reference path under test: gpu_ops.py:193-263 (+ kernel :98-176).  Bar: final_means and the
keep-mask identical bit for bit (integer/index work and IEEE float32 with a fixed op order).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(xyz_np, k, sigma, mode, cuda):
    import torch
    from gsx import sor
    x = torch.from_numpy(xyz_np).to(cuda)
    mask, means = sor.sor_filter(x, k, sigma, hash_mode=mode, return_means=True)
    return mask.cpu().numpy(), means.cpu().numpy()


@pytest.mark.parametrize("kind", ["mixed", "uniform", "clustered"])
@pytest.mark.parametrize("mode", ["i32wrap", "i64"])
@pytest.mark.parametrize("n,k", [(100_000, 16), (100_000, 27), (30_000, 50), (300_000, 16), (60_000, 7), (40_000, 1)])
def test_sor_matches_oracle(kind, mode, n, k, cuda, gsx_lib):
    import oracle
    from gsx import synth
    xyz = synth.xyz(n, kind)
    want = oracle.sor_taichi_mean_dists(xyz, k, mode)
    for sigma in (2.0,):
        mask, means = _run(xyz, k, sigma, mode, cuda)
        assert np.array_equal(means.view(np.uint32), want.view(np.uint32)), \
            f"mean dists differ at {np.flatnonzero(means != want)[:5]}"
        assert np.array_equal(mask, oracle.threshold_mask(want, sigma))


@pytest.mark.parametrize("mode", ["i32wrap", "i64"])
def test_sor_1m_mixed_wrapped_hash_diverges(mode, cuda, gsx_lib):
    """At 1 M points the grid exceeds the int32-safe range: i32wrap != i64 (SURVEY F8) and both must match."""
    import oracle
    from gsx import synth
    xyz = synth.xyz(1_000_000, "mixed")
    want = oracle.sor_taichi_mean_dists(xyz, 16, mode)
    mask, means = _run(xyz, 16, 2.0, mode, cuda)
    assert np.array_equal(means.view(np.uint32), want.view(np.uint32))
    removed = int((~mask).sum())
    assert removed == {"i32wrap": 15932, "i64": 1385}[mode]  # SURVEY §8(c) anchor counts


def test_sor_edge_cases(cuda, gsx_lib):
    import oracle
    rng = np.random.default_rng(5)
    cases = {
        "tiny": rng.normal(size=(5, 3)),
        "single": np.zeros((1, 3)),
        "all_same": np.ones((100, 3)),
        "planar": np.c_[rng.uniform(-1, 1, (5000, 2)), np.zeros(5000)],
        "duplicates": np.repeat(rng.normal(size=(500, 3)), 4, axis=0),
        "line": np.c_[np.linspace(0, 1, 2000), np.zeros(2000), np.zeros(2000)],
        "two_blobs_far": np.r_[rng.normal(0, 0.01, (3000, 3)), rng.normal(1000, 0.01, (3000, 3))],
        "big_bucket": rng.normal(0, 1e-3, (20000, 3)),
    }
    for name, pts in cases.items():
        xyz = pts.astype(np.float32)
        for k in (3, 16):
            for mode in ("i32wrap", "i64"):
                want = oracle.sor_taichi_mean_dists(xyz, k, mode)
                mask, means = _run(xyz, k, 1.0, mode, cuda)
                assert np.array_equal(means.view(np.uint32), want.view(np.uint32)), (name, k, mode)
                assert np.array_equal(mask, oracle.threshold_mask(want, 1.0)), (name, k, mode)


def test_sor_host_entry_and_errors(cuda, gsx_lib):
    import oracle
    from gsx import sor, synth, GsxError
    xyz = synth.xyz(50_000, "mixed")
    mask, means = sor.sor_filter_host(xyz, 16, 2.0, return_means=True)
    want = oracle.sor_taichi_mean_dists(xyz, 16, "i32wrap")
    assert np.array_equal(means.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(mask, oracle.threshold_mask(want, 2.0))
    with pytest.raises(ValueError):
        sor.sor_filter_host(np.zeros((10, 2), np.float32))
    with pytest.raises(GsxError):
        sor.sor_filter_host(xyz, 0, 1.0)


def test_mean_std_matches_numpy(cuda, gsx_lib):
    import torch
    from gsx import sor
    rng = np.random.default_rng(11)
    for n in (1, 5, 8, 9, 27, 100, 128, 129, 264, 1000, 4097, 100_003, 131_073, 3_000_001, 16_777_216 + 5):
        a = rng.gamma(2.0, 0.3, n).astype(np.float32)
        want = np.array([np.mean(a), np.std(a)], dtype=np.float32)
        # 16-byte aligned vector: two lanes per leaf with float4 loads; offset by one element: the 8-lanes-per-leaf kernel
        for shift in (0, 1):
            buf = torch.empty(n + 4, dtype=torch.float32, device=cuda)
            dev = buf[shift: shift + n]
            dev.copy_(torch.from_numpy(a))
            got = sor.mean_std(dev).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (n, shift)


@pytest.mark.parametrize("cell_scale", [1.0, 0.25])
def test_build_from_sorted_equals_build(cuda, gsx_lib, cell_scale):
    """The stages of the distributed build on one GPU: partition by owner (3 pretend owners) -> per-owner sort
    -> concatenation in owner order -> build_from_sorted must give the same mean distances as the one-shot
    build (and as the oracle).  cell_scale 1: the reference's grid (~46 points per bucket, 79 buckets longer than 64
    -> the per-start threads plus the long-bucket kernel); 0.25: ~3 points per bucket, which overflows the start list
    (n/8 + 1024 entries) and must fall through to the re-hashing kernels on the device."""
    import ctypes as C
    import torch
    import oracle
    from gsx import sor, synth
    from gsx._abi import lib, check
    from gsx._abi import _ptr, _stream
    xyz_np = synth.xyz(200_000, "mixed")
    xyz = torch.from_numpy(xyz_np).to(cuda)
    n = xyz.shape[0]
    ref = sor.build_grid(xyz, cell_scale=cell_scale)
    bminp = ref.bmin.ctypes.data_as(C.POINTER(C.c_float))
    world = 3
    ws = sor.workspace(n, cuda)
    pos4 = torch.empty((n, 4), dtype=torch.float32, device=cuda)
    cuts = torch.zeros(world + 1, dtype=torch.int64, device=cuda)
    check(lib.gsx_sor_dist_local_run(_ptr(xyz), n, 0, n, world, bminp, ref.cell, _ptr(pos4), _ptr(cuts), _ptr(ws),
                                     ws.numel(), _stream()))
    c = cuts.tolist()
    assert c[0] == 0 and c[-1] == n and all(c[i] <= c[i + 1] for i in range(world))
    assert sorted(pos4[:, 3].view(torch.int32).tolist()) == list(range(n))      # a permutation of the slab
    off = lib.gsx_sor_spos_offset(n)
    want = {mode: oracle.sor_taichi_mean_dists(xyz_np, 16, mode) for mode in ("i32wrap", "i64")} if cell_scale == 1.0 else {}
    for with_flags in (False, True):   # stage C re-hashing every point / consuming the owners' per-point flags
        ws2 = torch.empty(lib.gsx_sor_grid_workspace_bytes(n), dtype=torch.uint8, device=cuda)   # grid-only blob
        spos_full = ws2[off: off + n * 16].view(torch.float32).view(n, 4)
        flags = torch.zeros(n, dtype=torch.uint8, device=cuda) if with_flags else None
        for o in range(world):                                                 # "owner o" sorts its range
            m = c[o + 1] - c[o]
            seg_in = pos4[c[o]: c[o + 1]].contiguous()
            blo, bhi = (o * n + world - 1) // world, ((o + 1) * n + world - 1) // world   # owner o's bucket range
            check(lib.gsx_sor_dist_merge(_ptr(seg_in), m, n, blo, bhi, bminp, ref.cell, _ptr(spos_full[c[o]: c[o + 1]]),
                                         _ptr(flags[c[o]: c[o + 1]]) if with_flags else None, _ptr(ws), ws.numel(),
                                         _stream()))
        check(lib.gsx_sor_build_from_sorted(_ptr(spos_full), _ptr(flags), n, bminp, ref.cell, _ptr(ws2), ws2.numel(),
                                            _stream()))
        grid2 = sor.SorGrid(n, ws2, ref.bmin, ref.cell)
        for mode in ("i32wrap", "i64"):
            a = sor.mean_dists(ref, 16, mode).cpu().numpy()
            b = sor.mean_dists(grid2, 16, mode).cpu().numpy()
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (with_flags, mode)
            if want:
                assert np.array_equal(a.view(np.uint32), want[mode].view(np.uint32))
            # cost-balanced sharding: 3 pretend ranks, batches dealt round-robin, union == the whole result
            u = torch.zeros(n, dtype=torch.float32, device=cuda)
            for r in range(3):
                sor.mean_dists_strided(grid2, 16, mode, u, 3, r)
            assert np.array_equal(u.cpu().numpy().view(np.uint32), a.view(np.uint32)), (with_flags, mode, "strided")

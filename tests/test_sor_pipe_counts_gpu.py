"""The SOR query kernel's counters of warp-collective work (gsx_sor_query_counters), and the two edges of the forms
that spend fewer of them: the lazy tau of a scan step and the lane-carrying, truncated box key.

  * a 200 k `mixed` cloud, K on both sides of every template form, both hash modes: mean distances bit-equal to the
    oracle, and the counters satisfy the identities that pin what each one counts;
  * `symmetric_pair`: a query with two candidates at the same distance in one serial scan step -- whichever comes
    second is >= the tau the first one produced, and is inserted all the same (TopK::insert keeps the list exact);
  * `lattice`: a cubic lattice, where bucket-box lower bounds and K-th best distances coincide up to rounding -- boxes
    whose lower bound is less than 32 ulp above tau, which the truncated key visits where the exact test would
    not.  An unmarked CPU test asserts that the lattice really produces such boxes.
"""
import functools

import numpy as np
import pytest

import oracle
from test_sor_kernel_paths_gpu import (MODES, _assert_bits, _candidates, _f32, _grid, _probe_hashes, _sorted_rows)

KS = (1, 8, 16, 17, 32, 50)
COUNTERS = ("inserts", "merges_first", "merges_full", "probe_visits", "super_visits", "chunk_groups", "chunk_visits",
            "scan_steps")


@functools.lru_cache(None)
def mixed_200k():
    from gsx import synth
    return _f32(synth.xyz(200_000, "mixed"))


@functools.lru_cache(None)
def symmetric_pair():
    """q at the origin, a and b at distance 1 on either side, c and d at distance 2, two far corners that make the
    cell larger than the cloud: one bucket of 7 points, 6 candidates per query (< kMergeThreshold: serial inserts)."""
    return _f32([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 2, 0], [0, -2, 0], [-1000, -1000, -1000], [1000, 1000, 1000]])


@functools.lru_cache(None)
def lattice():
    """16^3 points at i * 0.1f: every query has neighbours and bucket faces at (almost) the same distances."""
    i = np.arange(16, dtype=np.float32) * np.float32(0.1)
    return _f32(np.stack(np.meshgrid(i, i, i, indexing="ij"), -1).reshape(-1, 3))


@functools.lru_cache(None)
def lattice_one_cell():
    """14^3 lattice points inside one grid cell (corners at +-1000 set the cell): one long bucket, so the same
    coincidences meet the chunk boxes of the flat walk."""
    i = np.arange(14, dtype=np.float32) * np.float32(0.3) - np.float32(2.0)
    c = [[x, y, z] for x in (-1000, 1000) for y in (-1000, 1000) for z in (-1000, 1000)]
    return _f32(np.r_[np.stack(np.meshgrid(i, i, i, indexing="ij"), -1).reshape(-1, 3), np.array(c, np.float32)])


def _d2(a):
    return (a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1]) + a[:, 2] * a[:, 2]


def near_tau_boxes(xyz, k, mode):
    """Number of probed bucket boxes whose lower bound lb (the kernel's float32 op sequence) lies less than 32 ulp
    above the query's final K-th best d^2 with key(lb) < tau <= lb: visited under the truncated key, skipped by the
    exact test."""
    lo, cell, gi, order, start, count = _grid(xyz)
    spos = xyz[order]
    box = {h: (spos[start[h]:start[h] + count[h]].min(0), spos[start[h]:start[h] + count[h]].max(0))
           for h in np.flatnonzero(count)}
    extra = 0
    zero = np.float32(0)
    for r, hs in enumerate(_probe_hashes(gi, len(xyz), mode)):
        hs = [h for h in hs if start[h] != -1]
        idx = np.concatenate([np.arange(start[h], start[h] + count[h]) for h in hs])
        d2 = np.sort(_d2(xyz[r] - spos[idx]))
        d2 = d2[d2 > np.float32(1e-12)]
        if len(d2) < k:
            continue
        tau = d2[k - 1]
        blo, bhi = np.array([box[h][0] for h in hs]), np.array([box[h][1] for h in hs])
        lb = _d2(np.maximum(np.maximum(blo - xyz[r], xyz[r] - bhi), zero))
        bits, tbits = lb.view(np.uint32).astype(np.int64), int(tau.view(np.uint32))
        near = np.abs(bits - tbits) < 32
        extra += int(np.sum(near & (lb >= tau) & ((bits & ~31) < tbits)))
    return extra


def test_lattice_has_boxes_within_32_ulp_of_tau():
    for k in (1, 6, 16):
        assert near_tau_boxes(lattice(), k, "i64") > 100, k


def _mean_dists(xyz, k, mode, cuda, q_range=None):
    import torch
    from gsx import sor
    grid = sor.build_grid(torch.from_numpy(np.array(xyz)).to(cuda))
    out, st = sor.mean_dists(grid, k, mode, want_stats=True, q_range=q_range)
    return grid, out.cpu().numpy(), st


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_counters_mixed_cloud(mode, cuda, gsx_lib):
    import torch
    from gsx import sor
    xyz = mixed_200k()
    n = len(xyz)
    grid = sor.build_grid(torch.from_numpy(np.array(xyz)).to(cuda))
    rows = _sorted_rows(grid)
    qb, qe = 100_000, 101_024            # the K-lists of these queries are restated on the CPU
    cands = _candidates(xyz, mode, rows[qb:qe])
    for k in KS:
        want = oracle.sor_taichi_mean_dists(xyz, k, mode)
        out, st = sor.mean_dists(grid, k, mode, want_stats=True)
        _assert_bits(out.cpu().numpy(), want, f"k={k} {mode}")
        assert st["queries"] == n
        assert st["chunk_visits"] <= st["box_tests"], st
        assert st["chunk_visits"] <= st["scan_steps"], st
        assert st["scanned"] <= 32 * st["scan_steps"], st
        assert st["probe_visits"] <= 27 * n and st["super_visits"] <= st["box_tests"], st
        assert st["chunk_groups"] * 32 >= st["chunk_visits"], st
        if k > 32:
            assert st["merges_first"] == st["merges_full"] == 0, st        # two registers per lane: serial inserts only
        else:
            assert st["merges_first"] <= n, st
        # every distinct distance of a K-list entered it by a serial insert or as one of a merge's 32 candidates
        _, sq = sor.mean_dists(grid, k, mode, want_stats=True, q_range=(qb, qe))
        distinct = sum(len(np.unique(c[c < np.float32(1e10)][:min(k, 50)])) for c in cands)
        assert sq["queries"] == qe - qb
        assert sq["inserts"] + 32 * (sq["merges_first"] + sq["merges_full"]) >= distinct, (k, sq, distinct)
        # an empty range zeroes every counter
        _, s0 = sor.mean_dists(grid, k, mode, want_stats=True, q_range=(qb, qb))
        assert all(s0[c] == 0 for c in COUNTERS) and s0["queries"] == 0, s0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_lazy_tau_symmetric_pair(mode, cuda, gsx_lib):
    xyz = symmetric_pair()
    lo, cell, gi, order, start, count = _grid(xyz)
    assert count.max() == len(xyz)                         # one bucket: one serial scan step holds both a and b
    for k in (1, 2, 3, 6):
        grid, got, st = _mean_dists(xyz, k, mode, cuda)
        _assert_bits(got, oracle.sor_taichi_mean_dists(xyz, k, mode), f"k={k} {mode}")
        assert st["merges_first"] == st["merges_full"] == 0 and st["inserts"] >= 6 * len(xyz), st


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("geometry", ["lattice", "lattice_one_cell"])
def test_truncated_key_lattice(geometry, mode, cuda, gsx_lib):
    xyz = globals()[geometry]()
    for k in (1, 6, 16, 26, 50):
        grid, got, st = _mean_dists(xyz, k, mode, cuda)
        _assert_bits(got, oracle.sor_taichi_mean_dists(xyz, k, mode), f"{geometry} k={k} {mode}")
    if geometry == "lattice_one_cell":
        assert st["chunk_visits"] > 0 and st["chunk_groups"] > 0, st

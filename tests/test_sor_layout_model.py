"""CPU: the in-cell Hilbert code and the k-d leaf layout rule of scripts/sor_layout_model.py."""
import importlib.util
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
_spec = importlib.util.spec_from_file_location("sor_layout_model", ROOT / "scripts" / "sor_layout_model.py")
lm = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(lm)


def test_kd_split_picks_the_chunk_boundary_nearest_the_middle():
    assert lm.kd_split(0, 1024) == 512
    assert lm.kd_split(0, 64) == 32
    assert lm.kd_split(10, 40) == 32            # the only boundary inside (10, 40)
    assert lm.kd_split(5, 100) == 64            # (5 + 100) / 2 = 52.5 is nearer 64 than 32
    assert lm.kd_split(1000, 2049) == 1536      # translation by a super keeps the split relative to it
    for a in range(0, 200, 7):
        for b in range(a + 2, 400, 13):
            if (a >> 5) != ((b - 1) >> 5):
                m = lm.kd_split(a, b)
                assert m % 32 == 0 and a < m < b


def test_kd_layout_is_a_per_segment_permutation_that_the_checker_accepts():
    rng = np.random.default_rng(0)
    pts = np.r_[rng.normal(0, 0.01, (5000, 3)), rng.normal(1, 0.05, (3000, 3)), rng.uniform(-3, 3, (4000, 3))].astype(np.float32)
    lo = pts.min(0)
    order, sh = lm.cell_order(pts, lo, 0.5, "morton")
    sp = pts[order]
    starts, ends = lm.bucket_ranges(sh)
    segs = [(a, b) for a, b in lm.long_segments(starts, ends) if (a >> 5) != ((b - 1) >> 5)]
    assert len(segs) >= 5 and max(b - a for a, b in segs) >= 512
    assert all(a // lm.SUPER == (b - 1) // lm.SUPER for a, b in segs)
    perm = lm.kd_layout(sp, starts, ends)
    kd = sp[perm]
    moved = np.flatnonzero(perm != np.arange(len(sp)))
    assert all(any(a <= j < b for a, b in segs) for j in moved[:: max(1, len(moved) // 200)])
    for a, b in segs:
        assert sorted(perm[a:b].tolist()) == list(range(a, b))
        assert lm.check_kd_leaves(kd[a:b], a, b)
    assert not all(lm.check_kd_leaves(sp[a:b], a, b) for a, b in segs)   # the Morton order is not such a layout


def test_hilbert_code_is_a_face_adjacent_walk_of_the_cell():
    g = np.stack(np.meshgrid(*[np.arange(32)] * 3, indexing="ij"), -1).reshape(-1, 3)
    code = lm.hilbert_code(g)
    assert sorted(code.tolist()) == list(range(32 ** 3))
    walk = g[np.argsort(code)]
    assert (np.abs(np.diff(walk, axis=0)).sum(1) == 1).all()
    # hierarchical: the top 3k bits are the curve over 2^k sub-cells per axis, so every aligned run of 8^j codes is a cube
    for j in (1, 2, 3):
        runs = walk.reshape(-1, 8 ** j, 3)
        assert ((runs.max(1) - runs.min(1)) == 2 ** j - 1).all()

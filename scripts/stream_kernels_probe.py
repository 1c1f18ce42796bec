"""Achieved HBM bandwidth of the streaming stages (SURVEY §8d: bbox / alpha / density / compaction / stats are
HBM-bound).  Algorithmic bytes per splat are the ones listed in DESIGN.md; times are CUDA events, inputs larger
than L2 (N = 64 M splats: xyz 768 MB).  Prints one JSON object."""
import json
import sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
import numpy as np
import torch
from gsx import sor, masks, density, pipeline


def ev(fn, reps=5):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 64_000_000
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(7)
    xyz = torch.rand((n, 3), device=dev, generator=g) * 20 - 10
    xyz[: n // 2] = torch.randn((n // 2, 3), device=dev, generator=g) * 0.8
    op = torch.randn(n, device=dev, generator=g) * 2
    peak = 3350.0   # H100 SXM data-sheet HBM3 bandwidth, GB/s
    out = {"n": n, "peak_GBps": peak, "stages": {}}

    def rec(name, ms, bytes_per_pt, note=""):
        gbs = n * bytes_per_pt / (ms * 1e-3) / 1e9
        out["stages"][name] = {"ms": round(ms, 3), "bytes_per_splat": bytes_per_pt, "GBps": round(gbs, 1),
                               "frac_of_hbm_peak": round(gbs / peak, 3), "note": note}

    rec("bbox_mask", ev(lambda: masks.bbox_mask(xyz, -2, -2, -2, 2, 2, 2)), 13, "12 B xyz read + 1 B mask written")
    rec("alpha_mask", ev(lambda: masks.alpha_mask(op, 5)), 5, "4 B opacity read + 1 B mask written")
    means = torch.rand(n, device=dev, generator=g)
    ms_t = sor.mean_std(means)
    rec("mean_std_numpy_order", ev(lambda: sor.mean_std(means)), 8, "two passes over 4 B (mean, then variance)")
    rec("threshold_mask", ev(lambda: sor.threshold_mask(means, ms_t, 2.0)), 5, "4 B read + 1 B written")
    mask = torch.rand(n, device=dev, generator=g) < 0.5
    rec("compact_points(50%)", ev(lambda: pipeline.compact(mask, xyz, op, None)), 1 + 1 + 16 + 0.5 * 20,
        "mask read twice, xyz+opacity read, 20 B written per survivor")
    voxel, thr = density.slider(0.5)
    mp = int(n * thr / 100)
    rec("density_voxel_count(dense grid)", ev(lambda: density.dense_voxels(xyz, voxel, mp)), 12 + 12,
        "min/max pass (12 B) + 12 B xyz read + one int32 atomic per splat (grid is L2-resident)")
    vox, cnt, nu, ws = density.dense_voxels(xyz, voxel, mp)
    keep, _, _ = density.select_clusters(vox, True)
    rec("density_member_mask", ev(lambda: density.member_mask(xyz, voxel, keep, ws)), 13, "12 B read + 1 B written")
    wsb = sor.workspace(n, dev)
    t_build = ev(lambda: sor.build_grid(xyz, wsb), reps=3)
    rec("sor_grid_build", t_build, 12 + 24 + 6 * 32 + 8 + 32 + 28 + 16 + 1,
        "min/max 12, keys 24, 6 radix passes x 32, table 8 + 32 memset, gather 28 (random 12 B reads), boxes 17")
    print(json.dumps(out))


if __name__ == "__main__":
    main()

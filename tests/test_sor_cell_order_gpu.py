"""GPU: the grid build orders each hash bucket by the in-cell Hilbert code (scripts/sor_layout_model.py restates it).

The built float4 array must be exactly the NumPy order (bucket, 15-bit Hilbert code, original index), from the one-shot
build and from the distributed stage C with and without the owners' flags, on a cloud with long buckets.
"""
import ctypes as C
import importlib.util
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
_spec = importlib.util.spec_from_file_location("sor_layout_model", ROOT / "scripts" / "sor_layout_model.py")
lm = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(lm)


def _spos(ws, n):
    from gsx._abi import lib
    off = lib.gsx_sor_spos_offset(n)
    return ws[off: off + 16 * n].cpu().numpy().view(np.float32).reshape(n, 4).copy()


@pytest.mark.parametrize("kind", ["mixed", "clustered"])
def test_build_orders_buckets_by_hilbert_code(kind, cuda, gsx_lib):
    import torch
    from gsx import sor, synth
    from gsx._abi import lib, check
    from gsx._abi import _ptr, _stream
    xyz_np = synth.xyz(200_000, kind)
    n = len(xyz_np)
    xyz = torch.from_numpy(xyz_np).to(cuda)
    ref = sor.build_grid(xyz)
    want, sh = lm.cell_order(xyz_np, ref.bmin, np.float32(ref.cell), "hilbert")
    starts, ends = lm.bucket_ranges(sh)
    assert (ends - starts).max() > 1024                      # long buckets: the order inside them is what changed
    got = _spos(ref.ws, n)
    assert np.array_equal(got[:, 3].view(np.int32), want.astype(np.int32))
    assert np.array_equal(got[:, :3], xyz_np[want])
    morton, _ = lm.cell_order(xyz_np, ref.bmin, np.float32(ref.cell), "morton")
    assert not np.array_equal(morton, want)

    # stage C: 3 pretend owners sort their bucket ranges; the segments in owner order must give the same array
    bminp = ref.bmin.ctypes.data_as(C.POINTER(C.c_float))
    world = 3
    ws = sor.workspace(n, cuda)
    pos4 = torch.empty((n, 4), dtype=torch.float32, device=cuda)
    cuts = torch.zeros(world + 1, dtype=torch.int64, device=cuda)
    check(lib.gsx_sor_dist_local_run(_ptr(xyz), n, 0, n, world, bminp, ref.cell, _ptr(pos4), _ptr(cuts), _ptr(ws),
                                     ws.numel(), _stream()))
    c = cuts.tolist()
    off = lib.gsx_sor_spos_offset(n)
    for with_flags in (False, True):
        ws2 = torch.empty(lib.gsx_sor_grid_workspace_bytes(n), dtype=torch.uint8, device=cuda)
        spos_full = ws2[off: off + n * 16].view(torch.float32).view(n, 4)
        flags = torch.zeros(n, dtype=torch.uint8, device=cuda) if with_flags else None
        for o in range(world):
            seg_in = pos4[c[o]: c[o + 1]].contiguous()
            blo, bhi = (o * n + world - 1) // world, ((o + 1) * n + world - 1) // world
            check(lib.gsx_sor_dist_merge(_ptr(seg_in), c[o + 1] - c[o], n, blo, bhi, bminp, ref.cell,
                                         _ptr(spos_full[c[o]: c[o + 1]]),
                                         _ptr(flags[c[o]: c[o + 1]]) if with_flags else None, _ptr(ws), ws.numel(),
                                         _stream()))
        check(lib.gsx_sor_build_from_sorted(_ptr(spos_full), _ptr(flags), n, bminp, ref.cell, _ptr(ws2), ws2.numel(),
                                            _stream()))
        assert np.array_equal(_spos(ws2, n), got), with_flags

"""Fixed workload for `ncu --metrics gpu__time_duration.sum`: the single-GPU grid build and the replicated stage C of
the distributed build (gsx_sor_build_from_sorted) at n points."""
import ctypes as C
import sys
from pathlib import Path
import torch
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))
from gsx import sor  # noqa: E402
from gsx._abi import lib, check  # noqa: E402
from gsx._abi import _ptr, _stream  # noqa: E402
import importlib.util  # noqa: E402
spec = importlib.util.spec_from_file_location("b", ROOT / "bench.py"); b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b)
from gsx import synth  # noqa: E402
n = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000_000
dev = torch.device("cuda:0")
xyz, _ = b.device_cloud(n, dev, 1, synth)
ws = sor.workspace(n, dev)
for _ in range(2):
    grid = sor.build_grid(xyz, ws)
torch.cuda.synchronize()
off = lib.gsx_sor_spos_offset(n)
spos = ws[off: off + n * 16].view(torch.float32).view(n, 4).clone()
gws = torch.empty(lib.gsx_sor_grid_workspace_bytes(n), dtype=torch.uint8, device=dev)
sp2 = gws[off: off + n * 16].view(torch.float32).view(n, 4)
sp2.copy_(spos)
# owner-computed flags for the same array (one pretend owner): stage B on the whole cloud
bminp = grid.bmin.ctypes.data_as(C.POINTER(C.c_float))
pos4_in = spos.clone()
flags = torch.zeros(n, dtype=torch.uint8, device=dev)
wsb = sor.workspace(n, dev)
check(lib.gsx_sor_dist_merge(_ptr(pos4_in), n, n, 0, n, bminp, grid.cell, _ptr(sp2), _ptr(flags), _ptr(wsb), wsb.numel(), _stream()))
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for it in range(3):
    ev[0].record()
    check(lib.gsx_sor_build_from_sorted(_ptr(sp2), _ptr(flags), n, bminp, grid.cell, _ptr(gws), gws.numel(), _stream()))
    ev[1].record()
    torch.cuda.synchronize()
    print(f"n={n} build_from_sorted(with owner flags) ms={ev[0].elapsed_time(ev[1]):.3f}")
for it in range(3):
    ev[0].record()
    check(lib.gsx_sor_build_from_sorted(_ptr(sp2), None, n, grid.bmin.ctypes.data_as(C.POINTER(C.c_float)), grid.cell, _ptr(gws),
                                        gws.numel(), _stream()))
    ev[1].record()
    torch.cuda.synchronize()
    print(f"n={n} build_from_sorted ms={ev[0].elapsed_time(ev[1]):.3f}")

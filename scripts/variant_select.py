"""A/B of libgsx build variants on the GPU box, with a parity digest per variant; optionally installs the fastest one
as 3dgsconverter_b200/lib/libgsx.so so that the tests and bench that follow use it.

    python scripts/variant_select.py [--install] [--n 10000000]

Variants = 3dgsconverter_b200/lib/variants/libgsx_*.so (scripts/build_variants.sh).  A variant is eligible only if its
keep-mask digests (mixed and uniform cloud, i32wrap, k=16, sigma=2) equal those of the variant called `base`.
Timing: CUDA events around gsx_sor_filter_device on a resident cloud, min of 5 after 2 warm-ups."""
import json
import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
VAR = ROOT / "3dgsconverter_b200" / "lib" / "variants"

CHILD = r'''
import sys, json, hashlib
sys.path.insert(0, "."); sys.path.insert(0, "3dgsconverter_b200")
import numpy as np, torch
from gsx import sor, synth
n = int(sys.argv[1])
res = {}
for kind in ("mixed", "uniform"):
    x = torch.from_numpy(synth.xyz(n, kind)).cuda()
    ws = sor.workspace(n, x.device)
    grid = sor.build_grid(x, ws)
    ts, tk = [], []
    for it in range(7):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record(); m = sor.sor_filter(x, 16, 2.0, hash_mode="i32wrap", ws=ws); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    grid = sor.build_grid(x, ws)
    for it in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record(); sor.mean_dists(grid, 16, "i32wrap"); b.record(); torch.cuda.synchronize()
        tk.append(a.elapsed_time(b))
    res[kind] = dict(filter_ms=round(min(ts[2:]), 3), knn_ms=round(min(tk[1:]), 3),
                     mask_sha=hashlib.sha256(np.packbits(m.cpu().numpy()).tobytes()).hexdigest()[:16], kept=int(m.sum()))
    del x, ws, grid
print(json.dumps(res))
'''


def main():
    install = "--install" in sys.argv
    n = int(sys.argv[sys.argv.index("--n") + 1]) if "--n" in sys.argv else 10_000_000
    out = {}
    for so in sorted(VAR.glob("libgsx_*.so")):
        name = so.stem[len("libgsx_"):]
        env = dict(os.environ, GSX_LIB=str(so))
        r = subprocess.run([sys.executable, "-c", CHILD, str(n)], cwd=ROOT, env=env, capture_output=True, text=True,
                           timeout=300)
        if r.returncode != 0:
            out[name] = {"error": r.stderr[-400:]}
        else:
            out[name] = json.loads(r.stdout.strip().splitlines()[-1])
        print(name, json.dumps(out[name]), flush=True)
    base = out.get("base", {})
    ok = {k: v for k, v in out.items() if "error" not in v and "error" not in base and
          all(v[c]["mask_sha"] == base[c]["mask_sha"] for c in ("mixed", "uniform"))}
    choice = min(ok, key=lambda k: ok[k]["mixed"]["filter_ms"]) if ok else None
    rec = {"n": n, "variants": out, "eligible": sorted(ok), "choice": choice, "installed": False}
    if install and choice:
        lib = ROOT / "3dgsconverter_b200" / "lib" / "libgsx.so"
        shutil.copyfile(VAR / f"libgsx_{choice}.so", lib)
        rec["installed"] = True
    (ROOT / "gpurun_out").mkdir(exist_ok=True)
    (ROOT / "gpurun_out" / "variant_choice.json").write_text(json.dumps(rec, indent=1))
    print("CHOICE", choice, flush=True)


if __name__ == "__main__":
    main()

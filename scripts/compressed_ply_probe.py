"""Compressed PLY encode on one GPU: CUDA-event times of its stages on N resident DeviceRecords (default 10 M `mixed`
SH-3 splats), the pack kernel's achieved bandwidth, the card it ran on, and a parity check of the timed run's outputs
against the NumPy oracle (tests/compressed_ply_oracle.py) in the device's Morton order.

    python scripts/compressed_ply_probe.py [N] [--reps R] [--out FILE]

Prints one JSON object (and writes it to FILE if given)."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "3dgsconverter_b200"), str(ROOT / "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gsx import compressed_ply, morton, records, synth  # noqa: E402
from gsx._abi import check, lib  # noqa: E402
from gsx._abi import _ptr, _stream  # noqa: E402

PEAK_GBPS = 3350.0   # H100 SXM data-sheet HBM3 bandwidth


def ev(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3),
            "max_ms": round(float(np.max(ts)), 3), "reps": reps}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("n", type=int, nargs="?", default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    a = synth.structured(args.n, "mixed")
    r = records.DeviceRecords.from_structured(a, dev)
    n, F = len(r), r.F
    out = {"n": n, "row_bytes": 4 * F, "card": card(), "stages": {}}

    xyz = r.xyz_opacity()[0]
    order = morton.morton_order(xyz)
    cols = [r.col[f] for f in compressed_ply.PACK_FIELDS]
    rest = [r.col[f"f_rest_{i}"] for i in range(45) if f"f_rest_{i}" in r.col]
    out["stages"]["morton_order"] = ev(lambda: morton.morton_order(xyz), args.reps)
    out["stages"]["chunk_bounds_x2"] = ev(lambda: (morton.chunk_minmax(r.rows, cols[:6], order),
                                                   morton.chunk_minmax(r.rows, cols[7:10], order, clip=(-20.0, 20.0))),
                                          args.reps)
    lo6, hi6 = morton.chunk_minmax(r.rows, cols[:6], order)
    lo3, hi3 = morton.chunk_minmax(r.rows, cols[7:10], order, clip=(-20.0, 20.0))
    chunk = torch.empty((lo6.shape[0], 18), dtype=torch.float32, device=dev)
    vertex = torch.empty((n, 4), dtype=torch.int32, device=dev)
    sh = torch.empty((n, len(rest)), dtype=torch.uint8, device=dev)
    nz = torch.empty(1, dtype=torch.int64, device=dev)
    c14, crest = (C.c_int32 * 14)(*cols), (C.c_int32 * max(len(rest), 1))(*rest)

    def pack():
        check(lib.gsx_cply_pack(_ptr(r.rows), n, F, _ptr(order), c14, crest, len(rest), _ptr(lo6), _ptr(hi6), _ptr(lo3),
                                _ptr(hi3), _ptr(chunk), _ptr(vertex), _ptr(sh), _ptr(nz), _stream()), "gsx_cply_pack")

    t = ev(pack, args.reps)
    moved = n * (4 * F + 16 + len(rest))          # gathered row read + packed words and SH bytes written
    gbps = moved / (t["median_ms"] * 1e-3) / 1e9
    t.update(bytes=moved, GBps=round(gbps, 1), frac_of_hbm_peak=round(gbps / PEAK_GBPS, 3),
             bytes_note=f"{4 * F} B row read + {16 + len(rest)} B written per splat")
    out["stages"]["pack_kernel"] = t
    out["stages"]["encode"] = ev(lambda: compressed_ply.encode(r), args.reps)
    out["stages"]["encode_to_host"] = ev(lambda: compressed_ply.encode(r).to_host(), args.reps)

    # parity of one more (identical) run against the oracle, in the device's own order
    enc = compressed_ply.encode(r)
    got = enc.to_host()
    t0 = time.perf_counter()
    import compressed_ply_oracle as cpo
    want = cpo.encode(a, enc.order.cpu().numpy())
    cpo.assert_packed_equal(got, want)
    da = np.count_nonzero((got[1]["packed_color"] & 0xFF) != (want[1]["packed_color"] & 0xFF))
    out["parity"] = {"ok": True, "alpha_bytes_differing": int(da), "sh_columns": len(enc.sh_names),
                     "oracle_s": round(time.perf_counter() - t0, 1)}
    out["card_after"] = card()
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")


if __name__ == "__main__":
    main()

"""Time the device readers on 10 M `mixed` SH-3 splats: each format's file (written by the device writer), then the
host parse (+ gunzip for SPZ), the H2D of the file's bytes, the whole `decode` call (CUDA events, 2 warm-ups, median of
10), the decode kernels alone (torch.profiler with CUDA activities over 10 more calls: the mean device time per call of
the k_*_decode kernels; bytes read and written and their share of 3.35 TB/s) and to_host; the output is checked
against the NumPy oracle (tests/readers_oracle.py) in the same run, whose time is reported as the oracle's.  Prints one
JSON line per format and the card's name and power limit.

    python scripts/readers_probe.py [--n 10000000] [--out results.json]
"""
import argparse
import gzip
import json
import re
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT / "3dgsconverter_b200"), str(ROOT / "tests")]

from gsx import compressed_ply, ksplat, readers, records, splat, spz, synth  # noqa: E402
import readers_oracle as ro  # noqa: E402

PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def events_median(fn, warm=2, reps=10):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return float(np.median(ts))


def kernel_time(fn, warm=2, reps=10):
    """Mean device time per call of the decode kernels (k_splat_decode, k_ksplat_decode, k_spz_decode, k_cply_decode)
    that `fn` launches, from torch.profiler's CUDA activity records."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.key_averages():
        if re.search(r"\bk_(splat|ksplat|spz|cply)_decode\b", e.key):
            us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    if us == 0.0:
        raise RuntimeError("no decode kernel in the profile")
    return us / 1e6 / reps


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    a = synth.structured(args.n, "mixed")
    r = records.DeviceRecords.from_structured(a, "cuda")
    files = {"splat": splat.encode(r).to_host(), "ksplat_l0": ksplat.encode(r, 0).to_host(),
             "ksplat_l1": ksplat.encode(r, 1).to_host(), "ksplat_l2": ksplat.encode(r, 2).to_host(),
             "spz": gzip.compress(spz.encode(r).to_host(), compresslevel=1)}
    with tempfile.TemporaryDirectory() as tmp:   # the PLY writer takes a path; nothing is written into the tree
        cp = Path(tmp) / "probe.compressed.ply"
        compressed_ply.write_ply(cp, *compressed_ply.encode(r).to_host())
        files["cply"] = cp.read_bytes()
    del r
    torch.cuda.empty_cache()
    results = {"card": card(), "n": args.n}
    for name, blob in files.items():
        fmt = name.split("_")[0]
        mod = {"splat": splat, "ksplat": ksplat, "spz": spz, "cply": compressed_ply}[fmt]
        dec, total = wall(lambda: mod.decode(blob, "cuda"))
        # the stages, separately: host parse / gunzip, H2D, the kernel alone, D2H
        t0 = time.perf_counter()
        buf = readers.file_bytes(blob)
        if fmt == "spz":
            buf = memoryview(gzip.decompress(buf))
        t_host = time.perf_counter() - t0
        raw, t_h2d = wall(lambda: readers.upload(buf, "cuda"))
        t_call = events_median(lambda: mod.decode(blob, "cuda"))
        t_kernel = kernel_time(lambda: mod.decode(blob, "cuda"))
        host, t_d2h = wall(dec.to_host)
        t0 = time.perf_counter()
        with np.errstate(all="ignore"):
            want, meta = ro.READERS[fmt](blob)
        t_oracle = time.perf_counter() - t0
        ok = host.tobytes() == np.ascontiguousarray(want).tobytes() and repr(meta) == repr(dec.metadata)
        moved = len(buf) + dec.rows.numel()   # every record byte read once, every row byte written once
        results[name] = {"file_bytes": len(blob), "rows_bytes": dec.rows.numel(), "first_decode_s": total,
                         "host_parse_s": t_host, "h2d_s": t_h2d, "decode_call_median_s": t_call,
                         "kernel_s": t_kernel, "kernel_bytes": moved,
                         "kernel_share_of_3.35TBps": moved / t_kernel / PEAK,
                         "to_host_s": t_d2h, "numpy_oracle_s": t_oracle, "equal_to_oracle": bool(ok)}
        print(json.dumps({name: results[name]}), flush=True)
        del dec, raw, host, want
        torch.cuda.empty_cache()
    print(json.dumps({"card": results["card"]}))
    if args.out:
        Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()

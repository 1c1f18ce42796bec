"""gzip of the .spz payload on one GPU: gsx.deflate (Spz.compress) against CPython's gzip.compress, for N `mixed` SH-3
splats (default 10 M) and the sparse-SH variant (90 % of the splats with zero f_rest, seeded), resident as
DeviceRecords.  Reports, with the card and its power limit read in the same run:
  * Spz.compress at level 6 (CUDA events around the call, which ends in a device synchronise; 2 warm-ups, median of
    --reps) and its kernels (torch.profiler, a separate pass), with the bytes they must move against 3.35 TB/s;
  * write_spz wall time, host gzip and device gzip, at level 0 (the CLI default) and 6;
  * gzip.compress on the host at levels 0, 1 and 6 (one run each; level 9 on a 1 M-splat payload only);
  * every file's size over the payload's.

    python scripts/spz_gzip_probe.py [--n N] [--reps R] [--kind mixed|sparse|both] [--no-level9] [--out FILE]

Prints one JSON object (and writes it to FILE if given)."""
import argparse
import gzip
import json
import re
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "3dgsconverter_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gsx import records, spz, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def cloud(n, sparse):
    a = synth.structured(n, "mixed", 3)
    if sparse:
        zero = np.random.default_rng(2024).random(n) < 0.9
        for i in range(45):
            a[f"f_rest_{i}"][zero] = 0
    return a


def event_ms(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    out = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e))
    return statistics.median(out)


def wall_s(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def kernels_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" and ("deflate" in ev.key or "crc" in ev.key):
            out[re.search(r"k_\w+", ev.key).group(0)] = round(ev.device_time_total / 1e3, 3)
    return out


def probe(n, sparse, reps, dev):
    enc = spz.encode(records.DeviceRecords.from_writer_input(cloud(n, sparse), dev))
    size = enc.payload.numel()
    r = {"splats": n, "sparse_sh": sparse, "payload_bytes": size}
    blob = enc.compress(6)
    r["device_level6_ratio"] = round(len(blob) / size, 4)
    r["compress_level6_ms"] = round(event_ms(lambda: enc.compress(6), reps), 2)
    r["compress_level0_ms"] = round(event_ms(lambda: enc.compress(0), reps), 2)
    k = kernels_ms(lambda: enc.compress(6))
    r["level6_kernels_ms"] = k
    moved = 3 * size + len(blob)              # plan, emit and CRC read the payload; emit writes the body
    r["level6_kernel_bytes"] = moved
    r["level6_kernel_floor_ms"] = round(moved / HBM_BYTES_PER_S * 1e3, 3)
    with tempfile.TemporaryDirectory() as td:
        for level in (0, 6):
            for where in ("host", "device") if level == 0 else ("device",):
                r[f"write_spz_{where}_level{level}_s"] = round(
                    wall_s(lambda: spz.write_spz(Path(td) / "x.spz", enc, level, where=where)), 3)
    payload = enc.to_host()
    for level in (0, 1, 6) if not sparse else (1, 6):
        t = time.perf_counter()
        z = gzip.compress(payload, level, mtime=0)
        r[f"host_gzip_level{level}_s"] = round(time.perf_counter() - t, 2)
        r[f"host_gzip_level{level}_ratio"] = round(len(z) / size, 4)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--kind", choices=("mixed", "sparse", "both"), default="both")
    ap.add_argument("--no-level9", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    kinds = {"mixed": (False,), "sparse": (True,), "both": (False, True)}[args.kind]
    res = {"card": card(), "runs": [probe(args.n, s, args.reps, dev) for s in kinds]}
    if not args.no_level9:
        level9(res, dev)
    res["card_after"] = card()
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(txt)


def level9(res, dev):
    enc = spz.encode(records.DeviceRecords.from_writer_input(cloud(1_000_000, False), dev))
    payload = enc.to_host()
    t = time.perf_counter()
    z = gzip.compress(payload, 9, mtime=0)
    res["host_gzip_level9_1m"] = {"s": round(time.perf_counter() - t, 2), "ratio": round(len(z) / len(payload), 4),
                                  "device_level6_ratio": round(len(enc.compress(6)) / len(payload), 4)}


if __name__ == "__main__":
    main()

"""gunzip of .spz files on one GPU: gsx.deflate.gunzip against CPython's gzip.decompress, for N `mixed` SH-3 splats
(default 10 M) packed on the device, gzipped by gzip.compress at --levels (default 0, 1, 6, 9) and by gsx.deflate.gzip
at level 6.  Reports per file, with the card and its power limit read in the same run:
  * gzip.decompress wall time (one run), and that the device result equals it byte for byte;
  * gunzip time including the file's H2D (CUDA events around the call, which ends in a device synchronise;
    2 warm-ups, median of --reps) and the chain's counts: chunks, finder false starts, re-decodes, overflow re-runs;
  * its kernels and copies by torch.profiler, in a separate pass;
  * the whole spz.decode call (which gunzips on the device) against the same call handed the body gunzipped by
    gzip.decompress, as the reader did before (wall time, median of 3);
and for the level-1 file cut into two members (two gzip.compress calls), gunzip's time against the one-member file.

    python scripts/spz_gunzip_probe.py [--n N] [--reps R] [--levels 0,1,6,9] [--out FILE]

Prints one JSON object (and writes it to FILE if given)."""
import argparse
import gzip
import json
import re
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "3dgsconverter_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gsx import deflate, records, spz, synth  # noqa: E402
from gsx.hostcopy import to_host  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


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


def wall_s(fn, reps=3):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return statistics.median(out)


def say(*a):
    print(*a, file=sys.stderr, flush=True)


def kernels_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" and ("inflate" in ev.key or "crc" in ev.key):
            k = re.search(r"k_\w+", ev.key).group(0)
            out[k] = round(out.get(k, 0) + ev.device_time_total / 1e3, 3)
        elif ev.device_type.name == "CUDA" and "Memcpy" in ev.key:
            out[ev.key] = round(out.get(ev.key, 0) + ev.device_time_total / 1e3, 3)
    return out


def probe_file(name, blob, payload, reps, dev):
    r = {"file": name, "file_bytes": len(blob)}
    t = time.perf_counter()
    want = gzip.decompress(blob)
    r["gzip_decompress_s"] = round(time.perf_counter() - t, 3)
    st = {}
    got = deflate.gunzip(blob, dev, stats=st)
    r["equal_to_gzip_decompress"] = bool(got.numel() == len(want) and to_host(got).tobytes() == want)
    r["equal_to_payload"] = want == payload
    r.update(st)
    del got
    r["gunzip_ms"] = round(event_ms(lambda: deflate.gunzip(blob, dev), reps), 2)
    r["kernels_ms"] = kernels_ms(lambda: deflate.gunzip(blob, dev))
    r["spz_decode_s"] = round(wall_s(lambda: spz.decode(blob, dev)), 4)
    r["spz_decode_host_gunzip_s"] = round(wall_s(lambda: spz.decode(gzip.decompress(blob), dev)), 4)
    say(json.dumps(r))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--levels", default="0,1,6,9")
    ap.add_argument("--out")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = {"card": card(), "splats": args.n}
    enc = spz.encode(records.DeviceRecords.from_writer_input(synth.structured(args.n, "mixed", 3), dev))
    payload = enc.to_host()
    res["payload_bytes"] = len(payload)
    files = []
    for level in (int(x) for x in args.levels.split(",")):
        t = time.perf_counter()
        files.append((f"gzip.compress level {level}", gzip.compress(payload, level, mtime=0)))
        res[f"gzip_compress_level{level}_s"] = round(time.perf_counter() - t, 2)
        say(f"compressed level {level}: {res[f'gzip_compress_level{level}_s']} s")
    files.append(("gsx.deflate.gzip level 6", enc.compress(6)))
    del enc
    res["runs"] = [probe_file(name, blob, payload, args.reps, dev) for name, blob in files]
    half = len(payload) // 2
    two = gzip.compress(payload[:half], 1, mtime=0) + gzip.compress(payload[half:], 1, mtime=0)
    one = gzip.compress(payload, 1, mtime=0)
    same = to_host(deflate.gunzip(two, dev)).tobytes() == payload
    res["two_members_level1"] = {"equal_to_payload": same,
                                 "gunzip_ms": round(event_ms(lambda: deflate.gunzip(two, dev), args.reps), 2),
                                 "one_member_gunzip_ms": round(event_ms(lambda: deflate.gunzip(one, dev), args.reps), 2)}
    res["card_after"] = card()
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(txt)


if __name__ == "__main__":
    main()

"""Time the plain PLY codec (gsx.ply) on 10 M `mixed` SH-3 splats, a 2.5 GB file: for each flavour the host parse, the
H2D of the file's bytes, the whole `decode` and `encode` calls (CUDA events, 2 warm-ups, median of 10), the transcode
kernel alone (torch.profiler with CUDA activities over 10 more calls: mean device time per call of k_ply_transcode;
bytes read and written and their share of 3.35 TB/s), to_host and the file write; the outputs are checked against the
NumPy oracle (tests/ply_oracle.py) in the same run, whose wall-clock time is reported.  Prints one JSON line per stage
group and the card's name and power limit.

    python scripts/ply_probe.py [--n 10000000] [--out results.json]
"""
import argparse
import json
import re
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT / "3dgsconverter_b200"), str(ROOT / "tests"), str(ROOT / "scripts")]

from gsx import ply, readers, synth  # noqa: E402
import ply_oracle as po  # noqa: E402
from readers_probe import PEAK, card, events_median, wall  # noqa: E402


def kernel_time(fn, warm=2, reps=10):
    """Mean device time per call of k_ply_transcode that `fn` launches, from torch.profiler's CUDA activity records."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
             for e in prof.key_averages() if re.search(r"\bk_ply_transcode\b", e.key))
    if us == 0.0:
        raise RuntimeError("no k_ply_transcode in the profile")
    return us / 1e6 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    a = synth.structured(args.n, "mixed")
    results = {"card": card(), "n": args.n}
    for flavor in ("3dgs", "cc"):
        blob = po.file(po.write(a, flavor))
        dec, first = wall(lambda: ply.decode(blob, flavor, "cuda"))
        t0 = time.perf_counter()
        vx, dtype, table = ply.read_plan(readers.file_bytes(blob), flavor)
        t_parse = time.perf_counter() - t0
        raw, t_h2d = wall(lambda: readers.upload(readers.file_bytes(blob), "cuda"))
        t_decode = events_median(lambda: ply.decode(blob, flavor, "cuda"))
        t_kdec = kernel_time(lambda: ply.transcode(raw, vx.offset, vx.count, vx.dtype.itemsize, dtype.itemsize, table))
        host, t_d2h = wall(dec.to_host)
        t0 = time.perf_counter()
        want = po.read(blob, flavor)
        t_oracle_read = time.perf_counter() - t0
        ok_read = host.tobytes() == want.tobytes()
        r = dec.records()
        t_encode = events_median(lambda: ply.encode(r, flavor))
        enc = ply.encode(r, flavor)
        out, t_eh = wall(enc.to_host)
        t_kenc = kernel_time(lambda: ply.encode(r, flavor))
        with tempfile.TemporaryDirectory() as tmp:   # nothing is written into the tree
            _, t_write = wall(lambda: ply.write_ply(Path(tmp) / "probe.ply", enc))
            ok_file = (Path(tmp) / "probe.ply").read_bytes() == blob
        t0 = time.perf_counter()
        want_enc = po.write(want, flavor)
        t_oracle_write = time.perf_counter() - t0
        ok_write = out.tobytes() == want_enc.tobytes()
        moved_dec = vx.count * (vx.dtype.itemsize + dtype.itemsize)   # every row byte read once and written once
        moved_enc = len(enc) * (4 * r.F + enc.dtype.itemsize)
        results[flavor] = {
            "file_bytes": len(blob), "first_decode_s": first, "host_parse_s": t_parse, "h2d_s": t_h2d,
            "decode_call_median_s": t_decode, "decode_kernel_s": t_kdec, "decode_kernel_bytes": moved_dec,
            "decode_kernel_share_of_3.35TBps": moved_dec / t_kdec / PEAK, "decode_to_host_s": t_d2h,
            "encode_call_median_s": t_encode, "encode_kernel_s": t_kenc, "encode_kernel_bytes": moved_enc,
            "encode_kernel_share_of_3.35TBps": moved_enc / t_kenc / PEAK, "encode_to_host_s": t_eh,
            "write_ply_s": t_write, "numpy_oracle_read_s": t_oracle_read, "numpy_oracle_write_s": t_oracle_write,
            "equal_to_oracle": bool(ok_read and ok_write and ok_file)}
        print(json.dumps({flavor: results[flavor]}), flush=True)
        del dec, raw, host, want, r, enc, out, want_enc, blob
        torch.cuda.empty_cache()
    print(json.dumps({"card": results["card"]}))
    if args.out:
        Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()

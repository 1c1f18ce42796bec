"""Time the SOG reader (gsx.sog_reader) on 10 M `mixed` SH-3 splats: the bundle is encoded on the device (gsx.sog.encode
with a quantile codebook fit instead of scikit-learn) and bundled by write_sog in a temporary directory.  Stages: the
unzip (meta.json and the member bytes), the WebP decode serial against threaded (GSX_HOST_THREADS), the H2D of the
pixels, the two kernels alone (torch.profiler CUDA activities over 5 decode_textures calls on device-resident pixels;
bytes read and written and their share of 3.35 TB/s), the whole `decode` call (CUDA events, 1 warm-up, median of 5),
to_host, and the NumPy oracle (tests/sog_reader_oracle.py) on the same bytes, whose output is compared in the same
run.  Prints one JSON line with the card's name and power limit.

    python scripts/sog_reader_probe.py [--n 10000000] [--out results.json]
"""
import argparse
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

from gsx import records, sog, sog_reader, synth  # noqa: E402
from gsx.hostcopy import to_device  # noqa: E402
import sog_reader_oracle as sro  # noqa: E402

PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def cheap_fit(values):
    return np.quantile(values.reshape(-1), np.linspace(0, 1, 256)).reshape(-1, 1)


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def events_median(fn, warm=1, reps=5):
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


def kernel_times(fn, warm=2, reps=5):
    """Mean device time per call of k_sog_palette and k_sog_decode, from torch.profiler's CUDA activity records."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {"k_sog_palette": 0.0, "k_sog_decode": 0.0}
    for e in prof.key_averages():
        for k in out:
            if re.search(rf"\b{k}\b", e.key):
                out[k] += (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)) / 1e6 / reps
    if not all(out.values()):
        raise RuntimeError(f"a kernel is missing from the profile: {out}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    a = synth.structured(args.n, "mixed")
    np.random.seed(0)
    tex = sog.encode(records.DeviceRecords.from_structured(a, "cuda"), codebook_fit=cheap_fit)
    del a
    with tempfile.TemporaryDirectory() as tmp:   # nothing is written into the tree
        p = Path(tmp) / "probe.sog"
        sog.write_sog(p, tex.to_host(), tex.meta)
        blob = p.read_bytes()
    del tex
    torch.cuda.empty_cache()
    res = {"card": card(), "n": args.n, "bundle_bytes": len(blob)}
    dec, res["first_decode_s"] = wall(lambda: sog_reader.decode(blob, "cuda"))
    del dec
    t0 = time.perf_counter()
    zf, meta = sog_reader.open_bundle(blob)
    lay = sog_reader.parse_meta(meta)
    for name in lay.members():
        zf.read(name)
    res["unzip_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    flat = sog_reader.decode_members(zf, lay.members(), threads=1)
    res["webp_serial_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    flat = sog_reader.decode_members(zf, lay.members())
    res["webp_threaded_s"] = time.perf_counter() - t0
    res["webp_threads"] = sog_reader.host_threads(len(lay.members()))
    dev, res["h2d_s"] = wall(lambda: to_device(flat, "cuda"))
    res["pixel_bytes"] = int(flat.nbytes)
    pixels, off = {}, 0
    for name, need in lay.members().items():
        pixels[name] = dev[off:off + 4 * need]
        off += 4 * need
    kt = kernel_times(lambda: sog_reader.decode_textures(pixels, lay))
    res.update({f"{k}_s": v for k, v in kt.items()})
    d = sog_reader.decode_textures(pixels, lay)
    # k_sog_decode: 24 texture bytes per splat read (6 RGBA pixels), one row written, the palette rows from L2
    moved = 24 * lay.count + d.rows.numel()
    res["k_sog_decode_bytes"] = moved
    res["k_sog_decode_share_of_3.35TBps"] = moved / kt["k_sog_decode"] / PEAK
    res["decode_call_median_s"] = events_median(lambda: sog_reader.decode(blob, "cuda"))
    host, res["to_host_s"] = wall(d.to_host)
    t0 = time.perf_counter()
    with np.errstate(all="ignore"):
        want = sro.decode(blob)
    res["numpy_oracle_s"] = time.perf_counter() - t0
    res["equal_to_oracle"] = bool(host.tobytes() == np.ascontiguousarray(want).tobytes())
    print(json.dumps(res), flush=True)
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

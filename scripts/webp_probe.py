"""Lossless WebP of a SOG bundle on one GPU: gsx.webp against Pillow for the seven textures of N `mixed` SH-3 splats
(default 10 M).  Reports, with the card and its power limit read in the same run:
  * per member: gsx_webp_analyze and the whole encode_lossless (CUDA events around a device synchronise, 3 warm-ups,
    median of 10), and the bytes of both encoders;
  * per kernel: device time summed over one encode of every member (torch.profiler, a separate pass);
  * the whole write_sog from SogTextures (device WebP) and from the host dict (Pillow), wall time, and bundle sizes.

    python scripts/webp_probe.py [--n N] [--reps R] [--out FILE]

Prints one JSON object (and writes it to FILE if given)."""
import argparse
import io
import json
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

from gsx import records, sog, synth, webp  # noqa: E402
from gsx._abi import lib  # noqa: E402
from gsx._abi import _ptr, _stream  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def pillow_bytes(img):
    from PIL import Image
    bio = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(img), "RGBA").save(bio, format="WEBP", lossless=True, quality=100, method=1)
    return len(bio.getvalue())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    a = synth.structured(args.n, "mixed", 3)
    np.random.seed(1)
    fit = lambda v: np.quantile(v.reshape(-1), np.linspace(0, 1, 256)).astype(np.float32)  # noqa: E731
    tex = sog.encode(records.DeviceRecords.from_structured(a, dev), 0, codebook_fit=fit)
    host = tex.to_host()
    res = {"n": args.n, "card": card(), "members": {}}
    for name, t in tex.textures.items():
        w, h = tex.sizes[name]
        ws = torch.empty(lib.gsx_webp_workspace_bytes(w, h), dtype=torch.uint8, device=dev)
        hist = torch.empty(5 * webp.TREE_SYMS + 1, dtype=torch.int32, device=dev)
        analyze = lambda: lib.gsx_webp_analyze(_ptr(t), w, h, _ptr(ws), ws.numel(), _ptr(hist), None,  # noqa: E731
                                               _stream())
        info = {}
        data = webp.encode_lossless(t, w, h, info=info)
        pil = pillow_bytes(host[name])
        res["members"][name] = {
            "size": [w, h], "analyze_ms": round(timed(analyze, args.reps), 3),
            "encode_ms": round(timed(lambda: webp.encode_lossless(t, w, h), args.reps), 3),
            "candidate": info["candidate"], "gsx_bytes": len(data), "pillow_bytes": pil,
            "ratio": round(len(data) / pil, 4)}
        del ws, hist
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, t in tex.textures.items():
            webp.encode_lossless(t, *tex.sizes[name])
        torch.cuda.synchronize()
    res["kernels_ms_all_members"] = {e.key: round(e.device_time_total / 1e3, 3) for e in prof.key_averages()
                                     if e.device_time_total > 0}
    with tempfile.TemporaryDirectory() as d:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sog.write_sog(Path(d) / "dev.sog", tex, tex.meta)
        res["write_sog_device_s"] = round(time.perf_counter() - t0, 4)
        t0 = time.perf_counter()
        sog.write_sog(Path(d) / "pil.sog", tex.to_host(), tex.meta)
        res["write_sog_pillow_s"] = round(time.perf_counter() - t0, 3)
        res["bundle_bytes"] = {"device": (Path(d) / "dev.sog").stat().st_size,
                               "pillow": (Path(d) / "pil.sog").stat().st_size}
    res["bundle_ratio"] = round(res["bundle_bytes"]["device"] / res["bundle_bytes"]["pillow"], 4)
    res["encode_ms_all_members"] = round(sum(m["encode_ms"] for m in res["members"].values()), 3)
    res["card_after"] = card()
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s)


if __name__ == "__main__":
    main()

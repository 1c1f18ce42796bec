"""Time the device VP8L decoder (gsx.webp_decode) on the WebP members of a 10 M `mixed` SH-3 SOG bundle written
(a) by Pillow (lossless, quality 100, method 1, as the reference writer does) and (b) by gsx's device encoder.  The
textures come from gsx.sog.encode with a quantile codebook fit instead of scikit-learn; bundles live in a temporary
directory.  Per member: Pillow's decode + convert('RGBA') on one thread (1 warm-up, median / min / max of 3),
decode_lossless by CUDA events (1 warm-up, median / min / max of 3; the warm-up's own wall time when it takes over
2 s), its peak device memory above what was allocated before, its kernels by torch.profiler over one further call
(members under 2 s), its chain counts and stream features, and whether its pixels equal Pillow's.  Then the whole
sog_reader.decode with webp="host" (threaded Pillow) and webp="device" (CUDA events, as above), rows compared byte
for byte.  --profile writes the full torch.profiler table of one decode_lossless of bundle (b)'s means_l.  Prints
one JSON line with the card's name and power limit.

    python scripts/webp_decode_probe.py [--n 10000000] [--out results.json] [--profile prof.txt]
"""
import argparse
import io
import json
import re
import subprocess
import sys
import tempfile
import time
import zipfile
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT / "3dgsconverter_b200")]

from gsx import records, sog, sog_reader, synth  # noqa: E402
from gsx.webp_decode import decode_lossless  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def cheap_fit(values):
    return np.quantile(values.reshape(-1), np.linspace(0, 1, 256)).reshape(-1, 1)


def events_median(fn, reps=3):
    """(median, min, max) of `reps` timed calls after one untimed call; that call's wall time alone when it took over
    2 s."""
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter() - t
    if t > 2.0:
        return t, t, t
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return float(np.median(ts)), min(ts), max(ts)


def log(msg):
    print(msg, file=sys.stderr, flush=True)


def pillow_once(blob):
    from PIL import Image
    img = Image.open(io.BytesIO(blob))
    return np.asarray(img if img.mode == "RGBA" else img.convert("RGBA"))


def pillow(blob, reps=3):
    """The pixels, and (median, min, max) wall time of `reps` decodes on this thread after one warm-up."""
    px = pillow_once(blob)
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        pillow_once(blob)
        ts.append(time.perf_counter() - t)
    return px, (float(np.median(ts)), min(ts), max(ts))


def kernels(fn):
    """ms per kernel name (gsx kernels only) over one call, from torch.profiler's CUDA activity records."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"(k_vp8l_\w+)", e.key)
        if m:
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            out[m.group(1)] = round(out.get(m.group(1), 0.0) + t / 1e3, 3)
    return out


def members(blob):
    with zipfile.ZipFile(io.BytesIO(blob)) as zf:
        return {n: zf.read(n) for n in zf.namelist() if n.endswith(".webp")}


def probe_bundle(blob):
    out = {"bundle_bytes": len(blob), "members": {}}
    for name, data in members(blob).items():
        want, t_pil = pillow(data)
        st = {}
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        got = decode_lossless(data, "cuda", stats=st)
        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        same = bool(np.array_equal(got.cpu().numpy(), want))
        del got
        t_dev = events_median(lambda: decode_lossless(data, "cuda"))
        ks = kernels(lambda: decode_lossless(data, "cuda")) if t_dev[0] < 2.0 else None
        log(f"{name}: pillow {t_pil} s, device {t_dev} s, peak {peak:.0f} MiB, equal {same}, {st}, {ks}")
        out["members"][name] = dict(bytes=len(data), pillow_s=[round(v, 4) for v in t_pil],
                                    device_s=[round(v, 4) for v in t_dev], peak_mib=round(peak, 1), equal=same,
                                    kernels_ms=ks, **{k: v for k, v in st.items()})
    host = sog_reader.decode(blob, "cuda").to_host()
    dev = sog_reader.decode(blob, "cuda", webp="device").to_host()
    out["decode_rows_equal"] = host.tobytes() == dev.tobytes()
    log(f"rows equal {out['decode_rows_equal']}")
    out["decode_host_s"] = [round(v, 4) for v in events_median(lambda: sog_reader.decode(blob, "cuda"))]
    out["decode_device_s"] = [round(v, 4) for v in events_median(lambda: sog_reader.decode(blob, "cuda",
                                                                                          webp="device"))]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    a = synth.structured(args.n, "mixed")
    np.random.seed(0)
    tex = sog.encode(records.DeviceRecords.from_structured(a, "cuda"), codebook_fit=cheap_fit)
    del a
    blobs = {}
    with tempfile.TemporaryDirectory() as tmp:   # nothing is written into the tree
        for key, how in (("pillow_m1", tex.to_host()), ("gsx", tex)):
            p = Path(tmp) / f"{key}.sog"
            sog.write_sog(p, how, tex.meta)
            blobs[key] = p.read_bytes()
    del tex
    torch.cuda.empty_cache()
    log("bundles written")
    res = {"card": card(), "n": args.n}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        data = members(blobs["gsx"])["means_l.webp"]
        decode_lossless(data, "cuda")
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            decode_lossless(data, "cuda")
            torch.cuda.synchronize()
        Path(args.profile).write_text(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
        log("profiled")
    for key in ("gsx", "pillow_m1"):
        log(key)
        res[key] = probe_bundle(blobs[key])
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()

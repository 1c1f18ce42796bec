"""The .ksplat / .spz / .splat writers on one GPU: CUDA-event times of their device stages on N resident DeviceRecords
(default 10 M `mixed` SH-3 splats), bytes moved per stage and the share of HBM peak, the host stages (copy back, gzip,
file write), the card it ran on, and a check of the timed runs' outputs against the NumPy oracle
(tests/splat_codecs_oracle.py).

    python scripts/splat_codecs_probe.py [N] [--reps R] [--out FILE]

Prints one JSON object (and writes it to FILE if given)."""
import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "3dgsconverter_b200"), str(ROOT / "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gsx import ksplat, records, splat, spz, synth  # noqa: E402
from gsx._abi import check, lib  # noqa: E402
from gsx._abi import _ptr, _stream  # noqa: E402
from gsx.sor import sort_pairs  # noqa: E402

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


def wall(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": round(float(np.median(ts)), 1), "min_ms": round(float(np.min(ts)), 1), "reps": reps}


def roof(t, read, written):
    gbps = (read + written) / (t["median_ms"] * 1e-3) / 1e9
    t.update(bytes_read=read, bytes_written=written, GBps=round(gbps, 1), frac_of_hbm_peak=round(gbps / PEAK_GBPS, 3))
    return t


def sector_bytes(cols, F):
    """DRAM bytes per row of reading `cols` of a row-major float32 [N, F] matrix: the 32-byte sectors the columns touch,
    averaged over the row's alignment phases."""
    phases = [(4 * F * i) % 32 for i in range(32)]
    return sum(32 * len({(p + 4 * c) // 32 for c in cols}) for p in phases) / len(phases)


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
    fixed = [r.col[f] for f in ksplat.PACK_FIELDS]
    sh = {k: [r.col[f"f_rest_{i}"] for i in range(k)] for k in (24, 45)}
    row = {"ksplat_l0": sector_bytes(fixed + sh[24], F), "spz": sector_bytes(fixed + sh[45], F),
           "splat": sector_bytes(fixed, F)}
    out = {"n": n, "row_bytes": 4 * F, "sector_bytes_read_per_row": row, "card": card(), "stages": {}, "host": {}}
    st = out["stages"]
    for lv in (0, 1, 2):
        enc = ksplat.encode(r, lv)
        st[f"ksplat_l{lv}_encode"] = roof(ev(lambda: ksplat.encode(r, lv), args.reps), int(n * row["ksplat_l0"]),
                                          enc.records.numel() + (enc.centres.numel() * 4 if lv else 0))
    enc = spz.encode(r)
    st["spz_encode"] = roof(ev(lambda: spz.encode(r), args.reps), int(n * row["spz"]), enc.payload.numel())

    keys = torch.empty(n, dtype=torch.int64, device=dev)
    order = torch.empty(n, dtype=torch.int32, device=dev)
    c4 = (C.c_int32 * 4)(*[r.col[f] for f in ("scale_0", "scale_1", "scale_2", "opacity")])

    def metric_sort():
        check(lib.gsx_splat_sort_keys(_ptr(r.rows), n, F, c4, _ptr(keys), _ptr(order), _stream()), "sort_keys")
        sort_pairs(keys, order, 0, 32)

    st["splat_metric_sort"] = ev(metric_sort, args.reps)
    out_b = torch.empty((n, 32), dtype=torch.uint8, device=dev)
    c14 = (C.c_int32 * 14)(*[r.col[f] for f in ksplat.PACK_FIELDS])
    st["splat_pack"] = roof(ev(lambda: check(lib.gsx_splat_pack(_ptr(r.rows), n, F, _ptr(order), c14, _ptr(out_b),
                                                                 _stream()), "splat_pack"), args.reps),
                            int(n * (row["splat"] + 4)), 32 * n)
    st["splat_encode"] = ev(lambda: splat.encode(r), args.reps)

    host = out["host"]
    hreps = 3
    blobs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, enc in (("ksplat_l0", ksplat.encode(r, 0)), ("ksplat_l1", ksplat.encode(r, 1)),
                          ("ksplat_l2", ksplat.encode(r, 2)), ("spz", spz.encode(r)), ("splat", splat.encode(r))):
            torch.cuda.synchronize()
            host[f"{name}_to_host"] = wall(lambda: enc.to_host(), hreps)
            blobs[name] = enc.to_host()
            path = os.path.join(tmp, name)
            if name == "spz":
                host["spz_gzip_level0"] = wall(lambda: gzip.compress(blobs[name], compresslevel=0), hreps)
                data = gzip.compress(blobs[name], compresslevel=0)
            else:
                data = blobs[name]
            host[f"{name}_file_write"] = wall(lambda: Path(path).write_bytes(data), hreps)
            host[f"{name}_bytes"] = len(blobs[name])

    import splat_codecs_oracle as sco
    t0 = time.perf_counter()
    with np.errstate(all="ignore"):
        want = {"ksplat_l0": sco.ksplat_file(a, 0), "ksplat_l1": sco.ksplat_file(a, 1),
                "ksplat_l2": sco.ksplat_file(a, 2), "spz": sco.spz_payload(a), "splat": sco.splat_file(a)}
    out["parity"] = {k: blobs[k] == v for k, v in want.items()}
    out["parity"]["oracle_s"] = round(time.perf_counter() - t0, 1)
    out["card_after"] = card()
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")
    if not all(v for k, v in out["parity"].items() if k != "oracle_s"):
        sys.exit(1)


if __name__ == "__main__":
    main()

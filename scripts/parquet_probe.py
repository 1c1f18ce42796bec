"""Time gsx.parquet's device writer on 10 M-row SH-3 clouds (random records, and records decoded on the device from
gsx's own .spz of the same cloud), beside pandas' to_parquet of the same frame on the same host.

    python scripts/parquet_probe.py [--n 10000000] [--reps 5] [--out results.json]

Per cloud: the encode time (median of --reps runs after a warm-up, each ending in a synchronise), each entry point's
time from CUDA events in one more run, to_host and the file write, the file size; pandas to_parquet's time (median of
3) and size.  The card's name and power limit are read in the same run.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "3dgsconverter_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def kernel_times(src):
    """ms per libgsx entry point of one encode, from CUDA events around each call."""
    from gsx import _abi
    times, real = {}, {}
    for name in [k for k in _abi._SIGS if k.startswith("gsx_parquet_") and "bytes" not in k]:
        fn = getattr(_abi.lib, name)
        real[name] = fn

        def timed(*a, _fn=fn, _name=name):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = _fn(*a)
            e1.record()
            e1.synchronize()
            times[_name] = times.get(_name, 0.0) + e0.elapsed_time(e1)
            return rc
        setattr(_abi.lib, name, timed)
    try:
        from gsx import parquet as gp
        gp.encode(src)
        torch.cuda.synchronize()
    finally:
        for name, fn in real.items():
            setattr(_abi.lib, name, fn)
    return {k: round(v, 3) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    import pandas as pd
    from gsx import parquet as gp, spz, synth
    from gsx.records import DeviceRecords
    dev = torch.device("cuda:0")
    a = synth.structured(args.n, "mixed", 3)
    rec = DeviceRecords.from_structured(a, dev)
    dec = spz.decode(spz.encode(rec).to_host(), device=dev)
    res = {"card": card(), "n": args.n, "clouds": {}}
    for kind, src, host in (("random", rec, a), ("spz", dec, None)):
        gp.encode(src)
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            t = time.perf_counter()
            enc = gp.encode(src)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t)
        t = time.perf_counter()
        blob = enc.to_host()
        t_host = time.perf_counter() - t
        with tempfile.TemporaryDirectory() as tmp:
            t = time.perf_counter()
            with open(os.path.join(tmp, "f.parquet"), "wb") as fh:
                fh.write(blob)
            t_write = time.perf_counter() - t
        host = dec.to_host() if host is None else host
        df = pd.DataFrame({c.name: host[c.source] for c in gp.column_plan(host.dtype)})
        pt = []
        for _ in range(3):
            buf = io.BytesIO()
            t = time.perf_counter()
            df.to_parquet(buf)
            pt.append(time.perf_counter() - t)
        res["clouds"][kind] = {
            "encode_ms_median": round(1e3 * float(np.median(ts)), 2), "encode_ms_all": [round(1e3 * x, 2) for x in ts],
            "kernels_ms": kernel_times(src), "to_host_ms": round(1e3 * t_host, 2), "file_write_ms": round(1e3 * t_write, 2),
            "file_bytes": len(blob), "pandas_to_parquet_s_median": round(float(np.median(pt)), 3),
            "pandas_bytes": len(buf.getvalue()), "size_ratio": round(len(blob) / len(buf.getvalue()), 4)}
        print(kind, json.dumps(res["clouds"][kind]), flush=True)
    print(json.dumps(res))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

"""SOG encode on one GPU: where the time goes for N resident DeviceRecords (default 10 M `mixed` SH-3 splats; pass
--n 50000000 for the C3 size).  Reports the device stages (CUDA events), the host stages (the reference's NumPy RNG
draws, the scikit-learn codebook fit, WebP + ZIP), the card and its power limit, and a parity check of the timed run
against the NumPy oracle (tests/sog_oracle.py), whose chunk K-Means is gsx's own (same init draws), so that only the
non-K-Means arithmetic is compared.

    python scripts/sog_probe.py [--n N] [--level L] [--no-parity] [--out FILE]

Prints one JSON object (and writes it to FILE if given)."""
import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "3dgsconverter_b200"), str(ROOT / "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gsx import records, sog, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--level", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    t0 = time.perf_counter()
    a = synth.structured(args.n, "mixed")
    r = records.DeviceRecords.from_structured(a, dev)
    out = {"n": len(r), "level": args.level, "row_bytes": 4 * r.F, "card": card(),
           "synth_and_upload_s": round(time.perf_counter() - t0, 2)}

    fits = []

    def fit(values):
        c = sog.default_codebook_fit(values)
        fits.append(c)
        return c

    np.random.seed(args.seed)                          # warm-up run: module loads, allocator, kernels
    sog.encode(r, args.level, codebook_fit=fit)
    torch.cuda.synchronize()
    fits.clear()
    prof = {}
    np.random.seed(args.seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    enc = sog.encode(r, args.level, codebook_fit=fit, profile=prof)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    a_ev, b_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a_ev.record()
    host = enc.to_host()
    b_ev.record()
    torch.cuda.synchronize()
    device_names = ("lexsort", "positions", "quats", "sh_gather", "codebook_fits", "sh0_scales", "chunk_kmeans",
                    "palette_textures")
    out["device_ms"] = {k: round(prof.get(k, 0.0), 2) for k in device_names}
    out["device_ms"]["to_host"] = round(a_ev.elapsed_time(b_ev), 2)
    out["host_ms"] = {"rng_draws": round(prof.get("rng", 0.0), 1), "codebook_fit": round(prof.get("codebook_fit", 0.0), 1)}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        sog.write_sog(Path(tmp) / "out.sog", host, enc.meta)
        out["host_ms"]["webp_zip"] = round((time.perf_counter() - t0) * 1e3, 1)
        out["sog_bytes"] = (Path(tmp) / "out.sog").stat().st_size
    out["encode_wall_ms"] = round(wall * 1e3, 1)
    out["palette"] = {"count": enc.meta["shN"]["count"], "bands": enc.meta["shN"]["bands"]}

    if not args.no_parity:
        import sog_oracle as so
        from gsx.kmeans import kmeans_lloyd

        def chunk_kmeans(data, k, max_iter=10):
            if data.shape[1] == 1:                     # the 1-D codebooks: the oracle's own Lloyd
                return so.oracle_kmeans(data, k, max_iter)
            if k >= len(data):
                return data.copy(), np.arange(len(data), dtype=np.int32)
            init = data[np.random.choice(len(data), k, replace=False)]
            c, lab, _ = kmeans_lloyd(torch.from_numpy(np.ascontiguousarray(data)).to(dev), k, max_iter,
                                     torch.from_numpy(init).to(dev))
            return c.cpu().numpy(), lab.cpu().numpy()

        t0 = time.perf_counter()
        np.random.seed(args.seed)
        want, want_meta, _ = so.encode(a, args.level, codebook_fit=lambda v: fits[0], kmeans=chunk_kmeans)
        so.assert_sog_equal(host, enc.meta, want, want_meta)
        n = len(r)
        diff = {}
        for i, ax in enumerate("xyz"):
            g = host["means_l.webp"].reshape(-1, 4)[:n, i].astype(np.int64) | \
                host["means_u.webp"].reshape(-1, 4)[:n, i].astype(np.int64) << 8
            w = want["means_l.webp"].reshape(-1, 4)[:n, i].astype(np.int64) | \
                want["means_u.webp"].reshape(-1, 4)[:n, i].astype(np.int64) << 8
            diff[ax] = int(np.count_nonzero(g != w))
        da = int(np.count_nonzero(host["sh0.webp"].reshape(-1, 4)[:n, 3] != want["sh0.webp"].reshape(-1, 4)[:n, 3]))
        out["parity"] = {"ok": True, "means_u16_differing": diff, "sh0_alpha_differing": da,
                         "oracle_s": round(time.perf_counter() - t0, 1)}
    out["card_after"] = card()
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(s + "\n")


if __name__ == "__main__":
    main()

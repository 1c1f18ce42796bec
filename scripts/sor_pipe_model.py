"""What k_sor_knn spends on the warp-collective pipe, set against what the SM can do (DESIGN.md 4.2).  Needs a GPU.

Part (a): a micro-kernel times dependence-free streams of shfl.idx, shfl.up, vote.ballot, redux.min and FADD at full
occupancy (64 warps per SM, 8 independent chains per thread) and prints warp-instructions per clock per SM for each --
the measured rates on this card.  Clocks are read with clock64() inside the kernel, so the rate does not depend on the
SM clock the card happens to run at; the wall time of the same launch gives that clock.

Part (b): the c2 cloud (10 M points, `mixed` and `uniform`, k = 16) with want_stats=True: collective operations per
query by class, the pipe-clocks they imply at the rates of (a), and the measured kernel clocks per query (CUDA events
over 10 launches after warm-up, at the SM clock measured in (a)).

    python scripts/sor_pipe_model.py [n_points]
"""
import ctypes as C
import json
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "3dgsconverter_b200"))

MICRO_CU = r"""
#include <cuda_runtime.h>
#define FULL 0xffffffffu
constexpr int CHAINS = 8;
template <int OP>
__global__ void __launch_bounds__(256) k_stream(unsigned* out, long long* clocks, int iters, unsigned salt) {
    const int lane = threadIdx.x & 31;
    unsigned a[CHAINS];
#pragma unroll
    for (int j = 0; j < CHAINS; ++j) a[j] = threadIdx.x * 2654435761u + j + salt;
    const float fs = __uint_as_float(0x3f800000u + (salt & 1u));
    __syncthreads();
    const long long t0 = clock64();
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < CHAINS; ++j) {
            if (OP == 0) a[j] = __shfl_sync(FULL, a[j], (int)a[j]);   // source lane = value mod 32: nothing to fold
            if (OP == 1) a[j] = __shfl_up_sync(FULL, a[j], 1);
            if (OP == 2) a[j] = __ballot_sync(FULL, (int)a[j] < (int)salt) + lane;
            if (OP == 3) a[j] = __reduce_min_sync(FULL, a[j]) + lane;
            if (OP == 4) a[j] = __float_as_uint(__fadd_rn(__uint_as_float(a[j]), fs));
        }
    }
    const long long t1 = clock64();
    unsigned s = 0;
#pragma unroll
    for (int j = 0; j < CHAINS; ++j) s ^= a[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) clocks[blockIdx.x] = t1 - t0;
}
// one launch of 8 CTAs of 256 threads per SM; returns the largest per-CTA clock count and the wall time
extern "C" int run_stream(int op, int iters, int sms, long long* max_clocks, float* ms) {
    const int blocks = sms * 8;
    unsigned* out; long long* clk;
    if (cudaMalloc(&out, (size_t)blocks * 256 * 4) || cudaMalloc(&clk, (size_t)blocks * 8)) return 1;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int rep = 0; rep < 2; ++rep) {   // the first launch warms up
        cudaEventRecord(e0);
        switch (op) {
            case 0: k_stream<0><<<blocks, 256>>>(out, clk, iters, 7u); break;
            case 1: k_stream<1><<<blocks, 256>>>(out, clk, iters, 7u); break;
            case 2: k_stream<2><<<blocks, 256>>>(out, clk, iters, 7u); break;
            case 3: k_stream<3><<<blocks, 256>>>(out, clk, iters, 7u); break;
            default: k_stream<4><<<blocks, 256>>>(out, clk, iters, 7u); break;
        }
        cudaEventRecord(e1);
        if (cudaEventSynchronize(e1)) return 2;
    }
    cudaEventElapsedTime(ms, e0, e1);
    long long* h = new long long[blocks];
    cudaMemcpy(h, clk, (size_t)blocks * 8, cudaMemcpyDeviceToHost);
    long long m = 0;
    for (int b = 0; b < blocks; ++b) m = h[b] > m ? h[b] : m;
    *max_clocks = m;
    delete[] h;
    cudaFree(out); cudaFree(clk);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return cudaGetLastError() ? 3 : 0;
}
"""
OPS = ("shfl", "shfl_up", "ballot", "redux_min", "fadd")
# ballot and redux_min carry one integer add per operation (keeps the chain lane-dependent); the ALUs issue 4 per clock


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return q


def pipe_rates(sms, iters=20_000):
    with tempfile.TemporaryDirectory() as td:
        src, so = Path(td) / "pipe_micro.cu", Path(td) / "pipe_micro.so"
        src.write_text(MICRO_CU)
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
                        "-ccbin", "/usr/bin/g++", "-o", str(so), str(src)], check=True)
        lib = C.CDLL(str(so))
        lib.run_stream.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_float)]
        rates, mhz = {}, []
        for op, name in enumerate(OPS):
            clk, ms = C.c_longlong(0), C.c_float(0)
            rc = lib.run_stream(op, iters, sms, C.byref(clk), C.byref(ms))
            if rc:
                raise RuntimeError(f"micro-kernel {name} failed ({rc})")
            warp_instr_per_sm = 64 * iters * 8          # 64 warps per SM x iters x 8 chains
            rates[name] = warp_instr_per_sm / clk.value
            mhz.append(clk.value / (ms.value * 1e3))
        return rates, sorted(mhz)[len(mhz) // 2]


def model(st, rates):
    """Collective operations per query by class -> (table, pipe-clocks per query).  Operation counts per event are
    read off csrc/gsx_sor.cu for K <= 32; the tau refreshes of serial steps are bounded by min(inserts, scan steps -
    merges); the broadcasts done once per cell change and once per batch (under 0.3 per query) are left out."""
    q = st["queries"]
    serial_steps = min(st["inserts"], st["scan_steps"] - st["merges_first"] - st["merges_full"])
    ops = {   # class: (events, shfl, shfl_up, ballot, redux)
        "serial insert": (st["inserts"], 1, 1, 0, 0),
        "tau refresh of a serial step (upper bound)": (serial_steps, 1, 0, 0, 0),
        "first merge (sort only)": (st["merges_first"], 15 + 1, 0, 1, 0),
        "full merge": (st["merges_full"], 15 + 1 + 5 + 1, 0, 1, 0),
        "scan step (pass ballot)": (st["scan_steps"], 0, 0, 1, 0),
        "probe visit": (st["probe_visits"], 2, 0, 0, 1),
        "probe loop exit": (q, 0, 0, 0, 1),
        "super visit": (st["super_visits"], 0, 0, 0, 1),
        "chunk visit": (st["chunk_visits"], 0, 0, 0, 1),
        "chunk group exit": (st["chunk_groups"], 0, 0, 0, 1),
    }
    rows, total = [], 0.0
    for name, (ev, sh, up, bal, red) in ops.items():
        clocks = ev / q * (sh / rates["shfl"] + up / rates["shfl_up"] + bal / rates["ballot"] + red / rates["redux_min"])
        total += clocks
        rows.append((name, ev / q, sh + up, bal, red, clocks))
    return rows, total


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sor_pipe_model.py needs a CUDA device")
    from gsx import _abi, sor, synth
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    dev = torch.device("cuda:0")
    sms = _abi.lib.gsx_device_sm_count()
    print(f"card: {card()}  ({sms} SMs)")
    print(f"build: {_abi.lib.gsx_build_info().decode()}")
    rates, mhz = pipe_rates(sms)
    print(f"(a) warp-instructions per clock per SM, 64 warps/SM, 8 chains/thread; SM clock under load {mhz:.0f} MHz")
    for name in OPS:
        print(f"    {name:10s} {rates[name]:6.3f}")
    for kind in ("mixed", "uniform"):
        xyz = torch.from_numpy(synth.xyz(n, kind)).to(dev)
        grid = sor.build_grid(xyz)
        out = torch.empty(n, dtype=torch.float32, device=dev)
        _, st = sor.mean_dists(grid, 16, "i32wrap", out=out, want_stats=True)
        for _ in range(3):
            sor.mean_dists(grid, 16, "i32wrap", out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            sor.mean_dists(grid, 16, "i32wrap", out=out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        measured = ms * 1e-3 * mhz * 1e6 * sms / st["queries"]
        rows, total = model(st, rates)
        print(f"(b) {kind} n={n} k=16 i32wrap: k_sor_knn {ms:.3f} ms = {measured:.1f} SM-clocks per query")
        print(f"    scanned/query {st['scanned'] / n:.1f}  box tests/query {st['box_tests'] / n:.1f}")
        print(f"    {'class':44s} {'per query':>9s} {'shfl':>4s} {'vote':>4s} {'redux':>5s} {'pipe-clocks':>11s}")
        for name, per_q, sh, bal, red, clocks in rows:
            print(f"    {name:44s} {per_q:9.2f} {sh:4d} {bal:4d} {red:5d} {clocks:11.1f}")
        print(f"    modelled {total:.1f} pipe-clocks per query = {100 * total / measured:.0f} % of the measured {measured:.1f}")
        print("    " + json.dumps({"kind": kind, "n": n, "knn_ms": round(ms, 3), "counters": st}))
        del xyz, grid, out


if __name__ == "__main__":
    main()

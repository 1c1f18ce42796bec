// gsx_kmeans.cu -- batched Lloyd K-Means (SOG codebooks) for sm_90a (H100).
//
// Replaces gpu_ops.py:57-73 (k_means_assign), :75-96 (k_means_update) and the loop at :186-188.
// Arithmetic contract: SURVEY A.5 -- strict float32, no fma: dist = (((0 + d0^2) + d1^2) + ...),
// strict '<' with the lowest centroid index winning ties, min_dist = 1e20, update = float32 sums
// accumulated serially in point-index order, inv = 1.0f/cnt, empty clusters collapse to 0.
//
// Design:
//   * all independent problems (the <= 64 spatial chunks of sog.py:527-549) run in ONE launch per
//     phase; a CTA works on a tile of points of one problem.
//   * assign: x rows live in registers (D is a template parameter), centroids are staged through
//     shared memory in tiles and read as broadcast float4; every thread runs P points x 2 centroids
//     = 2P independent accumulation chains, so the dependent FADD chain of the contract does not
//     stall the FP32 pipes.  The contract's rounding sequence is not a GEMM; the tensor-core form
//     (gsx_kmeans_tc.cu) uses a GEMM score only to pick candidates for this same strict distance.
//   * update: a stable partition of the point indices by label (per-warp shared-memory counters,
//     match.any ranks -- O(N)), then one warp per (problem, cluster) walks its member list in index
//     order with 8 row loads in flight and accumulates lane-per-dimension.  This reproduces the
//     oracle's serial index-order float32 sum bit-for-bit and is run-to-run deterministic (the
//     reference's float atomics are neither).  K > 2047 falls back to a per-cluster label scan.
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_kmeans.cuh"

#include <vector>

namespace gsx {

#define GSX_FULL 0xffffffffu
constexpr int kAssignThreads = 128;
constexpr int kCentTile = 64;  // centroids per shared-memory tile


constexpr int kSubTile = 1024;     // points per warp in the stable label partition
constexpr int kMaxSortK = 2047;    // clusters (+1 overflow bin) whose per-warp counters fit shared memory

template <int D>
struct PointsPerThread {
    static constexpr int value = D <= 4 ? 4 : (D <= 24 ? 2 : 2);
};

template <int D, int P>
__global__ void __launch_bounds__(kAssignThreads)
    k_kmeans_assign(const float* __restrict__ X, const float* __restrict__ C, int* __restrict__ labels,
                    const KmProb* __restrict__ probs, int nprob, int K) {
    constexpr int DP = (D + 3) / 4 * 4;  // padded row stride in shared memory (float4 aligned)
    constexpr int G = DP / 4;
    __shared__ __align__(16) float sc[kCentTile * DP];

    // which problem does this tile belong to?
    int lo = 0, hi = nprob - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (probs[mid].tile0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const KmProb pr = probs[lo];
    const long long tile = (long long)blockIdx.x - pr.tile0;
    const float* Cp = C + (size_t)lo * K * D;

    float x[P][DP];
    long long row[P];
    bool live[P];
#pragma unroll
    for (int p = 0; p < P; ++p) {
        long long r = tile * (kAssignThreads * P) + p * kAssignThreads + threadIdx.x;
        live[p] = r < pr.rows;
        row[p] = pr.row0 + (live[p] ? r : 0);
        const float* xr = X + (size_t)row[p] * D;
#pragma unroll
        for (int d = 0; d < DP; ++d) x[p][d] = d < D ? xr[d] : 0.f;
    }
    float best_d[P];
    int best_k[P];
#pragma unroll
    for (int p = 0; p < P; ++p) {
        best_d[p] = 1e20f;
        best_k[p] = -1;
    }

    for (int k0 = 0; k0 < K; k0 += kCentTile) {
        const int kt = K - k0 < kCentTile ? K - k0 : kCentTile;
        __syncthreads();
        for (int t = threadIdx.x; t < kCentTile * DP; t += kAssignThreads) {
            int c = t / DP, d = t - c * DP;
            sc[t] = (c < kt && d < D) ? Cp[(size_t)(k0 + c) * D + d] : 0.f;
        }
        __syncthreads();
        // two centroids per step; an odd tail centroid is paired with a zero row and ignored
        for (int c = 0; c < kt; c += 2) {
            float acc0[P], acc1[P];
#pragma unroll
            for (int p = 0; p < P; ++p) acc0[p] = acc1[p] = 0.f;
            const float4* r0 = reinterpret_cast<const float4*>(sc + c * DP);
            const float4* r1 = reinterpret_cast<const float4*>(sc + (c + 1 < kCentTile ? c + 1 : c) * DP);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float4 a = r0[g], b = r1[g];
                const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (g * 4 + e < D) {
#pragma unroll
                        for (int p = 0; p < P; ++p) {
                            float d0 = __fsub_rn(x[p][g * 4 + e], av[e]);
                            acc0[p] = __fadd_rn(acc0[p], __fmul_rn(d0, d0));
                            float d1 = __fsub_rn(x[p][g * 4 + e], bv[e]);
                            acc1[p] = __fadd_rn(acc1[p], __fmul_rn(d1, d1));
                        }
                    }
                }
            }
#pragma unroll
            for (int p = 0; p < P; ++p) {
                if (acc0[p] < best_d[p]) {
                    best_d[p] = acc0[p];
                    best_k[p] = k0 + c;
                }
                if (c + 1 < kt && acc1[p] < best_d[p]) {
                    best_d[p] = acc1[p];
                    best_k[p] = k0 + c + 1;
                }
            }
        }
    }
#pragma unroll
    for (int p = 0; p < P; ++p)
        if (live[p]) labels[row[p]] = best_k[p];
}

// any D: one point per thread, x re-read through L1 (slow path for unusual dimensions)
__global__ void __launch_bounds__(kAssignThreads)
    k_kmeans_assign_generic(const float* __restrict__ X, const float* __restrict__ C, int* __restrict__ labels,
                            const KmProb* __restrict__ probs, int nprob, int K, int D) {
    int lo = 0, hi = nprob - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (probs[mid].tile0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const KmProb pr = probs[lo];
    long long r = ((long long)blockIdx.x - pr.tile0) * kAssignThreads + threadIdx.x;
    if (r >= pr.rows) return;
    const float* xr = X + (size_t)(pr.row0 + r) * D;
    const float* Cp = C + (size_t)lo * K * D;
    float best = 1e20f;
    int bk = -1;
    for (int c = 0; c < K; ++c) {
        float acc = 0.f;
        for (int d = 0; d < D; ++d) {
            float df = __fsub_rn(xr[d], __ldg(Cp + (size_t)c * D + d));
            acc = __fadd_rn(acc, __fmul_rn(df, df));
        }
        if (acc < best) {
            best = acc;
            bk = c;
        }
    }
    labels[pr.row0 + r] = bk;
}

// one warp per (problem, cluster): serial index-order float32 sums, then the 1/cnt scaling
__global__ void __launch_bounds__(256)
    k_kmeans_update(const float* __restrict__ X, float* __restrict__ C, const int* __restrict__ labels,
                    int* __restrict__ counts, const KmProb* __restrict__ probs, int nprob, int K, int D) {
    const int lane = threadIdx.x & 31;
    const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wid >= (long long)nprob * K) return;
    const int p = (int)(wid / K), c = (int)(wid - (long long)p * K);
    const KmProb pr = probs[p];
    const int* lab = labels + pr.row0;
    const float* Xp = X + (size_t)pr.row0 * D;
    float* out = C + ((size_t)p * K + c) * D;
    int cnt = 0;
    for (int d0 = 0; d0 < D; d0 += 64) {  // lanes cover dims d0+lane and d0+32+lane
        const int da = d0 + lane, db = d0 + 32 + lane;
        float sa = 0.f, sb = 0.f;
        int n_here = 0;
        for (long long base = 0; base < pr.rows; base += 32) {
            long long i = base + lane;
            bool hit = i < pr.rows && __ldg(lab + i) == c;
            unsigned m = __ballot_sync(GSX_FULL, hit);
            n_here += __popc(m);
            while (m) {
                int src = __ffs(m) - 1;
                m &= m - 1;
                const float* xr = Xp + (size_t)(base + src) * D;
                if (da < D) sa = __fadd_rn(sa, __ldg(xr + da));
                if (db < D) sb = __fadd_rn(sb, __ldg(xr + db));
            }
        }
        cnt = n_here;
        if (cnt > 0) {
            float inv = __fdiv_rn(1.0f, (float)cnt);
            sa = __fmul_rn(sa, inv);
            sb = __fmul_rn(sb, inv);
        }
        if (da < D) out[da] = sa;
        if (db < D) out[db] = sb;
    }
    if (lane == 0) counts[(size_t)p * K + c] = cnt;
}

// ---------------------------------------------------------------------------------------------
// Update, O(N) form: a stable partition of the point indices by label, then one warp per cluster
// walks its member list in index order.  Same sums, bit for bit, as the serial oracle; every phase
// is deterministic.  hist is [n_subtiles][K+1] (bin K collects label -1 rows, never accumulated).

__device__ __forceinline__ int find_problem_by_sub(const KmProb* __restrict__ probs, int nprob, int sub) {
    int lo = 0, hi = nprob - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (probs[mid].sub0 <= sub) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// phase 1: per-sub-tile label histogram (one warp per sub-tile, shared-memory counters)
__global__ void __launch_bounds__(256)
    k_km_hist(const int* __restrict__ labels, const KmProb* __restrict__ probs, int nprob, int K, int nsub,
              int* __restrict__ hist) {
    extern __shared__ int s_cnt[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int sub = blockIdx.x * 8 + w;
    if (sub >= nsub) return;
    int* cnt = s_cnt + w * (K + 1);
    for (int k = lane; k <= K; k += 32) cnt[k] = 0;
    __syncwarp();
    const int p = find_problem_by_sub(probs, nprob, sub);
    const KmProb pr = probs[p];
    const long long r0 = (long long)(sub - pr.sub0) * kSubTile;
    const long long r1 = r0 + kSubTile < pr.rows ? r0 + kSubTile : pr.rows;
    const int* lab = labels + pr.row0;
    for (long long i = r0 + lane; i < r1; i += 32) {
        int l = lab[i];
        atomicAdd(cnt + (l >= 0 && l < K ? l : K), 1);
    }
    __syncwarp();
    for (int k = lane; k <= K; k += 32) hist[(size_t)sub * (K + 1) + k] = cnt[k];
}

// phase 2: per (problem, cluster) exclusive prefix over the problem's sub-tiles; totals -> counts
__global__ void __launch_bounds__(256)
    k_km_scan(const KmProb* __restrict__ probs, int nprob, int K, int nsub_total, int* __restrict__ hist,
              int* __restrict__ totals) {
    const int p = blockIdx.y;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > K) return;
    const int s0 = probs[p].sub0;
    const int s1 = p + 1 < nprob ? probs[p + 1].sub0 : nsub_total;
    int run = 0;
#pragma unroll 8
    for (int sidx = s0; sidx < s1; ++sidx) {
        size_t at = (size_t)sidx * (K + 1) + k;
        int v = hist[at];
        hist[at] = run;
        run += v;
    }
    totals[(size_t)p * (K + 1) + k] = run;
}

// phase 3: cluster offsets inside the problem (exclusive scan over k of the totals), counts out
__global__ void k_km_offsets(int nprob, int K, const int* __restrict__ totals, int* __restrict__ offs,
                             int* __restrict__ counts) {
    const int p = blockIdx.x;
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    // block-wide scan in strips of blockDim.x
    for (int base = 0; base <= K; base += blockDim.x) {
        int k = base + threadIdx.x;
        int v = k <= K ? totals[(size_t)p * (K + 1) + k] : 0;
        if (k < K) counts[(size_t)p * K + k] = v;
        // inclusive warp scan, then scan of warp sums through shared memory
        int x = v;
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(GSX_FULL, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        __shared__ int wsum[32];
        if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int ws = threadIdx.x < (blockDim.x >> 5) ? wsum[threadIdx.x] : 0;
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(GSX_FULL, ws, o);
                if (threadIdx.x >= o) ws += y;
            }
            wsum[threadIdx.x] = ws;
        }
        __syncthreads();
        int excl = carry + (threadIdx.x >> 5 ? wsum[(threadIdx.x >> 5) - 1] : 0) + x - v;
        if (k <= K) offs[(size_t)p * (K + 1) + k] = excl;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = excl + v;
        __syncthreads();
    }
}

// phase 4: stable scatter of the row indices (problem-local) into cluster order
__global__ void __launch_bounds__(256)
    k_km_scatter(const int* __restrict__ labels, const KmProb* __restrict__ probs, int nprob, int K, int nsub,
                 const int* __restrict__ hist, const int* __restrict__ offs, int* __restrict__ member) {
    extern __shared__ int s_cnt[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int sub = blockIdx.x * 8 + w;
    if (sub >= nsub) return;
    int* cnt = s_cnt + w * (K + 1);
    const int p = find_problem_by_sub(probs, nprob, sub);
    const KmProb pr = probs[p];
    for (int k = lane; k <= K; k += 32) cnt[k] = offs[(size_t)p * (K + 1) + k] + hist[(size_t)sub * (K + 1) + k];
    __syncwarp();
    const long long r0 = (long long)(sub - pr.sub0) * kSubTile;
    const long long r1 = r0 + kSubTile < pr.rows ? r0 + kSubTile : pr.rows;
    const int* lab = labels + pr.row0;
    int* mem = member + pr.row0;
    for (long long base = r0; base < r1; base += 32) {
        const long long i = base + lane;
        const bool act = i < r1;
        int l = act ? lab[i] : -2 - lane;  // inactive lanes get unique dummy keys
        int bin = act ? (l >= 0 && l < K ? l : K) : l;
        unsigned peers = __match_any_sync(GSX_FULL, bin);
        int rank = __popc(peers & ((1u << lane) - 1u));
        int pos = 0;
        if (act) pos = cnt[bin] + rank;
        __syncwarp();
        if (act && rank == 0) cnt[bin] += __popc(peers);
        __syncwarp();
        if (act) mem[pos] = (int)i;
    }
}

// phase 5: one warp per (problem, cluster): serial index-order float32 sums over the member list.
// The chain of adds is inherently sequential (float32 addition does not associate), but it is short (~3 000 adds);
// what limits the warp is the latency of gathering its ~3 000 rows.  So a whole batch of 32 member rows is put in
// flight at once (64 independent loads per lane) before the 32 dependent adds are issued, in index order.
__global__ void __launch_bounds__(128)
    k_km_accum(const float* __restrict__ X, float* __restrict__ C, const int* __restrict__ member,
               const int* __restrict__ offs, const int* __restrict__ counts, const KmProb* __restrict__ probs,
               int nprob, int K, int D) {
    const int lane = threadIdx.x & 31;
    const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wid >= (long long)nprob * K) return;
    const int p = (int)(wid / K), c = (int)(wid - (long long)p * K);
    const KmProb pr = probs[p];
    const int cnt = counts[(size_t)p * K + c];
    const int* mem = member + pr.row0 + offs[(size_t)p * (K + 1) + c];
    const float* Xp = X + (size_t)pr.row0 * D;
    float* out = C + ((size_t)p * K + c) * D;
    const float inv = cnt > 0 ? __fdiv_rn(1.0f, (float)cnt) : 0.f;
    for (int d0 = 0; d0 < D; d0 += 64) {
        const int da = d0 + lane, db = d0 + 32 + lane;
        const bool ha = da < D, hb = db < D;
        const int oa = ha ? da : 0, ob = hb ? db : 0;  // clamped: every load is in bounds, unused lanes add nothing
        float sa = 0.f, sb = 0.f;
        int base = 0;
        int mine = lane < cnt ? __ldg(mem + lane) : 0;
        for (; base + 32 <= cnt; base += 32) {
            const int nxt = base + 32 + lane < cnt ? __ldg(mem + base + 32 + lane) : 0;  // next batch's indices
            float va[32], vb[32];
#pragma unroll
            for (int t = 0; t < 32; ++t) {
                const float* xr = Xp + (size_t)__shfl_sync(GSX_FULL, mine, t) * D;
                va[t] = __ldg(xr + oa);
                vb[t] = __ldg(xr + ob);
            }
#pragma unroll
            for (int t = 0; t < 32; ++t) {
                sa = __fadd_rn(sa, va[t]);
                sb = __fadd_rn(sb, vb[t]);
            }
            mine = nxt;
        }
        const int nn = cnt - base;  // ragged tail (< 32 rows)
        for (int u = 0; u < nn; ++u) {
            const float* xr = Xp + (size_t)__shfl_sync(GSX_FULL, mine, u) * D;
            sa = __fadd_rn(sa, __ldg(xr + oa));
            sb = __fadd_rn(sb, __ldg(xr + ob));
        }
        if (cnt > 0) {
            sa = __fmul_rn(sa, inv);
            sb = __fmul_rn(sb, inv);
        }
        if (ha) out[da] = sa;
        if (hb) out[db] = sb;
    }
}

static long long total_subtiles(const int64_t* row_off, int nprob) {
    long long t = 0;
    for (int p = 0; p < nprob; ++p) t += (row_off[p + 1] - row_off[p] + kSubTile - 1) / kSubTile;
    return t;
}

struct KmWs {
    KmProb* probs;
    int* member;
    int* hist;
    int* totals;
    int* offs;
    int* err;
    size_t total;
    bool ok;
};

static KmWs km_carve(void* ws, size_t bytes, int64_t n_total, int nprob, int K, long long nsub) {
    KmWs w;
    Carver c(ws, bytes);
    w.probs = c.take<KmProb>(nprob);
    w.member = c.take<int>((size_t)n_total);
    const bool sorted = K <= kMaxSortK;
    w.hist = c.take<int>(sorted ? (size_t)nsub * (K + 1) : 1);
    w.totals = c.take<int>(sorted ? (size_t)nprob * (K + 1) : 1);
    w.offs = c.take<int>(sorted ? (size_t)nprob * (K + 1) : 1);
    w.err = c.take<int>(8);
    w.total = align_up(c.off, 256);
    w.ok = c.ok();
    return w;
}

template <int D>
static void launch_assign(const float* X, const float* C, int* labels, const KmProb* probs, int nprob, int K,
                          int tiles, cudaStream_t st) {
    constexpr int P = PointsPerThread<D>::value;
    k_kmeans_assign<D, P><<<tiles, kAssignThreads, 0, st>>>(X, C, labels, probs, nprob, K);
}

static int points_per_thread(int D) {
    switch (D) {
        case 1: return PointsPerThread<1>::value;
        case 2: return PointsPerThread<2>::value;
        case 3: return PointsPerThread<3>::value;
        case 4: return PointsPerThread<4>::value;
        case 9: return PointsPerThread<9>::value;
        case 24: return PointsPerThread<24>::value;
        case 45: return PointsPerThread<45>::value;
        default: return 1;
    }
}

}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_kmeans_workspace_bytes(int64_t n_total, int32_t nprob, int32_t K, int32_t D) {
    (void)D;
    if (nprob < 1) nprob = 1;
    if (n_total < 1) n_total = 1;
    // worst case number of sub-tiles: every problem adds at most one partial tile
    long long nsub = n_total / kSubTile + nprob + 1;
    KmWs w = km_carve(nullptr, 0, n_total, nprob, K, nsub);
    return (int64_t)w.total + 1024;
}

int gsx_kmeans_lloyd_device(const float* X, const int64_t* row_off, int32_t nprob, int32_t K, int32_t D,
                            int32_t max_iter, float* C, int32_t* labels, int32_t* counts, void* ws, int64_t ws_bytes,
                            int32_t assign_mode, unsigned long long* tc_stats, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::kmeans_lloyd");
    GSX_REQUIRE(assign_mode == GSX_KM_ASSIGN_AUTO || assign_mode == GSX_KM_ASSIGN_STRICT ||
                    assign_mode == GSX_KM_ASSIGN_TENSOR,
                GSX_ERR_ARG, "kmeans: bad assign_mode %d", assign_mode);
    if (assign_mode == GSX_KM_ASSIGN_TENSOR)
        GSX_REQUIRE(kmeans_tc_supported(K, D), GSX_ERR_UNSUPPORTED,
                    "kmeans: tensor-core assign needs D in {9,24,45} and K <= 256 (got K=%d D=%d)", K, D);
    const bool use_tc = assign_mode == GSX_KM_ASSIGN_TENSOR ||
                        (assign_mode == GSX_KM_ASSIGN_AUTO && kmeans_tc_supported(K, D));
    GSX_REQUIRE(nprob >= 1 && K >= 1 && D >= 1 && max_iter >= 0, GSX_ERR_ARG, "kmeans: bad shape");
    const int64_t n_total = row_off[nprob] - row_off[0];
    GSX_REQUIRE(row_off[0] == 0, GSX_ERR_ARG, "kmeans: row_off[0] must be 0");
    GSX_REQUIRE(ws_bytes >= gsx_kmeans_workspace_bytes(n_total, nprob, K, D), GSX_ERR_WORKSPACE,
                "kmeans: workspace too small");
    const int per_tile = kAssignThreads * points_per_thread(D);
    std::vector<KmProb> hp(nprob);
    long long tiles = 0, nsub = 0, tc_tiles = 0;
    for (int p = 0; p < nprob; ++p) {
        hp[p].row0 = row_off[p];
        hp[p].rows = row_off[p + 1] - row_off[p];
        GSX_REQUIRE(hp[p].rows >= 1, GSX_ERR_ARG, "kmeans: empty problem %d", p);
        GSX_REQUIRE(hp[p].rows < 2147483647ll, GSX_ERR_UNSUPPORTED, "kmeans: problem %d has too many rows", p);
        hp[p].tile0 = (int)tiles;
        hp[p].sub0 = (int)nsub;
        hp[p].tc_tile0 = tc_tiles;
        tc_tiles += (hp[p].rows + 127) / 128;
        tiles += (hp[p].rows + per_tile - 1) / per_tile;
        nsub += (hp[p].rows + kSubTile - 1) / kSubTile;
    }
    GSX_REQUIRE(tiles < 2147483647ll, GSX_ERR_UNSUPPORTED, "kmeans: too many tiles");
    GSX_REQUIRE(nsub == total_subtiles(row_off, nprob), GSX_ERR_ARG, "kmeans: internal tile count mismatch");
    KmWs w = km_carve(ws, (size_t)ws_bytes, n_total, nprob, K, nsub);
    GSX_REQUIRE(w.ok, GSX_ERR_WORKSPACE, "kmeans: workspace too small");
    KmProb* dp = w.probs;
    GSX_CUDA_CHECK(cudaMemcpyAsync(dp, hp.data(), hp.size() * sizeof(KmProb), cudaMemcpyHostToDevice, st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));  // hp is a local pageable buffer
    const long long uwarps = (long long)nprob * K;
    const int ublocks = (int)((uwarps * 32 + 255) / 256);
    const int ablocks = (int)((uwarps * 32 + 127) / 128);
    const bool sorted = K <= kMaxSortK;
    const size_t smem = (size_t)8 * (K + 1) * sizeof(int);
    if (sorted && smem > 48 * 1024) {
        GSX_CUDA_CHECK(cudaFuncSetAttribute(k_km_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        GSX_CUDA_CHECK(cudaFuncSetAttribute(k_km_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    if (use_tc) GSX_CUDA_CHECK(cudaMemsetAsync(w.err, 0, sizeof(int), st));
    for (int it = 0; it < max_iter; ++it) {
        if (use_tc) {
            int rc = kmeans_assign_tc(X, (long long)n_total * D, C, labels, dp, nprob, K, D, tc_tiles, 0, nullptr,
                                      tc_stats, w.err, st);
            if (rc) return rc;
        } else
        switch (D) {
            case 1: launch_assign<1>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            case 2: launch_assign<2>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            case 3: launch_assign<3>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            case 4: launch_assign<4>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            case 9: launch_assign<9>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            case 24: launch_assign<24>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            case 45: launch_assign<45>(X, C, labels, dp, nprob, K, (int)tiles, st); break;
            default:
                k_kmeans_assign_generic<<<(int)tiles, kAssignThreads, 0, st>>>(X, C, labels, dp, nprob, K, D);
        }
        GSX_KERNEL_CHECK();
        if (!sorted) {  // very large K: O(N*K/32) label scan per cluster (no shared-memory counters needed)
            k_kmeans_update<<<ublocks, 256, 0, st>>>(X, C, labels, counts, dp, nprob, K, D);
            GSX_KERNEL_CHECK();
            continue;
        }
        const int sblocks = (int)((nsub + 7) / 8);
        k_km_hist<<<sblocks, 256, smem, st>>>(labels, dp, nprob, K, (int)nsub, w.hist);
        GSX_KERNEL_CHECK();
        k_km_scan<<<dim3((K + 1 + 255) / 256, nprob), 256, 0, st>>>(dp, nprob, K, (int)nsub, w.hist, w.totals);
        GSX_KERNEL_CHECK();
        k_km_offsets<<<nprob, 256, 0, st>>>(nprob, K, w.totals, w.offs, counts);
        GSX_KERNEL_CHECK();
        k_km_scatter<<<sblocks, 256, smem, st>>>(labels, dp, nprob, K, (int)nsub, w.hist, w.offs, w.member);
        GSX_KERNEL_CHECK();
        k_km_accum<<<ablocks, 128, 0, st>>>(X, C, w.member, w.offs, counts, dp, nprob, K, D);
        GSX_KERNEL_CHECK();
    }
    if (use_tc && max_iter > 0) {  // a timed-out mbarrier wait inside the tensor-core kernel (protocol bug) is an error
        int herr = 0;
        GSX_CUDA_CHECK(cudaMemcpyAsync(&herr, w.err, sizeof(int), cudaMemcpyDeviceToHost, st));
        GSX_CUDA_CHECK(cudaStreamSynchronize(st));
        GSX_REQUIRE(herr == 0, GSX_ERR_CUDA, "kmeans: tensor-core assign kernel timed out on an mbarrier");
    }
    return GSX_OK;
}

// debug / test hook: raw tensor-core scores of the first 128 rows against K centroids (one problem)
int gsx_kmeans_tc_debug_scores(const float* X, int64_t rows, const float* C, int32_t K, int32_t D, float* scores,
                               void* ws, int64_t ws_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(kmeans_tc_supported(K, D) && rows >= 1, GSX_ERR_UNSUPPORTED, "kmeans_tc_debug: unsupported shape");
    GSX_REQUIRE(ws_bytes >= 1024, GSX_ERR_WORKSPACE, "kmeans_tc_debug: workspace too small");
    KmProb hp;
    hp.row0 = 0, hp.rows = rows, hp.tile0 = 0, hp.sub0 = 0, hp.tc_tile0 = 0;
    KmProb* dp = reinterpret_cast<KmProb*>(ws);
    int* err = reinterpret_cast<int*>(reinterpret_cast<char*>(ws) + 512);
    GSX_CUDA_CHECK(cudaMemcpyAsync(dp, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
    GSX_CUDA_CHECK(cudaMemsetAsync(err, 0, sizeof(int), st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    int rc = kmeans_assign_tc(X, (long long)rows * D, C, nullptr, dp, 1, K, D, (rows + 127) / 128, 1, scores,
                              nullptr, err, st);
    if (rc) return rc;
    GSX_KERNEL_CHECK();
    int herr = 0;
    GSX_CUDA_CHECK(cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    GSX_REQUIRE(herr == 0, GSX_ERR_CUDA, "kmeans_tc_debug: mbarrier wait timed out");
    return GSX_OK;
}

}  // extern "C"

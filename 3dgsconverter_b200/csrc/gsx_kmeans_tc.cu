// gsx_kmeans_tc.cu -- K-Means assign step on the Hopper tensor cores (wgmma, TF32), sm_90a.
//
// Replaces gpu_ops.py:57-73 (k_means_assign) with bit-identical labels.  The contract (SURVEY A.5) is a strict
// float32 (sub, mul, add -- no fma, dims ascending) distance per (point, centroid), lowest index winning ties;
// that rounding sequence is not a GEMM.  What IS a GEMM is the score
//        s_c = x . c - 0.5 ||c||^2            (E_c = ||x||^2 - 2 s_c is the squared distance),
// so the kernel
//   1. computes S = [X | 1 1 1] . [C | b_hi b_mid b_lo]^T  for a tile of 128 points x (up to) 256 centroids with
//      wgmma.mma_async ... .tf32 (A = the points, B = the centroids, both K-major in shared memory; each of the two
//      warpgroups owns 64 point rows and holds their float32 scores in registers); the bias -0.5||c||^2 is split
//      into three TF32-exact pieces and rides in three padding columns of the K dimension, so the bias costs
//      nothing and adds no rounding;
//   2. takes the row maximum (a row is spread over the four threads of a quad in the wgmma accumulator layout) and
//      builds the set of centroids whose score is within a rounding-error margin M of it;
//   3. evaluates the strict contract distance only for those candidates (one candidate: it IS the answer, no
//      evaluation at all), ascending index, strict '<' -- the quad then keeps the lexicographic minimum of
//      (distance, index), which is exactly what the serial ascending scan returns.
// Margin (DESIGN.md 4.6): with |s~_c - t_c| <= eta for every centroid (t_c the real-arithmetic score, s~_c what
// the tensor core returns) and |a_c - E_c| <= g E_c for the strict float32 distance a_c, the contract's answer
// c* satisfies  s~_{c*} >= s~_max - (2 eta + g/(1-g) E_{c'}),  E_{c'} <= ||x||^2 - 2 s~_max + 2 eta.
// eta covers the TF32 conversion of both operands (relative 2^-10 each, truncation or rounding), the tensor
// core's float32 accumulation and the float32 evaluation of the bias; the kernel uses twice the proven bound.
// Anything non-finite, or an empty candidate set, falls back to the full strict scan inside the same kernel, so
// the labels are bit-identical to k_kmeans_assign in every case (tests/test_kmeans_tc_gpu.py).
//
// Data movement: a tile is 128 consecutive rows of X = 128*D*4 contiguous bytes; one elected thread moves it
// global -> shared with a 1-D TMA bulk copy (cp.async.bulk, completion on an mbarrier) one tile ahead of the
// MMA, then every thread re-lays its half row into the GMMA canonical K-major layout (no swizzle).
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_kmeans.cuh"

namespace gsx {

#define GSX_FULL 0xffffffffu

constexpr int kTcThreads = 256;   // two warpgroups; for the operand re-layout: two threads per point row
constexpr int kTcRows = 128;      // points per tile: 2 x wgmma M=64
constexpr int kTcMaxN = 256;      // max centroids of the tensor-core path (4 x wgmma N=64)
constexpr long long kWaitCycles = 1ll << 31;   // ~1 s: a protocol bug reports an error instead of hanging the GPU

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// returns false on timeout
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    const long long t0 = clock64();
    for (unsigned spin = 0;; ++spin) {
        if ((spin & 1023u) == 1023u && clock64() - t0 > kWaitCycles) break;
        uint32_t ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(addr), "r"(parity)
            : "memory");
        if (ok) return true;
    }
    return false;
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// GMMA shared-memory descriptor, K-major, no swizzle (layout type 0, cute::GMMA::GmmaDescriptor): core matrix =
// 8 rows x 16 B stored as 128 contiguous bytes, lbo = byte distance of the two core matrices adjacent in K,
// sbo = byte distance of adjacent 8-row groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
// d[64 x 64] (+)= A[64 x 8] . B[64 x 8]^T, TF32 inputs, float32 accumulate; issued by the whole warpgroup
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,"
        "%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA
template <int NB>
__device__ __forceinline__ void acc_fence(float (&acc)[NB][32]) {
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
        for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(acc[b][i])::"memory");
}

__device__ __forceinline__ float tf32_trunc(float v) { return __uint_as_float(__float_as_uint(v) & 0xFFFFE000u); }

// byte offset of element (row, k) of a K-major operand with KP (multiple of 8) padded K columns
template <int KP>
__device__ __forceinline__ uint32_t op_off(int row, int k) {
    return (uint32_t)((row >> 3) * (KP / 4) * 128 + (k >> 2) * 128 + (row & 7) * 16 + (k & 3) * 4);
}

struct TcShared {  // tail of the dynamic shared memory (after the operand tiles and the staging buffer)
    uint64_t bar_copy;
    float red[8];
    float xn[2][kTcRows];    // partial ||x||^2 of the two half rows
};

// Work split: 256 threads = 2 warpgroups.  Warpgroup g computes the scores of the tile rows 64g .. 64g+63 against
// NB*64 centroid columns.  In the accumulator layout, thread (warp w, lane l) of the warpgroup holds the rows
// 16(w%4) + l/4 and +8 and, in every 64-column block, the columns 8j + 2(l%4) + {0,1}, j = 0..7: register
// acc[b][4j + 2i + e] is (row + 8i, column 64b + 8j + 2(l%4) + e).  The four threads of a quad share their rows.
// mode 0: labels; mode 1 (debug): dump the raw scores of the first tile to dump[128*npad] and return
template <int D, int KP, int NB>
__global__ void __launch_bounds__(kTcThreads, 1)
    k_km_assign_tc(const float* __restrict__ X, long long x_floats, const float* __restrict__ C,
                   int* __restrict__ labels, const KmProb* __restrict__ probs, int nprob, int K, int npad,
                   long long tiles_total, int mode, float* __restrict__ dump, unsigned long long* __restrict__ tc_stats,
                   int* __restrict__ err_flag) {
    static_assert(KP % 8 == 0 && KP >= D + 3, "K padding");
    constexpr int NT = NB * 64;             // centroid columns computed (padding columns score -3e38)
    constexpr int G4 = KP / 4;              // float4 groups per operand row
    constexpr int GH = (G4 + 1) / 2;        // groups re-laid by the lower-half thread of a row
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char* sB = smem;                                   // [kTcMaxN x KP] float32, GMMA K-major layout
    unsigned char* sA = sB + kTcMaxN * KP * 4;                  // [128 x KP]
    float* sStage = reinterpret_cast<float*>(sA + kTcRows * KP * 4);  // 128*D floats + 8 (alignment slack)
    TcShared* sh = reinterpret_cast<TcShared*>(reinterpret_cast<unsigned char*>(sStage) + (kTcRows * D + 8) * 4);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // operand re-layout: thread -> (row, half of the K groups)
    const int lrow = (warp & 3) * 32 + lane, half = warp >> 2;
    // epilogue: thread -> two rows and the quad's column pattern
    const int wg = warp >> 2, quad = lane & 3;
    const int erow0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    if (tid == 0) {
        mbar_init(&sh->bar_copy, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const long long t0 = tiles_total * (long long)blockIdx.x / gridDim.x;
    const long long t1 = tiles_total * (long long)(blockIdx.x + 1) / gridDim.x;
    const bool x_aligned = (reinterpret_cast<uintptr_t>(X) & 15) == 0;
    constexpr uint32_t kLbo = 128u, kSbo = (uint32_t)G4 * 128u;
    constexpr float kU = 5.9604645e-8f;                        // 2^-24
    constexpr float kGs = 2.f * (D + 3) * kU * 1.02f;          // >= 2 gamma_{D+2} / (1 - gamma_{D+2})
    constexpr float kEpsIn = 1.953125e-3f * 1.01f;             // 2^-9 (+): two TF32 conversions, 2^-10 each
    constexpr float kEpsAcc = 3.0517578e-5f;                   // 2^-15: accumulation + bias evaluation slack

    struct TileGeo { int p; long long row0; int rows; long long off_floats; bool bulk; uint32_t pre, bytes; };
    auto geo = [&](long long t) {
        TileGeo g;
        int lo = 0, hi = nprob - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (probs[mid].tc_tile0 <= t) lo = mid; else hi = mid - 1;
        }
        g.p = lo;
        const long long lt = t - probs[lo].tc_tile0;
        const long long left = probs[lo].rows - lt * kTcRows;
        g.rows = left < kTcRows ? (int)left : kTcRows;
        g.row0 = probs[lo].row0 + lt * kTcRows;
        g.off_floats = g.row0 * D;
        const long long ob = g.off_floats * 4;
        g.pre = (uint32_t)(ob & 15);
        g.bytes = (g.pre + (uint32_t)g.rows * D * 4 + 15u) & ~15u;
        g.bulk = x_aligned && ((ob - g.pre) + g.bytes <= x_floats * 4);
        return g;
    };

    uint32_t copy_phase = 0;
    bool failed = false;
    TileGeo cur{};
    if (t0 < t1) {
        cur = geo(t0);
        if (tid == 0 && cur.bulk) {
            mbar_expect_tx(&sh->bar_copy, cur.bytes);
            bulk_g2s(sStage, reinterpret_cast<const char*>(X) + (cur.off_floats * 4 - cur.pre), cur.bytes, &sh->bar_copy);
        }
    }
    int cur_prob = -1;
    float Cm = 0.f;
    unsigned long long st_strict = 0, st_multi = 0, st_full = 0;
    float acc[NB][32];

    for (long long t = t0; t < t1; ++t) {
        const TileGeo g = cur;
        const float* Cp = C + (size_t)g.p * K * D;
        if (g.p != cur_prob) {  // (re)load the centroids of this problem as the B operand
            for (int idx = tid; idx < NT * G4; idx += kTcThreads) {
                const int c = idx / G4, j = idx - c * G4;
                float v[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int k = 4 * j + e;
                    v[e] = (c < K && k < D) ? __ldg(Cp + (size_t)c * D + k) : 0.f;
                }
                *reinterpret_cast<float4*>(sB + op_off<KP>(c, 4 * j)) = make_float4(v[0], v[1], v[2], v[3]);
            }
            __syncthreads();
            float mx = 0.f;
            for (int c = tid; c < NT; c += kTcThreads) {
                float cn = 0.f;
                if (c < K) {
                    for (int k = 0; k < D; ++k) {
                        const float v = *reinterpret_cast<const float*>(sB + op_off<KP>(c, k));
                        cn = __fmaf_rn(v, v, cn);
                    }
                }
                mx = fmaxf(mx, cn);
                // bias = -0.5||c||^2 as three TF32-exact pieces; padding centroids get a huge negative score
                const float b = c < K ? -0.5f * cn : -3.0e38f;
                const float bh = tf32_trunc(b);
                const float r1 = c < K ? b - bh : 0.f;       // exact: the low 13 bits
                const float bm = tf32_trunc(r1);
                const float bl = c < K ? r1 - bm : 0.f;      // <= 2 significant bits left: TF32-exact
                *reinterpret_cast<float*>(sB + op_off<KP>(c, D)) = bh;
                *reinterpret_cast<float*>(sB + op_off<KP>(c, D + 1)) = bm;
                *reinterpret_cast<float*>(sB + op_off<KP>(c, D + 2)) = bl;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(GSX_FULL, mx, o));
            if (lane == 0) sh->red[warp] = mx;
            __syncthreads();
            mx = sh->red[0];
#pragma unroll
            for (int w = 1; w < kTcThreads / 32; ++w) mx = fmaxf(mx, sh->red[w]);
            Cm = sqrtf(mx) * 1.0001f;  // inf/NaN propagate into the margin -> full strict scan below
            cur_prob = g.p;
        }

        // ---- this thread's half row: staging (bulk copy) or global -> GMMA layout, partial ||x||^2 on the way
        if (g.bulk) {
            if (!mbar_wait(&sh->bar_copy, copy_phase)) failed = true;
            copy_phase ^= 1;
        }
        {
            const bool live = lrow < g.rows;
            const float* src = g.bulk ? sStage + (g.pre >> 2) + lrow * D : X + g.off_floats + (long long)lrow * D;
            float xa = 0.f, xb = 0.f;  // two chains
            const int j0 = half == 0 ? 0 : GH, j1 = half == 0 ? GH : G4;
#pragma unroll
            for (int jj = 0; jj < GH; ++jj) {
                const int j = j0 + jj;
                if (j < j1) {
                    float v[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int k = 4 * j + e;
                        if (k < D) {
                            v[e] = live ? src[k] : 0.f;
                            if (e & 1) xb = __fmaf_rn(v[e], v[e], xb); else xa = __fmaf_rn(v[e], v[e], xa);
                        } else {
                            v[e] = k < D + 3 ? 1.0f : 0.f;
                        }
                    }
                    *reinterpret_cast<float4*>(sA + op_off<KP>(lrow, 4 * j)) = make_float4(v[0], v[1], v[2], v[3]);
                }
            }
            sh->xn[half][lrow] = xa + xb;
        }
        fence_proxy_async();   // generic-proxy writes of sA / sB -> visible to the tensor core (async proxy)
        if (__syncthreads_or(failed)) {
            failed = true;
            break;
        }
        if (t + 1 < t1) cur = geo(t + 1);
        if (tid == 0 && t + 1 < t1 && cur.bulk) {  // staging is free: every thread has copied its half row out
            mbar_expect_tx(&sh->bar_copy, cur.bytes);
            bulk_g2s(sStage, reinterpret_cast<const char*>(X) + (cur.off_floats * 4 - cur.pre), cur.bytes, &sh->bar_copy);
        }

        // ---- scores of this warpgroup's 64 rows: NB blocks of 64 columns, KP/8 TF32 k-steps each
        {
            const uint32_t a0 = smem_u32(sA) + (uint32_t)(wg * 8) * kSbo, b0 = smem_u32(sB);
            acc_fence<NB>(acc);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int j = 0; j < KP / 8; ++j)  // one instruction = 8 TF32 along K = two core matrices = 256 B
                    wgmma_tf32_n64(acc[b], gmma_desc(a0 + (uint32_t)j * 256u, kLbo, kSbo),
                                   gmma_desc(b0 + (uint32_t)(b * 8) * kSbo + (uint32_t)j * 256u, kLbo, kSbo), j > 0);
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            acc_fence<NB>(acc);
        }

        if (mode == 1) {  // debug: raw scores of the tile
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int r = 0; r < 32; ++r) {
                    const int row = erow0 + 8 * ((r >> 1) & 1);
                    const int col = 64 * b + 8 * (r >> 2) + 2 * quad + (r & 1);
                    if (col < npad) dump[(size_t)row * npad + col] = acc[b][r];
                }
            break;
        }

        // ---- epilogue, for each of this thread's two rows
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = erow0 + 8 * i;
            const bool live = row < g.rows;
            // pass 1: row maximum over this thread's columns, then over the quad
            float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    m0 = fmaxf(m0, acc[b][4 * j + 2 * i]);
                    m1 = fmaxf(m1, acc[b][4 * j + 2 * i + 1]);
                }
            float smax = fmaxf(m0, m1);
            smax = fmaxf(smax, __shfl_xor_sync(GSX_FULL, smax, 1));
            smax = fmaxf(smax, __shfl_xor_sync(GSX_FULL, smax, 2));
            const float xn = sh->xn[0][row] + sh->xn[1][row];
            const float xnu = xn * 1.0001f;
            const float xnorm = sqrtf(xnu) * 1.0001f;
            const float eta = (kEpsIn * xnorm * Cm + kEpsAcc * (xnorm * Cm + Cm * Cm)) * 1.5f + 1e-37f;
            const float e_ub = fmaxf(xnu - 2.f * smax + 2.f * eta, 0.f);
            const float marg = 2.f * eta + kGs * e_ub;
            const float thr = smax - marg;
            // pass 2: candidate mask of this thread's columns; bit 16b + 2j + e <-> column 64b + 8j + 2 quad + e
            uint64_t mask = 0;
#pragma unroll
            for (int b = 0; b < NB; ++b)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (acc[b][4 * j + 2 * i] >= thr) mask |= 1ull << (16 * b + 2 * j);
                    if (acc[b][4 * j + 2 * i + 1] >= thr) mask |= 1ull << (16 * b + 2 * j + 1);
                }
            const int cnt = __popcll(mask);
            int total = cnt + __shfl_xor_sync(GSX_FULL, cnt, 1);
            total += __shfl_xor_sync(GSX_FULL, total, 2);
            // the shortcut is only legal when the margin is finite, a real centroid scored, and the strict distance
            // of the winner cannot reach the contract's 1e20 "no label" sentinel.  The quad agrees on all of it.
            const bool bad = !(marg < 3.0e38f) || !(smax > -1.0e30f) || !(e_ub < 1.0e19f) || total == 0;
            auto col_of = [&](int bit) { return 64 * (bit >> 4) + 8 * ((bit & 15) >> 1) + 2 * quad + (bit & 1); };
            if (!bad && total == 1 && cnt == 1 && live) labels[g.row0 + row] = col_of(__ffsll((long long)mask) - 1);
            const bool need = live && (bad || total > 1);
            if (!need) {
                mask = 0;
            } else if (bad) {  // full strict scan over the real centroids of this thread
                mask = 0;
#pragma unroll
                for (int bit = 0; bit < NB * 16; ++bit)
                    if (col_of(bit) < K) mask |= 1ull << bit;
            }
            float best = 1e20f;
            int bk = -1;
            while (mask) {  // ascending column order
                const int c = col_of(__ffsll((long long)mask) - 1);
                mask &= mask - 1;
                float a = 0.f;
#pragma unroll
                for (int j = 0; j < (D + 3) / 4; ++j) {
                    const float4 xv = *reinterpret_cast<const float4*>(sA + op_off<KP>(row, 4 * j));
                    const float4 cv = *reinterpret_cast<const float4*>(sB + op_off<KP>(c, 4 * j));
                    const float xa[4] = {xv.x, xv.y, xv.z, xv.w}, ca[4] = {cv.x, cv.y, cv.z, cv.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (4 * j + e < D) {
                            const float df = __fsub_rn(xa[e], ca[e]);
                            a = __fadd_rn(a, __fmul_rn(df, df));
                        }
                }
                ++st_strict;
                if (a < best) best = a, bk = c;
            }
            // quad: lexicographic minimum of (distance, index) == the serial ascending scan with strict '<'
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                const float ob = __shfl_xor_sync(GSX_FULL, best, o);
                const int ok = __shfl_xor_sync(GSX_FULL, bk, o);
                if (ob < best || (ob == best && ok >= 0 && (bk < 0 || ok < bk))) best = ob, bk = ok;
            }
            if (need && quad == 0) {
                labels[g.row0 + row] = bk;
                ++st_multi;
                if (bad) ++st_full;
            }
        }
        __syncthreads();  // sA is rewritten for the next tile only after every strict evaluation and MMA read it
    }

    if (failed && err_flag) atomicExch(err_flag, 1);
    if (tc_stats) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            st_strict += __shfl_xor_sync(GSX_FULL, st_strict, o);
            st_multi += __shfl_xor_sync(GSX_FULL, st_multi, o);
            st_full += __shfl_xor_sync(GSX_FULL, st_full, o);
        }
        if (lane == 0) {
            atomicAdd(tc_stats + 0, st_strict);
            atomicAdd(tc_stats + 1, st_multi);
            atomicAdd(tc_stats + 2, st_full);
        }
    }
}

template <int D, int KP, int NB>
static int launch_tc(const float* X, long long x_floats, const float* C, int* labels, const KmProb* probs, int nprob,
                     int K, long long tiles, int mode, float* dump, unsigned long long* stats, int* err,
                     cudaStream_t st) {
    const int npad = (K + 31) / 32 * 32;
    const size_t smem = (size_t)(kTcMaxN + kTcRows) * KP * 4 + (size_t)(kTcRows * D + 8) * 4 + sizeof(TcShared) + 64;
    static int per_sm = 0;
    if (per_sm == 0) {
        GSX_CUDA_CHECK(cudaFuncSetAttribute(k_km_assign_tc<D, KP, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)smem));
        GSX_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_km_assign_tc<D, KP, NB>, kTcThreads, smem));
        if (per_sm < 1) per_sm = 1;
    }
    long long grid = (long long)sm_count() * per_sm;
    if (grid > tiles) grid = tiles;
    if (mode == 1) grid = 1;
    if (grid < 1) grid = 1;
    k_km_assign_tc<D, KP, NB><<<(int)grid, kTcThreads, smem, st>>>(X, x_floats, C, labels, probs, nprob, K, npad, tiles,
                                                                   mode, dump, stats, err);
    return GSX_OK;
}

template <int D, int KP>
static int launch_tc_n(const float* X, long long x_floats, const float* C, int* labels, const KmProb* probs, int nprob,
                       int K, long long tiles, int mode, float* dump, unsigned long long* stats, int* err,
                       cudaStream_t st) {
    if (K <= 64) return launch_tc<D, KP, 1>(X, x_floats, C, labels, probs, nprob, K, tiles, mode, dump, stats, err, st);
    if (K <= 128) return launch_tc<D, KP, 2>(X, x_floats, C, labels, probs, nprob, K, tiles, mode, dump, stats, err, st);
    return launch_tc<D, KP, 4>(X, x_floats, C, labels, probs, nprob, K, tiles, mode, dump, stats, err, st);
}

bool kmeans_tc_supported(int K, int D) { return (D == 9 || D == 24 || D == 45) && K >= 1 && K <= kTcMaxN; }

int kmeans_assign_tc(const float* X, long long x_floats, const float* C, int* labels, const KmProb* probs_dev, int nprob,
                     int K, int D, long long tiles, int mode, float* dump, unsigned long long* stats,
                     int* err_flag_dev, cudaStream_t st) {
    switch (D) {
        case 9: return launch_tc_n<9, 16>(X, x_floats, C, labels, probs_dev, nprob, K, tiles, mode, dump, stats, err_flag_dev, st);
        case 24: return launch_tc_n<24, 32>(X, x_floats, C, labels, probs_dev, nprob, K, tiles, mode, dump, stats, err_flag_dev, st);
        case 45: return launch_tc_n<45, 48>(X, x_floats, C, labels, probs_dev, nprob, K, tiles, mode, dump, stats, err_flag_dev, st);
        default: set_error("kmeans_tc: unsupported D=%d", D); return GSX_ERR_UNSUPPORTED;
    }
}

}  // namespace gsx

extern "C" int32_t gsx_kmeans_tensor_core_supported(int32_t K, int32_t D) {
    return gsx::kmeans_tc_supported(K, D) ? 1 : 0;
}

// gsx_stats.cu -- np.mean / np.std of a float32 vector, bit-for-bit, on device; threshold mask.
//
// Replaces gpu_ops.py:259-263 and data_processor.py:176-180 (glob_mean/glob_std/threshold/mask).
// NumPy reduces float32 with float32 accumulators in a fixed *pairwise* order (SURVEY A.1 step 9):
//   n < 8      : serial
//   n <= 128   : 8 interleaved accumulators, ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), serial tail
//   otherwise  : split at n2 = n/2 - (n/2)%8, sum(left) + sum(right)
// The split tree depends only on n, so it parallelises exactly: one thread per leaf block walks the
// tree from the root along the bits of its slot index, sums its <=128 elements in NumPy's order, and
// the inner nodes are then combined bottom-up in place (left + right, one float add per node).
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_sor.cuh"

#include <set>

namespace gsx {

static int pairwise_depth(int64_t n) {
    std::set<int64_t> level{n};
    int d = 0;
    for (;;) {
        std::set<int64_t> next;
        for (int64_t m : level)
            if (m > 128) {
                int64_t n2 = m / 2;
                n2 -= n2 % 8;
                next.insert(n2);
                next.insert(m - n2);
            }
        if (next.empty()) return d;
        // leaves (<=128) at this depth stay where they are; only split nodes go deeper
        level.swap(next);
        ++d;
    }
}

size_t mean_std_ws_bytes(int64_t n) {
    if (n < 1) n = 1;
    int d = pairwise_depth(n);
    return (((size_t)1 << d) + 64) * sizeof(float);
}

// walk from the root `depth` levels along the bits of `path` (MSB first).  Returns false if the
// walk hits a leaf (size <= 128) before `depth` levels; else sets (off, m) of the node reached.
__device__ __forceinline__ bool walk(int64_t n, int depth, uint32_t path, int64_t& off, int64_t& m, int& reached) {
    off = 0;
    m = n;
    for (int l = 0; l < depth; ++l) {
        if (m <= 128) {
            reached = l;
            return false;
        }
        int64_t n2 = m / 2;
        n2 -= n2 % 8;
        if ((path >> (depth - 1 - l)) & 1u) {
            off += n2;
            m -= n2;
        } else {
            m = n2;
        }
    }
    reached = depth;
    return true;
}

template <bool SQ>
__device__ __forceinline__ float elem(const float* __restrict__ a, int64_t i, float mean) {
    float v = a[i];
    if (SQ) {
        float t = __fsub_rn(v, mean);
        v = __fmul_rn(t, t);
    }
    return v;
}

// One leaf = 8 consecutive lanes: lane j IS NumPy's accumulator r[j] (elements j, j+8, j+16, ... of the leaf), so the
// 8 lanes read one 32-byte sector per step; the combine ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) is a 3-step xor butterfly
// (float addition is commutative, so both lanes of a pair compute the same bits); lane 0 adds the serial tail.
template <bool SQ, class Get>
__device__ __forceinline__ float leaf_sum8(int64_t off, int64_t m, int j, Get get) {
    const unsigned grp = 0xffu << ((threadIdx.x & 31) & ~7);
    float res;
    if (m < 8) {
        res = 0.f;
        if (j == 0)
            for (int64_t i = 0; i < m; ++i) res = __fadd_rn(res, get(off + i));
        return res;
    }
    // a leaf has at most 128 elements = 16 per lane: issue all the loads first (independent), then the ordered adds
    const int64_t body = m - (m % 8);
    const int cnt = (int)(body >> 3);
    float vals[16];
#pragma unroll
    for (int k = 0; k < 16; ++k)
        if (k < cnt) vals[k] = get(off + 8 * k + j);
    float r = vals[0];
#pragma unroll
    for (int k = 1; k < 16; ++k)
        if (k < cnt) r = __fadd_rn(r, vals[k]);
    r = __fadd_rn(r, __shfl_xor_sync(grp, r, 1));
    r = __fadd_rn(r, __shfl_xor_sync(grp, r, 2));
    r = __fadd_rn(r, __shfl_xor_sync(grp, r, 4));
    res = r;
    if (j == 0)
        for (int64_t i = body; i < m; ++i) res = __fadd_rn(res, get(off + i));
    return res;
}

template <bool SQ>
__global__ void __launch_bounds__(128) k_pw_leaves(const float* __restrict__ a, int64_t n, int dmax,
                                                   const float* __restrict__ meanp, float* __restrict__ slot) {
    const uint64_t gt = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t t = (uint32_t)(gt >> 3);
    const int j = (int)(gt & 7);
    if (t >= (1u << dmax)) return;   // (a whole group of 8 leaves together: the shuffles below stay converged)
    int64_t off, m;
    int reached;
    bool full = walk(n, dmax, t, off, m, reached);
    if (!full) {
        // a leaf at depth `reached` < dmax: owned by the slot whose remaining low bits are zero
        if (t & ((1u << (dmax - reached)) - 1u)) return;
    }
    const float mean = SQ ? meanp[0] : 0.f;
    const float res = leaf_sum8<SQ>(off, m, j, [&](int64_t i) { return elem<SQ>(a, i, mean); });
    if (j == 0) slot[t] = res;
}

// Fast path when `a` is 16-byte aligned (every leaf offset is a multiple of 8 elements): TWO lanes per leaf, lane h holds
// NumPy's accumulators r[4h .. 4h+3] and reads one float4 per step, so a warp sums 16 leaves with 16-byte loads (the
// 8-lane form issues 4x the instructions per byte and was instruction-bound: ~300 instructions per thread, most of
// them the tree walk).  All loads of a lane are issued before its ordered adds.
template <bool SQ>
__global__ void __launch_bounds__(128) k_pw_leaves2(const float* __restrict__ a, int64_t n, int dmax,
                                                    const float* __restrict__ meanp, float* __restrict__ slot) {
    const uint64_t gt = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t t = (uint32_t)(gt >> 1);
    const int h = (int)(gt & 1);
    if (t >= (1u << dmax)) return;   // (both lanes of a leaf together: the shuffle below stays converged)
    int64_t off, m;
    int reached;
    const bool full = walk(n, dmax, t, off, m, reached);
    if (!full && (t & ((1u << (dmax - reached)) - 1u))) return;
    const float mean = SQ ? meanp[0] : 0.f;
    const unsigned pair = 3u << ((threadIdx.x & 31) & ~1);
    float res;
    if (m < 8) {
        res = 0.f;
        if (h == 0)
            for (int64_t i = 0; i < m; ++i) res = __fadd_rn(res, elem<SQ>(a, off + i, mean));
    } else {
        const int64_t body = m - (m % 8);
        const int cnt = (int)(body >> 3);   // <= 16 steps of 8 elements
        const float4* p = reinterpret_cast<const float4*>(a + off) + h;
        float4 v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k)
            if (k < cnt) v[k] = __ldg(p + 2 * k);
        if (SQ) {
#pragma unroll
            for (int k = 0; k < 16; ++k)
                if (k < cnt) {
                    float tx = __fsub_rn(v[k].x, mean), ty = __fsub_rn(v[k].y, mean), tz = __fsub_rn(v[k].z, mean),
                          tw = __fsub_rn(v[k].w, mean);
                    v[k] = make_float4(__fmul_rn(tx, tx), __fmul_rn(ty, ty), __fmul_rn(tz, tz), __fmul_rn(tw, tw));
                }
        }
        float4 r = v[0];
#pragma unroll
        for (int k = 1; k < 16; ++k)
            if (k < cnt) {
                r.x = __fadd_rn(r.x, v[k].x), r.y = __fadd_rn(r.y, v[k].y);
                r.z = __fadd_rn(r.z, v[k].z), r.w = __fadd_rn(r.w, v[k].w);
            }
        // ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7)): the two inner sums are this lane's and the partner's
        const float half = __fadd_rn(__fadd_rn(r.x, r.y), __fadd_rn(r.z, r.w));
        const float other = __shfl_xor_sync(pair, half, 1);
        res = h == 0 ? __fadd_rn(half, other) : __fadd_rn(other, half);
        if (h == 0)
            for (int64_t i = body; i < m; ++i) res = __fadd_rn(res, elem<SQ>(a, off + i, mean));
    }
    if (h == 0) slot[t] = res;
}

// combine the nodes of depth d: node u = left(u) + right(u), in place at the left child's slot
__device__ __forceinline__ void combine_node(int64_t n, int dmax, int d, uint32_t u, float* slot) {
    int64_t off, m;
    int reached;
    if (!walk(n, d, u, off, m, reached)) return;  // no such node (an ancestor is a leaf)
    if (m <= 128) return;                         // a leaf: already final
    size_t li = (size_t)u << (dmax - d);
    size_t ri = ((size_t)(2 * u + 1)) << (dmax - d - 1);
    slot[li] = __fadd_rn(slot[li], slot[ri]);
}

// levels dhi..dlo in ONE launch: block b owns the subtree under node b of depth dlo (its slots are touched by no other
// block), so up to 9 tree levels cost one launch instead of nine (the level kernels were ~20 launches of a few
// microseconds each per mean_std, most of its time at 10 M elements)
__global__ void __launch_bounds__(256) k_pw_mid(int64_t n, int dmax, int dhi, int dlo, float* slot) {
    for (int d = dhi; d >= dlo; --d) {
        if (threadIdx.x < (1u << (d - dlo))) combine_node(n, dmax, d, (blockIdx.x << (d - dlo)) + threadIdx.x, slot);
        __syncthreads();
    }
}

// levels dmax-1 .. 10, nine at a time; returns the next level to combine (<= 9)
static int pairwise_mid_levels(int64_t n, int dmax, float* slot, cudaStream_t st) {
    int d = dmax - 1;
    while (d > 9) {
        const int dlo = d - 8 > 10 ? d - 8 : 10;
        k_pw_mid<<<1u << dlo, 1u << (d - dlo), 0, st>>>(n, dmax, d, dlo, slot);
        d = dlo - 1;
    }
    return d;
}

// levels dtop..0 in one block, then the final division (and sqrt for the variance pass)
template <bool SQ>
__global__ void __launch_bounds__(1024) k_pw_top(int64_t n, int dmax, int dtop, float* slot, float* out) {
    for (int d = dtop; d >= 0; --d) {
        if (threadIdx.x < (1u << d)) combine_node(n, dmax, d, threadIdx.x, slot);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // NumPy divides the float32 sum by the element COUNT (an intp scalar): float32 / int64 promotes to float64, and the
        // quotient is then rounded to float32 (_methods.py: ret.dtype.type(ret / rcount), true_divide(..., casting='unsafe')).
        // Up to 2^24 elements that equals the float32 division; beyond, float32(n) is no longer n and it does not.
        float v = __double2float_rn(__ddiv_rn((double)slot[0], (double)n));
        if (SQ) out[1] = __fsqrt_rn(v);
        else out[0] = v;
    }
}

template <bool SQ>
static int pairwise_pass(const float* a, int64_t n, int dmax, float* slot, float* out, cudaStream_t st) {
    uint32_t leaves = 1u << dmax;
    if ((reinterpret_cast<uintptr_t>(a) & 15) == 0)
        k_pw_leaves2<SQ><<<(unsigned)(((uint64_t)leaves * 2 + 127) / 128), 128, 0, st>>>(a, n, dmax, out, slot);
    else
        k_pw_leaves<SQ><<<(unsigned)(((uint64_t)leaves * 8 + 127) / 128), 128, 0, st>>>(a, n, dmax, out, slot);
    GSX_KERNEL_CHECK();
    const int d = pairwise_mid_levels(n, dmax, slot, st);
    GSX_KERNEL_CHECK();
    k_pw_top<SQ><<<1, 1024, 0, st>>>(n, dmax, d, slot, out);  // d may be -1 (single leaf): loop is skipped
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int mean_std_f32(const float* a, int64_t n, float* out_dev, void* ws, size_t ws_bytes, cudaStream_t st) {
    GSX_NVTX("gsx::mean_std_f32");
    GSX_REQUIRE(n >= 1, GSX_ERR_ARG, "mean_std: n must be >= 1");
    GSX_REQUIRE(ws_bytes >= mean_std_ws_bytes(n), GSX_ERR_WORKSPACE, "mean_std: workspace too small");
    int dmax = pairwise_depth(n);
    GSX_REQUIRE(dmax <= 31, GSX_ERR_UNSUPPORTED, "mean_std: n too large");
    float* slot = (float*)ws;
    int rc = pairwise_pass<false>(a, n, dmax, slot, out_dev, st);
    if (rc) return rc;
    return pairwise_pass<true>(a, n, dmax, slot, out_dev, st);
}

// ---------------------------------------------------------------------------------------------------------
// Sharded form (one process per GPU): the vector of n elements is cut into contiguous slabs, rank r holds
// a[bases[r] .. bases[r+1]).  NumPy's tree depends only on n, so every leaf (<= 128 consecutive elements) is
// summed by the rank whose slab contains the leaf's FIRST element; the (at most 127) elements of a leaf that
// spill into the following slabs come from `halo` = the first 128 elements of every slab (all-gathered by the
// caller).  Every slot is written by exactly one rank (0 elsewhere), so an all-reduce(sum) of the slot array is
// exact; the inner nodes are then combined replicated (pairwise_finish).  Same bits as mean_std_f32 on the
// concatenated vector.
template <bool SQ>
__global__ void __launch_bounds__(128)
    k_pw_leaves_dist(const float* __restrict__ a_local, int64_t base, int64_t n_local, int64_t n, int dmax,
                     const float* __restrict__ meanp, const float* __restrict__ halo,
                     const long long* __restrict__ bases, int world, float* __restrict__ slot) {
    const uint64_t gt = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t t = (uint32_t)(gt >> 3);
    const int j = (int)(gt & 7);
    if (t >= (1u << dmax)) return;
    int64_t off, m;
    int reached;
    bool full = walk(n, dmax, t, off, m, reached);
    if (!full && (t & ((1u << (dmax - reached)) - 1u))) return;
    if (off < base || off >= base + n_local) return;  // another rank owns this leaf
    const float mean = SQ ? meanp[0] : 0.f;
    auto get = [&](int64_t i) -> float {
        float v;
        if (i < base + n_local) {
            v = a_local[i - base];
        } else {   // spill-over into the following slab(s): the first 128 elements of every slab are in `halo`
            int hr = 0;
            while (hr + 1 < world && i >= bases[hr + 1]) ++hr;
            v = halo[(size_t)hr * 128 + (i - bases[hr])];
        }
        if (SQ) {
            float d = __fsub_rn(v, mean);
            v = __fmul_rn(d, d);
        }
        return v;
    };
    const float res = leaf_sum8<SQ>(off, m, j, get);
    if (j == 0) slot[t] = res;
}

// gpu_ops.py:261-263: thresh = mean + f32(tf) * std (float32 mul then add), mask = a < thresh
__global__ void __launch_bounds__(256) k_threshold_mask(const float* __restrict__ a, int64_t n,
                                                        const float* __restrict__ ms, float tf,
                                                        uint8_t* __restrict__ mask) {
    const float thresh = __fadd_rn(ms[0], __fmul_rn(tf, ms[1]));
    int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        float4 v = *reinterpret_cast<const float4*>(a + i);
        uchar4 o = make_uchar4(v.x < thresh, v.y < thresh, v.z < thresh, v.w < thresh);
        *reinterpret_cast<uchar4*>(mask + i) = o;
    } else {
        for (; i < n; ++i) mask[i] = a[i] < thresh;
    }
}

__global__ void __launch_bounds__(256) k_threshold_mask_scalar(const float* __restrict__ a, int64_t n,
                                                               const float* __restrict__ ms, float tf,
                                                               uint8_t* __restrict__ mask) {
    const float thresh = __fadd_rn(ms[0], __fmul_rn(tf, ms[1]));
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) mask[i] = a[i] < thresh;
}

int threshold_mask(const float* a, int64_t n, const float* meanstd_dev, float tf, uint8_t* mask, cudaStream_t st) {
    if (n == 0) return GSX_OK;
    if (((uintptr_t)a % 16 == 0) && ((uintptr_t)mask % 4 == 0)) {
        int64_t nv = (n + 3) / 4;
        k_threshold_mask<<<(int)((nv + 255) / 256), 256, 0, st>>>(a, n, meanstd_dev, tf, mask);
    } else {
        k_threshold_mask_scalar<<<(int)((n + 255) / 256), 256, 0, st>>>(a, n, meanstd_dev, tf, mask);
    }
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_pairwise_slots(int64_t n) {
    if (n < 1) n = 1;
    return (int64_t)1 << pairwise_depth(n);
}

int gsx_pairwise_leaves_dist(const float* a_local, int64_t base, int64_t n_local, int64_t n, int32_t sq,
                             const float* meanstd, const float* halo, const int64_t* bases_dev, int32_t world,
                             float* slot, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 1 && n_local >= 0 && base >= 0 && base + n_local <= n, GSX_ERR_ARG, "pairwise_dist: bad slab");
    int dmax = pairwise_depth(n);
    GSX_REQUIRE(dmax <= 31, GSX_ERR_UNSUPPORTED, "pairwise_dist: n too large");
    uint32_t leaves = 1u << dmax;
    GSX_CUDA_CHECK(cudaMemsetAsync(slot, 0, (size_t)leaves * sizeof(float), st));
    if (n_local == 0) return GSX_OK;
    const unsigned lb = (unsigned)(((uint64_t)leaves * 8 + 127) / 128);
    if (sq)
        k_pw_leaves_dist<true><<<lb, 128, 0, st>>>(a_local, base, n_local, n, dmax, meanstd, halo,
                                                   (const long long*)bases_dev, world, slot);
    else
        k_pw_leaves_dist<false><<<lb, 128, 0, st>>>(a_local, base, n_local, n, dmax, meanstd, halo,
                                                    (const long long*)bases_dev, world, slot);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_pairwise_finish(float* slot, int64_t n, int32_t sq, float* meanstd, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 1, GSX_ERR_ARG, "pairwise_finish: n must be >= 1");
    int dmax = pairwise_depth(n);
    const int d = pairwise_mid_levels(n, dmax, slot, st);
    GSX_KERNEL_CHECK();
    if (sq) k_pw_top<true><<<1, 1024, 0, st>>>(n, dmax, d, slot, meanstd);
    else k_pw_top<false><<<1, 1024, 0, st>>>(n, dmax, d, slot, meanstd);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int64_t gsx_mean_std_workspace_bytes(int64_t n) { return (int64_t)mean_std_ws_bytes(n); }

int gsx_mean_std_f32(const float* a_dev, int64_t n, float* out_dev, void* ws, int64_t ws_bytes, void* stream) {
    return mean_std_f32(a_dev, n, out_dev, ws, (size_t)ws_bytes, (cudaStream_t)stream);
}

int gsx_threshold_mask(const float* a_dev, int64_t n, const float* meanstd_dev, float threshold_factor,
                       uint8_t* mask_dev, void* stream) {
    return threshold_mask(a_dev, n, meanstd_dev, threshold_factor, mask_dev, (cudaStream_t)stream);
}

}  // extern "C"

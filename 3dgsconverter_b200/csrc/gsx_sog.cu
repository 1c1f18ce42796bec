// gsx_sog.cu -- device helpers for the steps either side of K-Means in the SOG writer (SURVEY §8(f) item 1).
//
//   gsx_lexsort_zyx            np.lexsort((z, y, x))                      formats/sog.py:264
//   gsx_quantize_to_codebook   sorted-codebook nearest entry               formats/sog.py:408-419
//
// lexsort: stable LSD over the three float32 keys with our radix sort -- first by z (32 bits), then by the
// 64-bit key x:y -- after mapping floats to order-preserving unsigned ints (-0.0 is folded into +0.0 because
// NumPy compares them equal; every NaN, whatever its sign and payload, gets one key above +inf because NumPy sorts
// NaN last and treats NaNs as equal, so they keep index order).  quantize: lower_bound in the (<= 4096-entry) codebook held in shared memory,
// clip, then the reference's left-neighbour test |v - cb[left]| < |v - cb[idx]| in float32.
#include "../../include/gsx.h"

#include "gsx_bits.cuh"
#include "gsx_common.cuh"
#include "gsx_numpy_scalar.cuh"
#include "gsx_sh_mask.cuh"
#include "gsx_radix.cuh"

namespace gsx {

__global__ void __launch_bounds__(256) k_lex_keys_z(const float* __restrict__ xyz, int64_t n,
                                                    uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = (uint64_t)numpy_sort_key(xyz[3 * i + 2]);
    vals[i] = (int32_t)i;
}

__global__ void __launch_bounds__(256) k_lex_keys_xy(const float* __restrict__ xyz, const int32_t* __restrict__ order,
                                                     int64_t n, uint64_t* __restrict__ keys) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    int64_t i = order[j];
    keys[j] = ((uint64_t)numpy_sort_key(xyz[3 * i]) << 32) | (uint64_t)numpy_sort_key(xyz[3 * i + 1]);
}

constexpr int kMaxCodebook = 4096;

// quantize_to_codebook of sog.py:408-419 for one value against the ascending codebook scb[0..m): np.searchsorted (side
// 'left'; NaN sorts after every number), clip, then the left neighbour if it is strictly closer.  A NaN value gives
// m - 1, as in NumPy.
__device__ __forceinline__ uint8_t codebook_index(const float* scb, int m, float v) {
    int lo = 0, hi = m;  // first index with cb[idx] >= v
    if (v != v) lo = m;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (scb[mid] < v) lo = mid + 1; else hi = mid;
    }
    int idx = lo < m - 1 ? lo : m - 1;          // np.clip(idx, 0, len(cb)-1)
    int left = idx - 1 > 0 ? idx - 1 : 0;        // np.maximum(idx-1, 0)
    float d_idx = fabsf(__fsub_rn(v, scb[idx])), d_left = fabsf(__fsub_rn(v, scb[left]));
    if (d_left < d_idx) idx = left;
    return (uint8_t)idx;                         // .astype(np.uint8)
}

__global__ void __launch_bounds__(256) k_quantize_codebook(const float* __restrict__ vals, int64_t n,
                                                           const float* __restrict__ cb, int m,
                                                           uint8_t* __restrict__ labels) {
    __shared__ float scb[kMaxCodebook];
    for (int t = threadIdx.x; t < m; t += blockDim.x) scb[t] = cb[t];
    __syncthreads();
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        labels[i] = codebook_index(scb, m, vals[i]);
}

// ------------------------------------------------------------------------------------------------------------------
// SogFormat.write on the device (formats/sog.py:258-602).  Every kernel reads record rows through the lexsort order
// (row order[j] is the j-th splat of the file); no sorted copy of the records is made.  Textures are uchar4 [pixels]
// with pixels >= n; the kernels write the padding pixels too.  Float steps are single __f*_rn operations in the
// reference's NumPy-2 float32 order; float -> u8/u16 conversions clip with fmaxf/fminf, which maps NaN to 0 as NumPy
// does on x86.  The logarithm of the positions and the exponential of the opacity are NumPy's SIMD float32 log and exp
// (gsx_numpy_scalar.cuh), so those bytes are exact too.

namespace {

constexpr int kSogMaxCols = 45;
constexpr int kSogMaxChunks = 64;
constexpr int kSogMaxCodebook = 256;
constexpr int kMinmaxBlocks = 1024;

struct SogCols {  // column positions inside a record row
    int32_t c[kSogMaxCols];
    int32_t n;
};

struct SogChunks {  // the shN chunk schedule of sog.py:527-549
    int64_t chunk_size;
    int32_t n;
    int32_t offset[kSogMaxChunks];       // palette index of the chunk's first centroid
    int32_t passthrough[kSogMaxChunks];  // this_k >= len(chunk): the chunk's labels are arange(len)
};

__device__ __forceinline__ float nan_min(float a, float b) { return a != a ? a : (b != b ? b : (b < a ? b : a)); }
__device__ __forceinline__ float nan_max(float a, float b) { return a != a ? a : (b != b ? b : (b > a ? b : a)); }

// sign(v) * log(|v| + 1) (sog.py:279-280): float32 add, NumPy's float32 log (its argument is >= 1 or NaN), float32
// product
__device__ __forceinline__ float log_transform(float v) {
    const float s = v > 0.f ? 1.f : (v < 0.f ? -1.f : (v == 0.f ? 0.f : v));
    return __fmul_rn(s, numpy_logf(__fadd_rn(fabsf(v), 1.f)));
}

// np.clip((l - min) / (max - min) * 65535, 0, 65535).astype(np.uint16) (sog.py:290-292)
__device__ __forceinline__ uint32_t norm_u16(float l, float mn, float mx) {
    const float t = __fmul_rn(__fdiv_rn(__fsub_rn(l, mn), __fsub_rn(mx, mn)), 65535.f);
    return (uint32_t)fminf(fmaxf(t, 0.f), 65535.f);
}

// quantize_vec of sog.py:352-353: np.clip((v * 0.5 + 0.5) * 255.0, 0, 255).astype(np.uint8)
__device__ __forceinline__ uint8_t quat_byte(float v) {
    return (uint8_t)fminf(fmaxf(__fmul_rn(__fadd_rn(__fmul_rn(v, 0.5f), 0.5f), 255.f), 0.f), 255.f);
}

__device__ __forceinline__ int64_t grid_start() { return (int64_t)blockIdx.x * blockDim.x + threadIdx.x; }
__device__ __forceinline__ int64_t grid_stride() { return (int64_t)gridDim.x * blockDim.x; }

// per-block min/max of the three log-transformed position columns (record order: min and max do not depend on it)
__global__ void __launch_bounds__(256) k_sog_log_minmax(const float* __restrict__ rows, int64_t n, int F, int cx, int cy,
                                                        int cz, float* __restrict__ partial) {
    const float inf = __int_as_float(0x7f800000);
    float mn[3] = {inf, inf, inf}, mx[3] = {-inf, -inf, -inf};
    const int c[3] = {cx, cy, cz};
    for (int64_t i = grid_start(); i < n; i += grid_stride()) {
        const float* r = rows + (size_t)i * F;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float l = log_transform(__ldg(r + c[a]));
            mn[a] = nan_min(mn[a], l), mx[a] = nan_max(mx[a], l);
        }
    }
#pragma unroll
    for (int off = 16; off; off >>= 1)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            mn[a] = nan_min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], off));
            mx[a] = nan_max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], off));
        }
    __shared__ float s[8][6];
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int a = 0; a < 3; ++a) s[w][a] = mn[a], s[w][3 + a] = mx[a];
    __syncthreads();
    if (threadIdx.x < 6) {
        const int t = threadIdx.x;
        float v = s[0][t];
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) v = t < 3 ? nan_min(v, s[k][t]) : nan_max(v, s[k][t]);
        partial[blockIdx.x * 6 + t] = v;
    }
}

__global__ void k_sog_minmax_final(const float* __restrict__ partial, int nblocks, float* __restrict__ minmax) {
    const int t = threadIdx.x;
    if (t >= 6) return;
    float v = partial[t];
    for (int b = 1; b < nblocks; ++b) v = t < 3 ? nan_min(v, partial[b * 6 + t]) : nan_max(v, partial[b * 6 + t]);
    minmax[t] = v;
}

// means_l / means_u (sog.py:294-309): low and high bytes of the three u16 positions, alpha 255; padding 255
__global__ void __launch_bounds__(256) k_sog_means(const float* __restrict__ rows, int64_t n, int F,
                                                   const int32_t* __restrict__ order, int cx, int cy, int cz,
                                                   const float* __restrict__ minmax, int64_t pixels,
                                                   uchar4* __restrict__ lo_out, uchar4* __restrict__ hi_out) {
    const float mn0 = minmax[0], mn1 = minmax[1], mn2 = minmax[2];
    const float mx0 = minmax[3], mx1 = minmax[4], mx2 = minmax[5];
    for (int64_t p = grid_start(); p < pixels; p += grid_stride()) {
        if (p >= n) {
            lo_out[p] = hi_out[p] = make_uchar4(255, 255, 255, 255);
            continue;
        }
        const float* r = rows + (size_t)order[p] * F;
        const uint32_t u0 = norm_u16(log_transform(__ldg(r + cx)), mn0, mx0);
        const uint32_t u1 = norm_u16(log_transform(__ldg(r + cy)), mn1, mx1);
        const uint32_t u2 = norm_u16(log_transform(__ldg(r + cz)), mn2, mx2);
        lo_out[p] = make_uchar4(u0 & 255, u1 & 255, u2 & 255, 255);
        hi_out[p] = make_uchar4(u0 >> 8, u1 >> 8, u2 >> 8, 255);
    }
}

// quats (sog.py:315-386): q / norm (serial sum of squares), largest = np.argmax(|q|) (first index wins, a NaN is the
// maximum), q *= sign(q[largest]), q *= np.sqrt(2.0) (a float64 scalar: product in double, rounded to float32), the
// three other components through quantize_vec in ascending order, alpha = 252 + largest; padding 255
__global__ void __launch_bounds__(256) k_sog_quats(const float* __restrict__ rows, int64_t n, int F,
                                                   const int32_t* __restrict__ order, int c0, int c1, int c2, int c3,
                                                   int64_t pixels, uchar4* __restrict__ out) {
    for (int64_t p = grid_start(); p < pixels; p += grid_stride()) {
        if (p >= n) {
            out[p] = make_uchar4(255, 255, 255, 255);
            continue;
        }
        const float* r = rows + (size_t)order[p] * F;
        float q[4] = {__ldg(r + c0), __ldg(r + c1), __ldg(r + c2), __ldg(r + c3)};
        float ss = __fmul_rn(q[0], q[0]);
        ss = __fadd_rn(ss, __fmul_rn(q[1], q[1]));
        ss = __fadd_rn(ss, __fmul_rn(q[2], q[2]));
        ss = __fadd_rn(ss, __fmul_rn(q[3], q[3]));
        const float nrm = __fsqrt_rn(ss);
        int L = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) q[k] = __fdiv_rn(q[k], nrm);
        float best = fabsf(q[0]);
#pragma unroll
        for (int k = 1; k < 4; ++k) {
            const float a = fabsf(q[k]);
            if (best == best && (a > best || a != a)) best = a, L = k;
        }
        float qL = q[0];
#pragma unroll
        for (int k = 1; k < 4; ++k) qL = L == k ? q[k] : qL;
        const float s = qL > 0.f ? 1.f : (qL < 0.f ? -1.f : (qL == 0.f ? 0.f : qL));
        uint8_t b[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
            b[k] = quat_byte(__double2float_rn(__dmul_rn((double)__fmul_rn(q[k], s), 1.4142135623730951)));
        uchar4 o;
        o.x = L == 0 ? b[1] : b[0];
        o.y = L <= 1 ? b[2] : b[1];
        o.z = L <= 2 ? b[3] : b[2];
        o.w = (uint8_t)(252 + L);
        out[p] = o;
    }
}

// out[t] = value s of np.concatenate([col_0, col_1, ...]) in file order, s = sel[t] (or t): the fit data of the 1-D
// codebooks (sog.py:392-400, 435-441) and their K-Means init rows
__global__ void __launch_bounds__(256) k_sog_gather_values(const float* __restrict__ rows, int64_t n, int F,
                                                           const int32_t* __restrict__ order,
                                                           const __grid_constant__ SogCols cols,
                                                           const int64_t* __restrict__ sel, int64_t m,
                                                           float* __restrict__ out) {
    for (int64_t t = grid_start(); t < m; t += grid_stride()) {
        const int64_t s = sel ? sel[t] : t;
        const int64_t a = s / n;
        out[t] = __ldg(rows + (size_t)order[s - a * n] * F + cols.c[a]);
    }
}

// scales (sog.py:421-429) and sh0 (:447-459) in one pass: the three scales and the three f_dc against their sorted
// codebooks (held in shared memory), alpha of scales 255, alpha of sh0 = clip(sigmoid(opacity) * 255); padding 0
__global__ void __launch_bounds__(256) k_sog_scales_sh0(const float* __restrict__ rows, int64_t n, int F,
                                                        const int32_t* __restrict__ order, const SogCols cols,
                                                        const float* __restrict__ scb, int ms,
                                                        const float* __restrict__ ccb, int mc, int64_t pixels,
                                                        uchar4* __restrict__ scales, uchar4* __restrict__ sh0) {
    __shared__ float s_scb[kSogMaxCodebook], s_ccb[kSogMaxCodebook];
    for (int t = threadIdx.x; t < ms; t += blockDim.x) s_scb[t] = scb[t];
    for (int t = threadIdx.x; t < mc; t += blockDim.x) s_ccb[t] = ccb[t];
    __syncthreads();
    for (int64_t p = grid_start(); p < pixels; p += grid_stride()) {
        if (p >= n) {
            scales[p] = sh0[p] = make_uchar4(0, 0, 0, 0);
            continue;
        }
        const float* r = rows + (size_t)order[p] * F;
        scales[p] = make_uchar4(codebook_index(s_scb, ms, __ldg(r + cols.c[0])),
                                codebook_index(s_scb, ms, __ldg(r + cols.c[1])),
                                codebook_index(s_scb, ms, __ldg(r + cols.c[2])), 255);
        const float a = __fdiv_rn(1.f, __fadd_rn(1.f, numpy_expf(-__ldg(r + cols.c[6]))));
        sh0[p] = make_uchar4(codebook_index(s_ccb, mc, __ldg(r + cols.c[3])),
                             codebook_index(s_ccb, mc, __ldg(r + cols.c[4])),
                             codebook_index(s_ccb, mc, __ldg(r + cols.c[5])),
                             (uint8_t)fminf(fmaxf(__fmul_rn(a, 255.f), 0.f), 255.f));
    }
}

// out[j, k] = f_rest column k of the j-th splat (sog.py:503), one warp per row (lane k and k + 32), plus the
// "column k holds a value != 0" mask of the band detection (:483-487); -0.0 counts as zero, as `!= 0` does
__global__ void __launch_bounds__(256) k_sog_sh_gather(const float* __restrict__ rows, int64_t n, int F,
                                                       const int32_t* __restrict__ order,
                                                       const __grid_constant__ SogCols cols, float* __restrict__ out,
                                                       unsigned long long* __restrict__ nonzero) {
    const int lane = threadIdx.x & 31;
    const int w = cols.n;
    const int c_a = lane < w ? cols.c[lane] : 0, c_b = lane + 32 < w ? cols.c[lane + 32] : 0;
    const int64_t nwarps = grid_stride() >> 5;
    unsigned long long nz = 0ull;
    for (int64_t j = grid_start() >> 5; j < n; j += nwarps) {
        const float* r = rows + (size_t)order[j] * F;
        float* dst = out + (size_t)j * w;
        if (lane < w) {
            const float v = __ldg(r + c_a);
            if (v != 0.f) nz |= 1ull << lane;
            dst[lane] = v;
        }
        if (lane + 32 < w) {
            const float v = __ldg(r + c_b);
            if (v != 0.f) nz |= 1ull << (lane + 32);
            dst[lane + 32] = v;
        }
    }
    warp_or_column_mask(nz, nonzero);
}

// shN_labels (sog.py:594-600): (label + chunk offset) as u16 -> (lo, hi, 0, 255); padding 0
__global__ void __launch_bounds__(256) k_sog_labels(const int32_t* __restrict__ labels, int64_t n,
                                                    const __grid_constant__ SogChunks ch, int64_t pixels,
                                                    uchar4* __restrict__ out) {
    for (int64_t p = grid_start(); p < pixels; p += grid_stride()) {
        if (p >= n) {
            out[p] = make_uchar4(0, 0, 0, 0);
            continue;
        }
        const int64_t c = p / ch.chunk_size;
        const int64_t local = ch.passthrough[c] ? p - c * ch.chunk_size : (int64_t)labels[p];
        const uint32_t v = (uint32_t)(local + ch.offset[c]) & 0xffffu;
        out[p] = make_uchar4(v & 255, v >> 8, 0, 255);
    }
}

// shN_centroids (sog.py:566-588): the palette [P, coeffs] against the sorted codebook, laid out (P, C, 3) with
// C = coeffs / 3 (pixel p * C + j holds the three colour channels of coefficient j), alpha 255; padding 255
__global__ void __launch_bounds__(256) k_sog_centroids(const float* __restrict__ pal, int64_t P, int coeffs,
                                                       const float* __restrict__ cb, int m, int64_t pixels,
                                                       uchar4* __restrict__ out) {
    __shared__ float s_cb[kSogMaxCodebook];
    for (int t = threadIdx.x; t < m; t += blockDim.x) s_cb[t] = cb[t];
    __syncthreads();
    const int C = coeffs / 3;
    const int64_t valid = P * C;
    for (int64_t q = grid_start(); q < pixels; q += grid_stride()) {
        if (q >= valid) {
            out[q] = make_uchar4(255, 255, 255, 255);
            continue;
        }
        const int64_t p = q / C;
        const float* v = pal + p * coeffs + (q - p * C);
        out[q] = make_uchar4(codebook_index(s_cb, m, v[0]), codebook_index(s_cb, m, v[C]),
                             codebook_index(s_cb, m, v[2 * C]), 255);
    }
}

int grid_for(int64_t items) {
    const int64_t want = (items + 255) / 256;
    const int64_t cap = 8 * (int64_t)sm_count();
    return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

int load_cols(SogCols* cols, const int32_t* host, int ncols, int F, const char* what) {
    GSX_REQUIRE(host != nullptr && ncols >= 1 && ncols <= kSogMaxCols, GSX_ERR_ARG, "%s: %d columns (need 1..%d)",
                what, ncols, kSogMaxCols);
    for (int a = 0; a < ncols; ++a) {
        GSX_REQUIRE(host[a] >= 0 && host[a] < F, GSX_ERR_ARG, "%s: column %d out of range [0,%d)", what, host[a], F);
        cols->c[a] = host[a];
    }
    cols->n = ncols;
    return GSX_OK;
}

#define SOG_REQUIRE_N(what)                                                                                     \
    GSX_REQUIRE(n >= 0 && n < 2147483648ll, GSX_ERR_ARG, what ": n=%lld out of range [0, 2^31)", (long long)n); \
    GSX_REQUIRE(F >= 1, GSX_ERR_ARG, what ": bad row width %d", F)

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_lexsort_workspace_bytes(int64_t n) {
    if (n < 1) n = 1;
    return (int64_t)(2 * align_up((size_t)n * 8, 256) + 2 * align_up((size_t)n * 4, 256) + radix_ws_bytes(n) + 1024);
}

int gsx_lexsort_zyx(const float* xyz, int64_t n, int32_t* order_out, void* ws, int64_t ws_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(n < 2147483584ll, GSX_ERR_ARG, "lexsort: n out of range");
    GSX_REQUIRE(ws_bytes >= gsx_lexsort_workspace_bytes(n), GSX_ERR_WORKSPACE, "lexsort: workspace too small");
    Carver c(ws, (size_t)ws_bytes);
    uint64_t* k0 = c.take<uint64_t>((size_t)n);
    uint64_t* k1 = c.take<uint64_t>((size_t)n);
    int32_t* v0 = c.take<int32_t>((size_t)n);
    int32_t* v1 = c.take<int32_t>((size_t)n);
    char* rws = c.take<char>(radix_ws_bytes(n));
    int blocks = (int)((n + 255) / 256);
    k_lex_keys_z<<<blocks, 256, 0, st>>>(xyz, n, k0, v0);
    GSX_KERNEL_CHECK();
    uint64_t* ks = nullptr;
    int32_t* vs = nullptr;
    int rc = radix_sort_pairs(k0, k1, v0, v1, n, 0, 32, rws, radix_ws_bytes(n), &ks, &vs, st);
    if (rc) return rc;
    // second (more significant) key pair, gathered in the current order; reuse the buffer vs does not occupy
    uint64_t* kin = (ks == k0) ? k0 : k1;  // keys are dead: overwrite the buffer that pairs with vs
    uint64_t* kalt = (ks == k0) ? k1 : k0;
    int32_t* valt = (vs == v0) ? v1 : v0;
    k_lex_keys_xy<<<blocks, 256, 0, st>>>(xyz, vs, n, kin);
    GSX_KERNEL_CHECK();
    uint64_t* ks2 = nullptr;
    int32_t* vs2 = nullptr;
    rc = radix_sort_pairs(kin, kalt, vs, valt, n, 0, 64, rws, radix_ws_bytes(n), &ks2, &vs2, st);
    if (rc) return rc;
    GSX_CUDA_CHECK(cudaMemcpyAsync(order_out, vs2, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    return GSX_OK;
}

int gsx_quantize_to_codebook(const float* vals, int64_t n, const float* codebook_host, int32_t m, uint8_t* labels,
                             void* ws, int64_t ws_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(m >= 1 && m <= kMaxCodebook, GSX_ERR_UNSUPPORTED, "quantize: codebook size must be in [1,%d]",
                kMaxCodebook);
    GSX_REQUIRE(ws_bytes >= (int64_t)m * 4, GSX_ERR_WORKSPACE, "quantize: workspace too small");
    if (m == 1) {  // sog.py:410
        GSX_CUDA_CHECK(cudaMemsetAsync(labels, 0, (size_t)n, st));
        return GSX_OK;
    }
    GSX_CUDA_CHECK(cudaMemcpyAsync(ws, codebook_host, (size_t)m * 4, cudaMemcpyHostToDevice, st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));  // codebook_host may be a temporary
    int blocks = sm_count() * 8;
    int64_t need = (n + 255) / 256;
    if ((int64_t)blocks > need) blocks = (int)need;
    k_quantize_codebook<<<blocks, 256, 0, st>>>(vals, n, (const float*)ws, m, labels);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_means_minmax(const float* rows, int64_t n, int32_t F, const int32_t* cols3_host, float* ws,
                         int64_t ws_bytes, float* minmax, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_means_minmax");
    SOG_REQUIRE_N("sog_means_minmax");
    GSX_REQUIRE(n >= 1, GSX_ERR_ARG, "sog_means_minmax: the min and max of no splats are undefined");
    GSX_REQUIRE(ws_bytes >= (int64_t)kMinmaxBlocks * 6 * 4, GSX_ERR_WORKSPACE, "sog_means_minmax: workspace too small");
    SogCols c{};
    int rc = load_cols(&c, cols3_host, 3, F, "sog_means_minmax");
    if (rc) return rc;
    GSX_REQUIRE(rows && ws && minmax, GSX_ERR_ARG, "sog_means_minmax: null device pointer");
    int blocks = grid_for(n);
    if (blocks > kMinmaxBlocks) blocks = kMinmaxBlocks;
    k_sog_log_minmax<<<blocks, 256, 0, st>>>(rows, n, F, c.c[0], c.c[1], c.c[2], ws);
    GSX_KERNEL_CHECK();
    k_sog_minmax_final<<<1, 32, 0, st>>>(ws, blocks, minmax);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_means(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols3_host,
                  const float* minmax, int64_t pixels, uint8_t* means_l, uint8_t* means_u, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_means");
    SOG_REQUIRE_N("sog_means");
    GSX_REQUIRE(pixels >= n, GSX_ERR_ARG, "sog_means: %lld pixels < n", (long long)pixels);
    if (pixels == 0) return GSX_OK;
    SogCols c{};
    int rc = load_cols(&c, cols3_host, 3, F, "sog_means");
    if (rc) return rc;
    GSX_REQUIRE(((uintptr_t)means_l & 3) == 0 && ((uintptr_t)means_u & 3) == 0 && means_l && means_u &&
                    (n == 0 || (rows && order && minmax)),
                GSX_ERR_ARG, "sog_means: null or unaligned device pointer");
    k_sog_means<<<grid_for(pixels), 256, 0, st>>>(rows, n, F, order, c.c[0], c.c[1], c.c[2], minmax, pixels,
                                                  reinterpret_cast<uchar4*>(means_l), reinterpret_cast<uchar4*>(means_u));
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_quats(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols4_host,
                  int64_t pixels, uint8_t* quats, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_quats");
    SOG_REQUIRE_N("sog_quats");
    GSX_REQUIRE(pixels >= n, GSX_ERR_ARG, "sog_quats: %lld pixels < n", (long long)pixels);
    if (pixels == 0) return GSX_OK;
    SogCols c{};
    int rc = load_cols(&c, cols4_host, 4, F, "sog_quats");
    if (rc) return rc;
    GSX_REQUIRE(quats && ((uintptr_t)quats & 3) == 0 && (n == 0 || (rows && order)), GSX_ERR_ARG,
                "sog_quats: null or unaligned device pointer");
    k_sog_quats<<<grid_for(pixels), 256, 0, st>>>(rows, n, F, order, c.c[0], c.c[1], c.c[2], c.c[3], pixels,
                                                  reinterpret_cast<uchar4*>(quats));
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_gather_values(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols_host,
                          int32_t ncols, const int64_t* sel, int64_t m, float* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_gather_values");
    SOG_REQUIRE_N("sog_gather_values");
    GSX_REQUIRE(m >= 0 && (sel != nullptr || m <= n * ncols), GSX_ERR_ARG, "sog_gather_values: m=%lld out of range",
                (long long)m);
    if (m == 0) return GSX_OK;
    SogCols c{};
    int rc = load_cols(&c, cols_host, ncols, F, "sog_gather_values");
    if (rc) return rc;
    GSX_REQUIRE(n >= 1 && rows && order && out, GSX_ERR_ARG, "sog_gather_values: null device pointer or n = 0");
    k_sog_gather_values<<<grid_for(m), 256, 0, st>>>(rows, n, F, order, c, sel, m, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_scales_sh0(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols7_host,
                       const float* scale_cb, int32_t m_scale, const float* color_cb, int32_t m_color, int64_t pixels,
                       uint8_t* scales, uint8_t* sh0, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_scales_sh0");
    SOG_REQUIRE_N("sog_scales_sh0");
    GSX_REQUIRE(pixels >= n, GSX_ERR_ARG, "sog_scales_sh0: %lld pixels < n", (long long)pixels);
    GSX_REQUIRE(m_scale >= 1 && m_scale <= kSogMaxCodebook && m_color >= 1 && m_color <= kSogMaxCodebook,
                GSX_ERR_ARG, "sog_scales_sh0: codebook sizes %d, %d (need 1..%d)", m_scale, m_color, kSogMaxCodebook);
    if (pixels == 0) return GSX_OK;
    SogCols c{};
    int rc = load_cols(&c, cols7_host, 7, F, "sog_scales_sh0");
    if (rc) return rc;
    GSX_REQUIRE(scales && sh0 && ((uintptr_t)scales & 3) == 0 && ((uintptr_t)sh0 & 3) == 0 && scale_cb && color_cb &&
                    (n == 0 || (rows && order)),
                GSX_ERR_ARG, "sog_scales_sh0: null or unaligned device pointer");
    k_sog_scales_sh0<<<grid_for(pixels), 256, 0, st>>>(rows, n, F, order, c, scale_cb, m_scale, color_cb, m_color,
                                                       pixels, reinterpret_cast<uchar4*>(scales),
                                                       reinterpret_cast<uchar4*>(sh0));
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_sh_gather(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols_host,
                      int32_t ncols, float* out, unsigned long long* nonzero, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_sh_gather");
    SOG_REQUIRE_N("sog_sh_gather");
    SogCols c{};
    int rc = load_cols(&c, cols_host, ncols, F, "sog_sh_gather");
    if (rc) return rc;
    GSX_REQUIRE(nonzero && (n == 0 || (rows && order && out)), GSX_ERR_ARG, "sog_sh_gather: null device pointer");
    GSX_CUDA_CHECK(cudaMemsetAsync(nonzero, 0, sizeof(unsigned long long), st));
    if (n == 0) return GSX_OK;
    const int64_t want = (n + 7) / 8;  // 8 rows (warps) per CTA
    const int64_t cap = 16 * (int64_t)sm_count();
    k_sog_sh_gather<<<(int)(want < cap ? want : cap), 256, 0, st>>>(rows, n, F, order, c, out, nonzero);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_labels(const int32_t* labels, int64_t n, int64_t chunk_size, int32_t nchunks, const int32_t* offsets_host,
                   const int32_t* passthrough_host, int64_t pixels, uint8_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_labels");
    GSX_REQUIRE(n >= 0 && n < 2147483648ll && pixels >= n, GSX_ERR_ARG, "sog_labels: n=%lld pixels=%lld",
                (long long)n, (long long)pixels);
    if (pixels == 0) return GSX_OK;
    GSX_REQUIRE(out && ((uintptr_t)out & 3) == 0, GSX_ERR_ARG, "sog_labels: null or unaligned output");
    SogChunks ch{};
    if (n > 0) {
        GSX_REQUIRE(nchunks >= 1 && nchunks <= kSogMaxChunks && chunk_size >= 1 &&
                        chunk_size * nchunks >= n && chunk_size * (nchunks - 1) < n && offsets_host &&
                        passthrough_host,
                    GSX_ERR_ARG, "sog_labels: bad chunk schedule (%d chunks of %lld rows for n=%lld)", nchunks,
                    (long long)chunk_size, (long long)n);
        for (int c = 0; c < nchunks; ++c) {
            ch.offset[c] = offsets_host[c];
            ch.passthrough[c] = passthrough_host[c] != 0;
            GSX_REQUIRE(ch.passthrough[c] || labels, GSX_ERR_ARG, "sog_labels: chunk %d needs labels", c);
        }
    }
    ch.chunk_size = chunk_size > 0 ? chunk_size : 1;
    ch.n = nchunks;
    k_sog_labels<<<grid_for(pixels), 256, 0, st>>>(labels, n, ch, pixels, reinterpret_cast<uchar4*>(out));
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_centroids(const float* palette, int64_t P, int32_t coeffs, const float* cb, int32_t m, int64_t pixels,
                      uint8_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::sog_centroids");
    GSX_REQUIRE(P >= 0 && coeffs >= 3 && coeffs <= kSogMaxCols && coeffs % 3 == 0, GSX_ERR_ARG,
                "sog_centroids: P=%lld coeffs=%d", (long long)P, coeffs);
    GSX_REQUIRE(pixels >= P * (coeffs / 3), GSX_ERR_ARG, "sog_centroids: %lld pixels < P * coeffs / 3",
                (long long)pixels);
    GSX_REQUIRE(m >= 1 && m <= kSogMaxCodebook, GSX_ERR_ARG, "sog_centroids: codebook size %d (need 1..%d)", m,
                kSogMaxCodebook);
    if (pixels == 0) return GSX_OK;
    GSX_REQUIRE(out && ((uintptr_t)out & 3) == 0 && cb && (P == 0 || palette), GSX_ERR_ARG,
                "sog_centroids: null or unaligned device pointer");
    k_sog_centroids<<<grid_for(pixels), 256, 0, st>>>(palette, P, coeffs, cb, m, pixels, reinterpret_cast<uchar4*>(out));
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

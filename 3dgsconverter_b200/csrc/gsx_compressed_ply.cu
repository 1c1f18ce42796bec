// gsx_compressed_ply.cu -- the per-splat packing of the PlayCanvas compressed PLY writer for sm_90a (H100).
//
//   k_cply_pack      formats/compressed_ply.py:174-246 (CompressedPlyFormat.write after the Morton sort): one 256-thread
//                    CTA per 256-splat chunk, one splat per thread, rows gathered through the Morton order.  Writes the
//                    chunk row (18 float32: position bounds, clipped scale bounds, colour bounds), the four packed
//                    words of every splat (11-10-11 position, 2+3x10 quaternion, 11-10-11 scale, 8888 colour), one
//                    quantised byte per present f_rest_i column (staged in shared memory, stored as 16-byte words) and
//                    a 64-bit "packed SH column k has a non-zero value" mask (:141-161, one atomicOr per warp).
//                    The chunk bounds themselves come from gsx_chunk_minmax (gsx_morton.cu).
//   k_cply_narrow_sh out[j, :keep] = sh[j, :keep]: the SH block cut down to the columns of the detected degree (:163-169).
//
// Arithmetic follows NumPy-2 float32 semantics (Python float constants are weak scalars, i.e. rounded to float32 first):
// every step is one __f*_rn operation in the reference's order, with no contraction, and the alpha channel's exp is
// NumPy's SIMD float32 exp (gsx_numpy_scalar.cuh): every byte is bit-exact.
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_numpy_scalar.cuh"
#include "gsx_sh_mask.cuh"

namespace gsx {

namespace {

constexpr int kChunk = 256;   // CompressedPlyFormat.CHUNK_SIZE
constexpr int kMaxRest = 45;  // f_rest_0 .. f_rest_44 (SH degree 3)

// the Python float constants of the reference, rounded to float32 the way NumPy 2 rounds a weak scalar
constexpr float kShC0 = (float)0.28209479177387814;
constexpr float kSqrt2_2 = (float)0.7071067811865476;
constexpr float kMinExtent = (float)1e-5;
constexpr float kQuatEps = (float)1e-10;

// column positions inside a record row, passed by value (indexed with compile-time constants only)
struct CplyCols {
    int32_t c[14];  // x y z f_dc_0 f_dc_1 f_dc_2 opacity scale_0 scale_1 scale_2 rot_0 rot_1 rot_2 rot_3
    int32_t rest[kMaxRest];
    int32_t n_rest;
};

// np.clip(np.floor(x), 0, t).astype(np.uint32); NumPy keeps the NaN through the clip and its x86 cast loop converts
// it to 0x80000000 (cvttps2dq), which the reference ORs into the packed word (DESIGN §4.5)
__device__ __forceinline__ uint32_t floor_clip(float x, float t) {
    return x != x ? 0x80000000u : (uint32_t)fminf(fmaxf(floorf(x), 0.f), t);
}

// np.clip(s, -20, 20), which keeps NaN
__device__ __forceinline__ float clip20(float s) { return s != s ? s : fminf(fmaxf(s, -20.f), 20.f); }

// normalize() of _normalize_and_pack_11_10_11 / _8888 (:300-304, :311-314)
__device__ __forceinline__ uint32_t unorm(float v, float mn, float mx, float t) {
    const float ext = __fsub_rn(mx, mn);
    if (ext < kMinExtent) return 0u;
    const float nv = __fdiv_rn(__fsub_rn(v, mn), ext);
    return floor_clip(__fadd_rn(__fmul_rn(nv, t), 0.5f), t);
}

// f_dc * SH_C0 + 0.5 (:196-198); monotone in f_dc, so it maps the f_dc bounds onto the colour bounds.  A NaN comes
// out as x86 float arithmetic returns it (the operand, quieted), so a NaN colour bound keeps the f_dc NaN's bits.
__device__ __forceinline__ float dc_color(float f) {
    return f != f ? __uint_as_float(__float_as_uint(f) | 0x00400000u) : __fadd_rn(__fmul_rn(f, kShC0), 0.5f);
}

// pack_unorm(q * sign, 10) of _pack_quaternions (:331-333)
__device__ __forceinline__ uint32_t quat_comp(float q, float s) {
    const float v = __fadd_rn(__fmul_rn(__fmul_rn(q, s), kSqrt2_2), 0.5f);
    return floor_clip(__fadd_rn(__fmul_rn(v, 1023.f), 0.5f), 1023.f);
}

// _pack_quaternions (:321-340): serial sum of squares (np.linalg.norm over 4 components), q /= norm + 1e-10, largest =
// first index of max |q| (np.argmax: the first NaN is the maximum), q *= sign(q[largest]) (sign(0) = 0, sign(NaN) =
// NaN), the other three in ascending order below 2 bits of index
__device__ __forceinline__ uint32_t pack_quat(float q0, float q1, float q2, float q3) {
    float ss = __fmul_rn(q0, q0);
    ss = __fadd_rn(ss, __fmul_rn(q1, q1));
    ss = __fadd_rn(ss, __fmul_rn(q2, q2));
    ss = __fadd_rn(ss, __fmul_rn(q3, q3));
    const float d = __fadd_rn(__fsqrt_rn(ss), kQuatEps);
    q0 = __fdiv_rn(q0, d), q1 = __fdiv_rn(q1, d), q2 = __fdiv_rn(q2, d), q3 = __fdiv_rn(q3, d);
    uint32_t L = 0;
    float best = fabsf(q0), qL = q0;
    if (best == best && (fabsf(q1) > best || q1 != q1)) best = fabsf(q1), qL = q1, L = 1;
    if (best == best && (fabsf(q2) > best || q2 != q2)) best = fabsf(q2), qL = q2, L = 2;
    if (best == best && (fabsf(q3) > best || q3 != q3)) best = fabsf(q3), qL = q3, L = 3;
    const float s = qL > 0.f ? 1.f : (qL < 0.f ? -1.f : (qL == 0.f ? 0.f : qL));
    uint32_t r = L;
    if (L != 0) r = (r << 10) | quat_comp(q0, s);
    if (L != 1) r = (r << 10) | quat_comp(q1, s);
    if (L != 2) r = (r << 10) | quat_comp(q2, s);
    if (L != 3) r = (r << 10) | quat_comp(q3, s);
    return r;
}

// uint8(clip((v / 8 + 0.5) * 256, 0, 255)) (:245-246)
__device__ __forceinline__ uint8_t sh_byte(float v) {
    const float s = __fmul_rn(__fadd_rn(__fdiv_rn(v, 8.f), 0.5f), 256.f);
    return (uint8_t)fminf(fmaxf(s, 0.f), 255.f);
}

__global__ void __launch_bounds__(kChunk) k_cply_pack(const float* __restrict__ rows, int64_t n, int F,
                                                      const int32_t* __restrict__ order, const CplyCols cols,
                                                      const float* __restrict__ lo6, const float* __restrict__ hi6,
                                                      const float* __restrict__ lo3, const float* __restrict__ hi3,
                                                      float* __restrict__ chunk_out, uint4* __restrict__ vertex_out,
                                                      uint8_t* __restrict__ sh_out,
                                                      unsigned long long* __restrict__ nonzero) {
    __shared__ float sb[18];
    __shared__ __align__(16) uint8_t ssh[kChunk * kMaxRest];
    const int64_t c = blockIdx.x;
    const int t = threadIdx.x;
    const int64_t c0 = c * kChunk;
    const int rows_here = (int)(n - c0 < kChunk ? n - c0 : kChunk);
    const int n_rest = cols.n_rest;

    // chunk row in the reference's field order: min_x..z, max_x..z, min/max_scale_x..z, min_r..b, max_r..b
    if (t < 18) {
        float v;
        if (t < 3) v = lo6[c * 6 + t];
        else if (t < 6) v = hi6[c * 6 + t - 3];
        else if (t < 9) v = lo3[c * 3 + t - 6];
        else if (t < 12) v = hi3[c * 3 + t - 9];
        else if (t < 15) v = dc_color(lo6[c * 6 + 3 + t - 12]);
        else v = dc_color(hi6[c * 6 + 3 + t - 15]);
        sb[t] = v;
        chunk_out[c * 18 + t] = v;
    }
    __syncthreads();

    unsigned long long nz = 0ull;
    if (t < rows_here) {
        const float* r = rows + (size_t)order[c0 + t] * F;
        const uint32_t pos = unorm(__ldg(r + cols.c[0]), sb[0], sb[3], 2047.f) << 21 |
                             unorm(__ldg(r + cols.c[1]), sb[1], sb[4], 1023.f) << 11 |
                             unorm(__ldg(r + cols.c[2]), sb[2], sb[5], 2047.f);
        const float s0 = clip20(__ldg(r + cols.c[7]));
        const float s1 = clip20(__ldg(r + cols.c[8]));
        const float s2 = clip20(__ldg(r + cols.c[9]));
        const uint32_t scl = unorm(s0, sb[6], sb[9], 2047.f) << 21 | unorm(s1, sb[7], sb[10], 1023.f) << 11 |
                             unorm(s2, sb[8], sb[11], 2047.f);
        const float a = __fdiv_rn(1.f, __fadd_rn(1.f, numpy_expf(-__ldg(r + cols.c[6]))));
        const uint32_t col = unorm(dc_color(__ldg(r + cols.c[3])), sb[12], sb[15], 255.f) << 24 |
                             unorm(dc_color(__ldg(r + cols.c[4])), sb[13], sb[16], 255.f) << 16 |
                             unorm(dc_color(__ldg(r + cols.c[5])), sb[14], sb[17], 255.f) << 8 |
                             floor_clip(__fadd_rn(__fmul_rn(a, 255.f), 0.5f), 255.f);
        const uint32_t rot = pack_quat(__ldg(r + cols.c[10]), __ldg(r + cols.c[11]), __ldg(r + cols.c[12]),
                                       __ldg(r + cols.c[13]));
        vertex_out[c0 + t] = make_uint4(pos, rot, scl, col);
        uint8_t* mine = ssh + t * n_rest;
#pragma unroll
        for (int k = 0; k < kMaxRest; ++k)
            if (k < n_rest) {
                const float v = __ldg(r + cols.rest[k]);
                if (v != 0.f) nz |= 1ull << k;   // -0.0 counts as zero, as `!= 0` does in NumPy
                mine[k] = sh_byte(v);
            }
    }
    warp_or_column_mask(nz, nonzero);
    if (n_rest == 0) return;
    __syncthreads();
    // the chunk's SH bytes are one contiguous run of rows_here * n_rest bytes; chunk starts are 256 * n_rest apart, so
    // every run starts 16-byte aligned
    const int bytes = rows_here * n_rest;
    uint8_t* dst = sh_out + c0 * n_rest;
    const int nvec = bytes >> 4;
    for (int i = t; i < nvec; i += kChunk) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(ssh)[i];
    for (int i = (nvec << 4) + t; i < bytes; i += kChunk) dst[i] = ssh[i];
}

__global__ void __launch_bounds__(256) k_cply_narrow_sh(const uint8_t* __restrict__ sh, int64_t n, int width, int keep,
                                                        uint8_t* __restrict__ out) {
    const int64_t total = n * keep;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = e / keep;
        out[e] = sh[j * width + (e - j * keep)];
    }
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_cply_pack(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols14_host,
                  const int32_t* rest_cols_host, int32_t n_rest, const float* lo_pos_dc, const float* hi_pos_dc,
                  const float* lo_scale, const float* hi_scale, float* chunk_out, uint32_t* vertex_out, uint8_t* sh_out,
                  uint64_t* rest_nonzero_out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::cply_pack");
    GSX_REQUIRE(n >= 0 && n < 2147483648ll, GSX_ERR_ARG, "cply_pack: n=%lld out of range [0, 2^31)", (long long)n);
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(F >= 1, GSX_ERR_ARG, "cply_pack: bad row width %d", F);
    GSX_REQUIRE(cols14_host != nullptr, GSX_ERR_ARG, "cply_pack: no column table");
    GSX_REQUIRE(n_rest >= 0 && n_rest <= kMaxRest && (n_rest == 0 || rest_cols_host != nullptr), GSX_ERR_ARG,
                "cply_pack: n_rest=%d out of range [0, %d]", n_rest, kMaxRest);
    GSX_REQUIRE(rows && order && lo_pos_dc && hi_pos_dc && lo_scale && hi_scale && chunk_out && vertex_out &&
                    rest_nonzero_out && (n_rest == 0 || sh_out),
                GSX_ERR_ARG, "cply_pack: null device pointer");
    GSX_REQUIRE(((uintptr_t)vertex_out & 15) == 0 && ((uintptr_t)sh_out & 15) == 0, GSX_ERR_ARG,
                "cply_pack: vertex_out and sh_out must be 16-byte aligned");
    CplyCols cols{};
    for (int a = 0; a < 14; ++a) {
        GSX_REQUIRE(cols14_host[a] >= 0 && cols14_host[a] < F, GSX_ERR_ARG, "cply_pack: column %d out of range [0,%d)",
                    cols14_host[a], F);
        cols.c[a] = cols14_host[a];
    }
    for (int k = 0; k < n_rest; ++k) {
        GSX_REQUIRE(rest_cols_host[k] >= 0 && rest_cols_host[k] < F, GSX_ERR_ARG,
                    "cply_pack: f_rest column %d out of range [0,%d)", rest_cols_host[k], F);
        cols.rest[k] = rest_cols_host[k];
    }
    cols.n_rest = n_rest;
    GSX_CUDA_CHECK(cudaMemsetAsync(rest_nonzero_out, 0, sizeof(unsigned long long), st));
    const int64_t nchunk = (n + kChunk - 1) / kChunk;
    k_cply_pack<<<(int)nchunk, kChunk, 0, st>>>(rows, n, F, order, cols, lo_pos_dc, hi_pos_dc, lo_scale, hi_scale,
                                                chunk_out, reinterpret_cast<uint4*>(vertex_out), sh_out,
                                                (unsigned long long*)rest_nonzero_out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_cply_narrow_sh(const uint8_t* sh, int64_t n, int32_t width, int32_t keep, uint8_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 0 && n < 2147483648ll, GSX_ERR_ARG, "cply_narrow_sh: n=%lld out of range [0, 2^31)", (long long)n);
    GSX_REQUIRE(keep >= 0 && keep <= width && width <= kMaxRest, GSX_ERR_ARG,
                "cply_narrow_sh: keep=%d width=%d (need 0 <= keep <= width <= %d)", keep, width, kMaxRest);
    if (n == 0 || keep == 0) return GSX_OK;
    GSX_REQUIRE(sh && out, GSX_ERR_ARG, "cply_narrow_sh: null device pointer");
    const int64_t total = n * keep;
    const int64_t want = (total + 255) / 256;
    const int blocks = (int)(want < 32 * (int64_t)sm_count() ? want : 32 * (int64_t)sm_count());
    k_cply_narrow_sh<<<blocks, 256, 0, st>>>(sh, n, width, keep, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

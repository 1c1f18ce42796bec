// gsx_splat_codecs.cu -- the .ksplat, .spz and .splat writers' per-splat packing for sm_90a (H100).
//
//   k_codec_sh_mask     "f_rest column k holds a value != 0" bits (NaN counts, as np.any(x != 0) / np.all(x == 0) do):
//                       the input of the ksplat (ksplat.py:340-368) and SPZ (spz.py:53-77) degree rules, which the
//                       caller applies on the host because the degree sets the record layout.
//   k_ksplat_centres    (min + max) / 2.0 of the bucket bounds (ksplat.py:439-445; bounds from gsx_chunk_minmax).
//   k_ksplat_pack       ksplat.py:419-536: one interleaved record per splat, levels 0 (float32), 1 (float16) and >= 2
//                       (float16, uint8 SH); positions quantised against the bucket centre at levels >= 1.
//   k_spz_pack          spz.py:106-173 (_pack_v3): the planar SPZ body -- 24-bit positions, alpha, colour, scales,
//                       smallest-three rotations (:298-343) and the interleaved, bucketed SH bytes.
//   k_splat_sort_keys   splat.py:92-98: an order-preserving uint32 key of -exp(s0+s1+s2) * sigmoid(opacity) (-0.0 folded
//                       onto +0.0, every NaN above +inf) and the row index, for the stable radix sort (gsx_sort_pairs).
//   k_splat_pack        splat.py:100-164: the 32-byte records, rows taken in the sorted order.
//   k_records_from_bytes the float32 fields of a structured array with other fields (the converter's trailing
//                       red/green/blue u1) as the packed float32 rows the writers read.
//
// Every pack kernel runs 128 threads (4 warps) per CTA and one splat per thread.  Each warp first loads the columns it
// needs of its 32 rows into shared memory, lanes striding over one row at a time (whole sectors, as k_gather_rows), then
// packs its splat into a shared staging buffer, which the CTA stores as 16-byte words whatever the byte alignment of
// the destination (records of 33 or 65 bytes, planar sections at any offset).  Arithmetic follows NumPy-2 float32
// semantics on x86-64 (gsx_numpy_scalar.cuh): Python float constants are weak scalars, one __f*_rn operation per NumPy
// operation in the reference's order.
#include "../../include/gsx.h"

#include "gsx_bits.cuh"
#include "gsx_common.cuh"
#include "gsx_numpy_scalar.cuh"
#include "gsx_sh_mask.cuh"
#include "gsx_staged.cuh"

namespace gsx {

namespace {

constexpr int kThreads = 128;   // rows per CTA
constexpr int kMaxSh = 45;      // f_rest_0 .. f_rest_44
constexpr int kMaxCols = 14 + kMaxSh;

// the Python float constants of the writers, rounded to float32 as NumPy 2 rounds a weak scalar
constexpr float kShC0 = (float)0.28209479177387814;
constexpr float kSpzColor = (float)0.15;
constexpr float kSpzRotScale = (float)(511.0 / 0.707106781186547524401);
constexpr float kSpzEps = (float)1e-9;

// tile column of each attribute: the 14 fixed columns, then the SH values
enum { X, Y, Z, DC0, DC1, DC2, OP, S0, S1, S2, R0, R1, R2, R3, SH };

struct CodecCols {
    int32_t c[kMaxCols];   // row column of tile column k
    int32_t ncol;
};

// Columns of this CTA's rows [base, base + rows_here) into tile[row * ncol + k]; warp w loads rows 32w .. 32w+31 with
// its lanes striding over the row's columns.  Only the warp's own rows are touched, so __syncwarp() is enough before a
// thread reads its row.
__device__ __forceinline__ void load_tile(const float* __restrict__ rows, int F, const int32_t* __restrict__ order,
                                          int64_t base, int rows_here, const int32_t* scols, int ncol, float* tile) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r0 = w * 32;
    const int nr = rows_here - r0 < 32 ? rows_here - r0 : 32;
    for (int e = lane; e < nr * ncol; e += 32) {
        const int i = e / ncol, k = e - i * ncol;
        const int64_t j = base + r0 + i;
        const int64_t src = order ? (int64_t)order[j] : j;
        tile[(r0 + i) * ncol + k] = __ldg(rows + (size_t)src * F + scols[k]);
    }
    __syncwarp();
}

__device__ __forceinline__ void load_cols(const CodecCols& cols, int32_t* scols) {
    for (int k = threadIdx.x; k < cols.ncol; k += blockDim.x) scols[k] = cols.c[k];
    __syncthreads();
}

// np.clip((0.5 + C0 * f) * 255, 0, 255).astype(np.uint8)  (splat.py:135-137, ksplat.py:479-481)
__device__ __forceinline__ uint8_t dc_u8(float f) {
    return np_u8(np_clip(__fmul_rn(__fadd_rn(0.5f, __fmul_rn(kShC0, f)), 255.f), 0.f, 255.f));
}

// np.clip((1 / (1 + np.exp(-op))) * 255, 0, 255).astype(np.uint8)  (splat.py:145, ksplat.py:482)
__device__ __forceinline__ uint8_t alpha_u8(float op) {
    const float a = __fdiv_rn(1.f, __fadd_rn(1.f, numpy_expf(-op)));
    return np_u8(np_clip(__fmul_rn(a, 255.f), 0.f, 255.f));
}

__device__ __forceinline__ void store_f32_or_f16(uint8_t*& p, float v, bool f16) {
    if (f16) put16(p, numpy_f2h(v)), p += 2;
    else put32(p, __float_as_uint(v)), p += 4;
}

__global__ void __launch_bounds__(256) k_codec_sh_mask(const float* __restrict__ rows, int64_t n, int F,
                                                       const CodecCols cols, unsigned long long* __restrict__ mask) {
    __shared__ int32_t scols[kMaxCols];
    load_cols(cols, scols);
    const int ncol = cols.ncol, lane = threadIdx.x & 31;
    const int64_t r0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x - lane);   // the warp's first row
    unsigned long long bits = 0ull;
    if (r0 < n) {
        const int nr = n - r0 < 32 ? (int)(n - r0) : 32;
        for (int e = lane; e < nr * ncol; e += 32) {
            const int i = e / ncol, k = e - i * ncol;
            const float v = __ldg(rows + (size_t)(r0 + i) * F + scols[k]);
            if (!(v == 0.f)) bits |= 1ull << k;   // NaN counts as non-zero, -0.0 as zero
        }
    }
    warp_or_column_mask(bits, mask);
}

__global__ void __launch_bounds__(256) k_ksplat_centres(const float* __restrict__ lo, const float* __restrict__ hi,
                                                        int64_t m, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    // x86 float arithmetic returns the first NaN operand, quieted, and 0xffc00000 for inf + -inf; the GPU returns
    // 0x7fffffff for both, and the centre's bytes go into the file
    const float l = lo[i], h = hi[i], s = __fadd_rn(l, h);
    out[i] = l != l   ? __uint_as_float(__float_as_uint(l) | 0x00400000u)
             : h != h ? __uint_as_float(__float_as_uint(h) | 0x00400000u)
             : s != s ? __uint_as_float(0xffc00000u)
                      : __fdiv_rn(s, 2.f);
}

// level: 0, 1, 2, or 3 for any stored level >= 3 (the reference casts the raw SH values to uint8 there, ksplat.py:533)
__global__ void __launch_bounds__(kThreads) k_ksplat_pack(const float* __restrict__ rows, int64_t n, int F,
                                                          const CodecCols cols, int level, int64_t bucket,
                                                          float sf_inv, const float* __restrict__ centres, int rec,
                                                          uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int32_t scols[kMaxCols];
    load_cols(cols, scols);
    const int ncol = cols.ncol, nsh = ncol - SH, t = threadIdx.x;
    const int64_t base = (int64_t)blockIdx.x * kThreads;
    const int rows_here = (int)(n - base < kThreads ? n - base : kThreads);
    float* tile = reinterpret_cast<float*>(smem);
    uint8_t* stage = smem + (size_t)kThreads * ncol * 4;
    load_tile(rows, F, nullptr, base, rows_here, scols, ncol, tile);
    if (t < rows_here) {
        const float* r = tile + t * ncol;
        uint8_t* p = stage + t * rec;
        const bool f16 = level >= 1;
        if (level == 0) {
            for (int a = X; a <= Z; ++a) put32(p, __float_as_uint(r[a])), p += 4;
        } else {
            const float* c = centres + ((base + t) / bucket) * 3;
            for (int a = X; a <= Z; ++a) {   // np.clip(np.round((x - c) * sf_inv) + 32767, 0, 65535).astype(np.uint16)
                const float q = __fadd_rn(rintf(__fmul_rn(__fsub_rn(r[a], c[a]), sf_inv)), 32767.f);
                put16(p, np_u16(np_clip(q, 0.f, 65535.f))), p += 2;
            }
        }
        for (int a = S0; a <= S2; ++a) store_f32_or_f16(p, numpy_expf(r[a]), f16);
        for (int a = R0; a <= R3; ++a) store_f32_or_f16(p, r[a], f16);
        p[0] = dc_u8(r[DC0]), p[1] = dc_u8(r[DC1]), p[2] = dc_u8(r[DC2]), p[3] = alpha_u8(r[OP]);
        p += 4;
        for (int k = 0; k < nsh; ++k) {
            const float v = r[SH + k];
            if (level <= 1) store_f32_or_f16(p, v, f16);
            else if (level == 2)   // np.clip((sh - -2.0) / 4.0 * 255, 0, 255).astype(np.uint8)
                *p++ = np_u8(np_clip(__fmul_rn(__fdiv_rn(__fsub_rn(v, -2.f), 4.f), 255.f), 0.f, 255.f));
            else
                *p++ = np_u8(v);
        }
    }
    __syncthreads();
    store_staged(out + base * rec, stage, rows_here * rec);
}

// smallest-three quaternion of _pack_rot_v3 (spz.py:298-343); w = rot_0, R = (x, y, z, w) / norm
__device__ __forceinline__ uint32_t spz_rot(float w, float x, float y, float z) {
    float ss = __fmul_rn(w, w);
    ss = __fadd_rn(ss, __fmul_rn(x, x));
    ss = __fadd_rn(ss, __fmul_rn(y, y));
    ss = __fadd_rn(ss, __fmul_rn(z, z));
    const float norm = __fsqrt_rn(__fadd_rn(ss, kSpzEps));
    const float R[4] = {__fdiv_rn(x, norm), __fdiv_rn(y, norm), __fdiv_rn(z, norm), __fdiv_rn(w, norm)};
    int m = 0;   // np.argmax(np.abs(R)): first maximum, the first NaN wins
    float best = fabsf(R[0]);
#pragma unroll
    for (int j = 1; j < 4; ++j)
        if (best == best && (fabsf(R[j]) > best || R[j] != R[j])) best = fabsf(R[j]), m = j;
    const bool neg = R[m] < 0.f;
    uint32_t packed = (uint32_t)m << 30;
    int slot = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j == m) continue;
        const float v = np_clip(__fadd_rn(__fmul_rn(fabsf(R[j]), kSpzRotScale), 0.5f), 0.f, 511.f);
        // NumPy's SIMD float -> uint32 loop gives 0x80000000 for NaN (DESIGN §4.5)
        const uint32_t mag = v != v ? 0x80000000u : (uint32_t)v;
        const uint32_t comp = (uint32_t)((R[j] < 0.f) != neg) << 9 | mag;
        packed |= comp << ((2 - slot) * 10);
        ++slot;
    }
    return packed;
}

// int32(rint(v * 128 + 128)), then np.clip((q + bs // 2) // bs * bs, 0, 255) with Python floor division (bs = 2^lb)
__device__ __forceinline__ uint8_t spz_sh(float v, int lb) {
    const int32_t q = np_i32(rintf(__fadd_rn(__fmul_rn(v, 128.f), 128.f)));
    const int32_t b = (q + (1 << (lb - 1))) & ~((1 << lb) - 1);
    return (uint8_t)(b < 0 ? 0 : (b > 255 ? 255 : b));
}

// body sections (offsets relative to out = the byte after the 16-byte header): pos 9N, alpha N, colour 3N, scale 3N,
// rot 4N, SH 3*sh_dim*N.  SH tile column 14 + 3i + c holds f_rest_{i + 15c}.
__global__ void __launch_bounds__(kThreads) k_spz_pack(const float* __restrict__ rows, int64_t n, int F,
                                                       const CodecCols cols, uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int32_t scols[kMaxCols];
    load_cols(cols, scols);
    const int ncol = cols.ncol, nsh = ncol - SH, t = threadIdx.x;
    const int64_t base = (int64_t)blockIdx.x * kThreads;
    const int rows_here = (int)(n - base < kThreads ? n - base : kThreads);
    float* tile = reinterpret_cast<float*>(smem);
    uint8_t* s_pos = smem + (size_t)kThreads * ncol * 4;
    uint8_t* s_alpha = s_pos + kThreads * 9;
    uint8_t* s_col = s_alpha + kThreads;
    uint8_t* s_scl = s_col + kThreads * 3;
    uint8_t* s_rot = s_scl + kThreads * 3;
    uint8_t* s_sh = s_rot + kThreads * 4;
    load_tile(rows, F, nullptr, base, rows_here, scols, ncol, tile);
    if (t < rows_here) {
        const float* r = tile + t * ncol;
        for (int a = X; a <= Z; ++a) {   // np.round(x * 4096).astype(np.int32), low three bytes
            const uint32_t c = (uint32_t)np_i32(rintf(__fmul_rn(r[a], 4096.f)));
            s_pos[t * 9 + 3 * a] = (uint8_t)c, s_pos[t * 9 + 3 * a + 1] = (uint8_t)(c >> 8);
            s_pos[t * 9 + 3 * a + 2] = (uint8_t)(c >> 16);
        }
        // (1.0 / (1.0 + np.exp(-np.clip(op, -20, 20))) * 255.0).astype(np.uint8)
        const float e = numpy_expf(-np_clip(r[OP], -20.f, 20.f));
        s_alpha[t] = np_u8(__fmul_rn(__fdiv_rn(1.f, __fadd_rn(1.f, e)), 255.f));
        for (int a = 0; a < 3; ++a) {
            // np.clip((f_dc * 0.15 + 0.5) * 255.0, 0, 255), np.clip((s + 10.0) * 16.0, 0, 255)
            s_col[t * 3 + a] = np_u8(np_clip(__fmul_rn(__fadd_rn(__fmul_rn(r[DC0 + a], kSpzColor), 0.5f), 255.f), 0.f, 255.f));
            s_scl[t * 3 + a] = np_u8(np_clip(__fmul_rn(__fadd_rn(r[S0 + a], 10.f), 16.f), 0.f, 255.f));
        }
        reinterpret_cast<uint32_t*>(s_rot)[t] = spz_rot(r[R0], r[R1], r[R2], r[R3]);
        for (int k = 0; k < nsh; ++k) s_sh[t * nsh + k] = spz_sh(r[SH + k], k < 9 ? 3 : 4);
    }
    __syncthreads();
    store_staged(out + base * 9, s_pos, rows_here * 9);
    store_staged(out + n * 9 + base, s_alpha, rows_here);
    store_staged(out + n * 10 + base * 3, s_col, rows_here * 3);
    store_staged(out + n * 13 + base * 3, s_scl, rows_here * 3);
    store_staged(out + n * 16 + base * 4, s_rot, rows_here * 4);
    if (nsh) store_staged(out + n * 20 + base * nsh, s_sh, rows_here * nsh);
}

// cols: scale_0 scale_1 scale_2 opacity
__global__ void __launch_bounds__(256) k_splat_sort_keys(const float* __restrict__ rows, int64_t n, int F, int c0,
                                                         int c1, int c2, int cop, uint64_t* __restrict__ keys,
                                                         int32_t* __restrict__ vals) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* r = rows + (size_t)i * F;
    const float ssum = __fadd_rn(__fadd_rn(__ldg(r + c0), __ldg(r + c1)), __ldg(r + c2));
    const float opt = __fdiv_rn(1.f, __fadd_rn(1.f, numpy_expf(-__ldg(r + cop))));
    const float v = -__fmul_rn(numpy_expf(ssum), opt);
    keys[i] = numpy_sort_key(v);
    vals[i] = (int32_t)i;
}

__global__ void __launch_bounds__(kThreads) k_splat_pack(const float* __restrict__ rows, int64_t n, int F,
                                                         const int32_t* __restrict__ order, const CodecCols cols,
                                                         uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int32_t scols[kMaxCols];
    load_cols(cols, scols);
    const int ncol = cols.ncol, t = threadIdx.x;
    const int64_t base = (int64_t)blockIdx.x * kThreads;
    const int rows_here = (int)(n - base < kThreads ? n - base : kThreads);
    float* tile = reinterpret_cast<float*>(smem);
    uint8_t* stage = smem + (size_t)kThreads * ncol * 4;
    load_tile(rows, F, order, base, rows_here, scols, ncol, tile);
    if (t < rows_here) {
        const float* r = tile + t * ncol;
        uint8_t* p = stage + t * 32;
        for (int a = X; a <= Z; ++a) put32(p + 4 * a, __float_as_uint(r[a]));
        for (int a = 0; a < 3; ++a) put32(p + 12 + 4 * a, __float_as_uint(numpy_expf(r[S0 + a])));
        p[24] = dc_u8(r[DC0]), p[25] = dc_u8(r[DC1]), p[26] = dc_u8(r[DC2]), p[27] = alpha_u8(r[OP]);
        // np.sqrt(r0**2 + r1**2 + r2**2 + r3**2); np.clip(r / norm * 128 + 128, 0, 255).astype(np.uint8)
        float ss = __fmul_rn(r[R0], r[R0]);
        ss = __fadd_rn(ss, __fmul_rn(r[R1], r[R1]));
        ss = __fadd_rn(ss, __fmul_rn(r[R2], r[R2]));
        ss = __fadd_rn(ss, __fmul_rn(r[R3], r[R3]));
        const float norm = __fsqrt_rn(ss);
        for (int a = 0; a < 4; ++a)
            p[28 + a] = np_u8(np_clip(__fadd_rn(__fmul_rn(__fdiv_rn(r[R0 + a], norm), 128.f), 128.f), 0.f, 255.f));
    }
    __syncthreads();
    store_staged(out + base * 32, stage, rows_here * 32);
}

struct ByteFields {
    int32_t off[256];
};

__global__ void __launch_bounds__(256) k_records_from_bytes(const uint8_t* __restrict__ src, int64_t n, int64_t row_bytes,
                                                            const ByteFields f, int nf, float* __restrict__ out) {
    const int64_t total = n * nf;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = e / nf;
        const uint8_t* p = src + j * row_bytes + f.off[e - j * nf];
        out[e] = __uint_as_float((uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24);
    }
}

int fill_cols(const int32_t* cols14, const int32_t* sh_cols, int nsh, int F, CodecCols& cols, const char* who) {
    GSX_REQUIRE(cols14 != nullptr && (nsh == 0 || sh_cols != nullptr), GSX_ERR_ARG, "%s: no column table", who);
    GSX_REQUIRE(nsh >= 0 && nsh <= kMaxSh, GSX_ERR_ARG, "%s: %d SH columns out of range [0, %d]", who, nsh, kMaxSh);
    for (int k = 0; k < 14 + nsh; ++k) {
        const int32_t c = k < 14 ? cols14[k] : sh_cols[k - 14];
        GSX_REQUIRE(c >= 0 && c < F, GSX_ERR_ARG, "%s: column %d out of range [0,%d)", who, c, F);
        cols.c[k] = c;
    }
    cols.ncol = 14 + nsh;
    return GSX_OK;
}

int check_n(int64_t n, int F, const char* who) {
    GSX_REQUIRE(n >= 0, GSX_ERR_ARG, "%s: n=%lld < 0", who, (long long)n);
    GSX_REQUIRE(n < 2147483648ll, GSX_ERR_UNSUPPORTED, "%s: n=%lld needs int32 row indices (n < 2^31)", who,
                (long long)n);
    GSX_REQUIRE(n == 0 || F >= 1, GSX_ERR_ARG, "%s: bad row width %d", who, F);
    return GSX_OK;
}

// at most 59 columns and a 140-byte record: every configuration stays below the 48 KB default
size_t tile_bytes(int ncol) { return (size_t)kThreads * ncol * 4; }

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_codec_sh_mask(const float* rows, int64_t n, int32_t F, const int32_t* sh_cols, int32_t nsh, uint64_t* mask,
                      void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_n(n, F, "codec_sh_mask");
    if (rc) return rc;
    GSX_REQUIRE(nsh >= 0 && nsh <= kMaxSh && (nsh == 0 || sh_cols), GSX_ERR_ARG, "codec_sh_mask: %d SH columns", nsh);
    GSX_REQUIRE(mask, GSX_ERR_ARG, "codec_sh_mask: null mask");
    CodecCols cols{};
    for (int k = 0; k < nsh; ++k) {
        GSX_REQUIRE(sh_cols[k] >= 0 && sh_cols[k] < F, GSX_ERR_ARG, "codec_sh_mask: column %d out of range [0,%d)",
                    sh_cols[k], F);
        cols.c[k] = sh_cols[k];
    }
    cols.ncol = nsh;
    GSX_CUDA_CHECK(cudaMemsetAsync(mask, 0, sizeof(unsigned long long), st));
    if (n == 0 || nsh == 0) return GSX_OK;
    GSX_REQUIRE(rows, GSX_ERR_ARG, "codec_sh_mask: null rows");
    k_codec_sh_mask<<<(int)((n + 255) / 256), 256, 0, st>>>(rows, n, F, cols, (unsigned long long*)mask);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int32_t gsx_ksplat_record_bytes(int32_t level, int32_t sh_count) {
    if (level < 0 || sh_count < 0) return -1;
    return level == 0 ? 44 + 4 * sh_count : 24 + (level == 1 ? 2 : 1) * sh_count;
}

int gsx_ksplat_centres(const float* lo, const float* hi, int64_t nbucket, float* centres, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(nbucket >= 0, GSX_ERR_ARG, "ksplat_centres: nbucket < 0");
    if (nbucket == 0) return GSX_OK;
    GSX_REQUIRE(lo && hi && centres, GSX_ERR_ARG, "ksplat_centres: null pointer");
    const int64_t m = nbucket * 3;
    k_ksplat_centres<<<(int)((m + 255) / 256), 256, 0, st>>>(lo, hi, m, centres);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_ksplat_pack(const float* rows, int64_t n, int32_t F, const int32_t* cols14, const int32_t* sh_cols,
                    int32_t sh_count, int32_t level, int64_t bucket_size, float sf_inv, const float* centres,
                    uint8_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_n(n, F, "ksplat_pack");
    if (rc) return rc;
    GSX_REQUIRE(level >= 0 && level <= 65535, GSX_ERR_ARG, "ksplat_pack: level %d", level);
    GSX_REQUIRE(sh_count == 0 || sh_count == 9 || sh_count == 24, GSX_ERR_ARG, "ksplat_pack: sh_count %d", sh_count);
    GSX_REQUIRE(level == 0 || bucket_size >= 1, GSX_ERR_ARG, "ksplat_pack: bucket_size %lld", (long long)bucket_size);
    if (n == 0) return GSX_OK;
    CodecCols cols{};
    if ((rc = fill_cols(cols14, sh_cols, sh_count, F, cols, "ksplat_pack"))) return rc;
    GSX_REQUIRE(rows && out && (level == 0 || centres), GSX_ERR_ARG, "ksplat_pack: null device pointer");
    const int lv = level < 3 ? level : 3;
    const int rec = gsx_ksplat_record_bytes(lv, sh_count);
    const size_t smem = tile_bytes(cols.ncol) + (size_t)kThreads * rec + 16;
    k_ksplat_pack<<<(int)((n + kThreads - 1) / kThreads), kThreads, smem, st>>>(rows, n, F, cols, lv, bucket_size, sf_inv,
                                                                                 centres, rec, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_spz_pack(const float* rows, int64_t n, int32_t F, const int32_t* cols14, const int32_t* sh_cols, int32_t sh_dim,
                 uint8_t* body, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_n(n, F, "spz_pack");
    if (rc) return rc;
    GSX_REQUIRE(sh_dim == 0 || sh_dim == 3 || sh_dim == 8 || sh_dim == 15, GSX_ERR_ARG, "spz_pack: sh_dim %d", sh_dim);
    if (n == 0) return GSX_OK;
    CodecCols cols{};
    if ((rc = fill_cols(cols14, sh_cols, 3 * sh_dim, F, cols, "spz_pack"))) return rc;
    GSX_REQUIRE(rows && body, GSX_ERR_ARG, "spz_pack: null device pointer");
    const size_t smem = tile_bytes(cols.ncol) + (size_t)kThreads * (20 + 3 * sh_dim) + 16;
    k_spz_pack<<<(int)((n + kThreads - 1) / kThreads), kThreads, smem, st>>>(rows, n, F, cols, body);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_splat_sort_keys(const float* rows, int64_t n, int32_t F, const int32_t* cols4, uint64_t* keys, int32_t* vals,
                        void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_n(n, F, "splat_sort_keys");
    if (rc) return rc;
    GSX_REQUIRE(cols4, GSX_ERR_ARG, "splat_sort_keys: no column table");
    for (int a = 0; a < 4; ++a)
        GSX_REQUIRE(cols4[a] >= 0 && cols4[a] < F, GSX_ERR_ARG, "splat_sort_keys: column %d out of range [0,%d)",
                    cols4[a], F);
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(rows && keys && vals, GSX_ERR_ARG, "splat_sort_keys: null device pointer");
    k_splat_sort_keys<<<(int)((n + 255) / 256), 256, 0, st>>>(rows, n, F, cols4[0], cols4[1], cols4[2], cols4[3], keys,
                                                              vals);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_splat_pack(const float* rows, int64_t n, int32_t F, const int32_t* order, const int32_t* cols14, uint8_t* out,
                   void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_n(n, F, "splat_pack");
    if (rc) return rc;
    if (n == 0) return GSX_OK;
    CodecCols cols{};
    if ((rc = fill_cols(cols14, nullptr, 0, F, cols, "splat_pack"))) return rc;
    GSX_REQUIRE(rows && order && out, GSX_ERR_ARG, "splat_pack: null device pointer");
    const size_t smem = tile_bytes(cols.ncol) + (size_t)kThreads * 32 + 16;
    k_splat_pack<<<(int)((n + kThreads - 1) / kThreads), kThreads, smem, st>>>(rows, n, F, order, cols, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_records_from_bytes(const uint8_t* src, int64_t n, int64_t row_bytes, const int32_t* offsets, int32_t nf,
                           float* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 0 && row_bytes >= 1, GSX_ERR_ARG, "records_from_bytes: bad sizes");
    GSX_REQUIRE(nf >= 1 && nf <= 256 && offsets, GSX_ERR_ARG, "records_from_bytes: %d fields (1..256)", nf);
    ByteFields f{};
    for (int k = 0; k < nf; ++k) {
        GSX_REQUIRE(offsets[k] >= 0 && offsets[k] + 4 <= row_bytes, GSX_ERR_ARG,
                    "records_from_bytes: field offset %d outside the %lld-byte row", offsets[k], (long long)row_bytes);
        f.off[k] = offsets[k];
    }
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(src && out, GSX_ERR_ARG, "records_from_bytes: null device pointer");
    const int64_t want = (n * nf + 255) / 256;
    const int blocks = (int)(want < 32 * (int64_t)sm_count() ? want : 32 * (int64_t)sm_count());
    k_records_from_bytes<<<blocks, 256, 0, st>>>(src, n, row_bytes, f, nf, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

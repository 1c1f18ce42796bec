// gsx_sog_decode.cu -- the SOG reader's per-splat decoding for sm_90a (H100): formats/sog.py:23-247 (SogFormat.read)
// after the WebP step, on the textures' RGBA pixels.
//
//   k_sog_palette  sog.py:181-211: the P x coeffs float32 palette, entry [i, c * C + j] = codebook[centroid byte c of
//                  pixel (i / 64) * w_c + (i % 64) * C + j], C = coeffs / 3, w_c = 64 * coeffs.  This is the reader's
//                  index formula, not the writer's (which packs entry (i, j) at pixel i * C + j), so palette entries
//                  >= 64 read other entries' bytes or the 255 padding, as the reference reader does.
//   k_sog_decode   sog.py:60-245: one splat per thread -> one row of define_dtype(sh_degree = bands): positions through
//                  three 65 536-entry tables, scale and DC codebook gathers, the opacity table, the quaternion rebuilt
//                  from its three stored components (max_comp = alpha - 252 as uint8; any other value leaves rot_* 0),
//                  nx / ny / nz 0, f_rest = palette[R | G << 8 of the labels texture].
//
// The position, quaternion-component and opacity maps are float32 tables the caller builds with the reference's own
// NumPy expressions (float64 exp for positions), so only the quaternion's sum of squares, 1 - s, max and sqrt are
// computed here, one __f*_rn operation per NumPy operation in NumPy's order ((a*a + b*b) + c*c).  An index the
// reference rejects with IndexError (a codebook index past the codebook's length, a label >= P) sets a bit of *err;
// the row gets 0 there and the caller refuses the file.  128 threads per CTA; rows are built in shared memory and
// stored as 16-byte words (gsx_staged.cuh): SH-3 rows are 248 bytes, not a multiple of 16.
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_staged.cuh"

#include <algorithm>

namespace gsx {

// bits of the error word: the index the reference reader rejects with IndexError
constexpr int32_t kSogErrScaleCodebook = 1, kSogErrSh0Codebook = 2, kSogErrShCodebook = 4, kSogErrLabel = 8;

struct SogTextures {   // RGBA pixels, 4-byte aligned; labels null without shN
    const uint8_t *means_l, *means_u, *quats, *scales, *sh0, *labels;
};

namespace {

constexpr int kRows = 128;         // rows per CTA
constexpr int kMaxRow = 4 * (17 + 45);

__device__ __forceinline__ uint32_t px(const uint8_t* __restrict__ t, int64_t i) {
    return __ldg(reinterpret_cast<const uint32_t*>(t) + i);
}

__global__ void __launch_bounds__(256) k_sog_palette(const uint8_t* __restrict__ cpx, int64_t P, int coeffs,
                                                     const float* __restrict__ cb, int ncb, float* __restrict__ pal,
                                                     int32_t* __restrict__ err) {
    const int C = coeffs / 3;
    const int64_t w_c = 64 * (int64_t)coeffs, total = P * coeffs;
    int bad = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = e / coeffs;
        const int k = (int)(e - i * coeffs), c = k / C, j = k - c * C;
        const int idx = __ldg(cpx + ((i / 64) * w_c + (i % 64) * C + j) * 4 + c);
        bad |= idx >= ncb;
        pal[e] = idx < ncb ? __ldg(cb + idx) : 0.f;
    }
    if (bad) atomicOr(err, kSogErrShCodebook);
}

__global__ void __launch_bounds__(kRows) k_sog_decode(const SogTextures tx, int64_t n, const float* __restrict__ pos,
                                                      const float* __restrict__ tables, int nscb, int nccb,
                                                      const float* __restrict__ pal, int64_t P, int coeffs,
                                                      uint8_t* __restrict__ out, int32_t* __restrict__ err) {
    __shared__ float qtab[256], otab[256], scb[256], ccb[256];
    __shared__ int32_t lab[kRows];
    __shared__ __align__(16) float stage[kRows * kMaxRow / 4 + 4];
    for (int k = threadIdx.x; k < 256; k += kRows) {
        qtab[k] = __ldg(tables + k), otab[k] = __ldg(tables + 256 + k);
        scb[k] = __ldg(tables + 512 + k), ccb[k] = __ldg(tables + 768 + k);
    }
    __syncthreads();
    const int t = threadIdx.x, F = 17 + coeffs;
    const int64_t base = (int64_t)blockIdx.x * kRows;
    const int rows_here = (int)(n - base < kRows ? n - base : kRows);
    int bad = 0;
    if (t < rows_here) {
        const int64_t i = base + t;
        float* r = stage + t * F;
        const uint32_t ml = px(tx.means_l, i), mu = px(tx.means_u, i), q = px(tx.quats, i), s = px(tx.scales, i),
                       c = px(tx.sh0, i);
#pragma unroll
        for (int a = 0; a < 3; ++a) {   // u16 = low | high << 8 per channel
            const uint32_t u = (ml >> 8 * a & 0xffu) | (mu >> 8 * a & 0xffu) << 8;
            r[a] = __ldg(pos + 65536 * a + u);
            r[3 + a] = 0.f;   // nx, ny, nz
            const uint32_t ci = c >> 8 * a & 0xffu, si = s >> 8 * a & 0xffu;
            bad |= (ci >= (uint32_t)nccb ? kSogErrSh0Codebook : 0) | (si >= (uint32_t)nscb ? kSogErrScaleCodebook : 0);
            r[6 + a] = ci < (uint32_t)nccb ? ccb[ci] : 0.f;
            r[10 + coeffs + a] = si < (uint32_t)nscb ? scb[si] : 0.f;
        }
        r[9 + coeffs] = otab[c >> 24];
        // sog.py:108-142: q_rest, max_comp = uint8(alpha - 252), missing = sqrt(max(1 - sum(q_rest**2), 0))
        const float x = qtab[q & 0xffu], y = qtab[q >> 8 & 0xffu], z = qtab[q >> 16 & 0xffu];
        const float ss = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
        const float m = __fsqrt_rn(fmaxf(__fsub_rn(1.f, ss), 0.f));
        const uint32_t mc = (q >> 24) - 252u & 0xffu;
        float* rot = r + 13 + coeffs;
        rot[0] = mc == 0 ? m : mc <= 3 ? x : 0.f;
        rot[1] = mc == 1 ? m : mc == 0 ? x : mc <= 3 ? y : 0.f;
        rot[2] = mc == 2 ? m : mc <= 1 ? y : mc == 3 ? z : 0.f;
        rot[3] = mc == 3 ? m : mc <= 2 ? z : 0.f;
        if (tx.labels) {
            const uint32_t l = px(tx.labels, i) & 0xffffu;
            bad |= (int64_t)l >= P ? kSogErrLabel : 0;
            lab[t] = (int64_t)l < P ? (int32_t)l : -1;
        }
    }
    if (coeffs) {   // f_rest: the rows' palette entries, consecutive threads on consecutive floats of one entry
        __syncthreads();
        for (int e = t; e < rows_here * coeffs; e += kRows) {
            const int row = e / coeffs, k = e - row * coeffs, l = lab[row];
            stage[row * F + 9 + k] = l >= 0 ? __ldg(pal + (int64_t)l * coeffs + k) : 0.f;
        }
    }
    if (bad) atomicOr(err, bad);
    __syncthreads();
    store_staged(out + base * 4 * F, reinterpret_cast<const uint8_t*>(stage), rows_here * 4 * F);
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_sog_decode_palette(const uint8_t* centroids, int64_t P, int32_t coeffs, const float* codebook, int32_t ncb,
                           float* palette, int32_t* err, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(coeffs == 0 || coeffs == 9 || coeffs == 24 || coeffs == 45, GSX_ERR_ARG,
                "sog_decode_palette: coeffs %d (0, 9, 24 or 45)", coeffs);
    GSX_REQUIRE(P >= 0 && P * coeffs < 2147483648ll, GSX_ERR_UNSUPPORTED,
                "sog_decode_palette: %lld palette entries of %d values", (long long)P, coeffs);
    GSX_REQUIRE(ncb >= 0, GSX_ERR_ARG, "sog_decode_palette: codebook length %d < 0", ncb);
    if (P == 0 || coeffs == 0) return GSX_OK;
    GSX_REQUIRE(centroids && palette && err && (ncb == 0 || codebook), GSX_ERR_ARG,
                "sog_decode_palette: null device pointer");
    const int64_t total = P * coeffs;
    const int grid = (int)std::min<int64_t>((total + 255) / 256, 132 * 16);
    k_sog_palette<<<grid, 256, 0, st>>>(centroids, P, coeffs, codebook, ncb < 256 ? ncb : 256, palette, err);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_sog_decode(const uint8_t* const* textures_host, int64_t n, const float* pos_tables, const float* tables,
                   int32_t nscb, int32_t nccb, const float* palette, int64_t P, int32_t coeffs, uint8_t* rows,
                   int32_t* err, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(textures_host, GSX_ERR_ARG, "gsx_sog_decode: no texture table");
    const SogTextures tx{textures_host[0], textures_host[1], textures_host[2],
                         textures_host[3], textures_host[4], textures_host[5]};
    GSX_REQUIRE(n >= 0, GSX_ERR_ARG, "sog_decode: n=%lld < 0", (long long)n);
    GSX_REQUIRE(n < 2147483648ll, GSX_ERR_UNSUPPORTED, "sog_decode: n=%lld needs n < 2^31", (long long)n);
    GSX_REQUIRE(coeffs == 0 || coeffs == 9 || coeffs == 24 || coeffs == 45, GSX_ERR_ARG,
                "sog_decode: coeffs %d (0, 9, 24 or 45)", coeffs);
    GSX_REQUIRE(nscb >= 0 && nccb >= 0, GSX_ERR_ARG, "sog_decode: negative codebook length");
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(coeffs == 0 || tx.labels, GSX_ERR_ARG, "sog_decode: SH coefficients without a labels texture");
    GSX_REQUIRE(!tx.labels || P >= 1, GSX_ERR_ARG, "sog_decode: a labels texture needs a palette (P=%lld)",
                (long long)P);
    GSX_REQUIRE(tx.means_l && tx.means_u && tx.quats && tx.scales && tx.sh0 && pos_tables && tables && rows && err &&
                    (coeffs == 0 || palette),
                GSX_ERR_ARG, "sog_decode: null device pointer");
    const uint8_t* const ptrs[6] = {tx.means_l, tx.means_u, tx.quats, tx.scales, tx.sh0, tx.labels};
    for (const uint8_t* p : ptrs)
        GSX_REQUIRE(((uintptr_t)p & 3) == 0, GSX_ERR_ARG, "sog_decode: texture pixels must be 4-byte aligned");
    k_sog_decode<<<(int)((n + kRows - 1) / kRows), kRows, 0, st>>>(tx, n, pos_tables, tables, nscb < 256 ? nscb : 256,
                                                                   nccb < 256 ? nccb : 256, palette, P, coeffs, rows,
                                                                   err);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

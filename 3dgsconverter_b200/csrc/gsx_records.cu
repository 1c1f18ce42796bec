// gsx_records.cu -- device-resident splat records (SURVEY 8(f) items 2 and 4) for sm_90a (H100).
//
// The reference's interchange record is a packed row of F float32 fields (structures.py:23-59: 62 fields = 248 bytes
// for SH degree 3).  Every filter of the reference extracts xyz / opacity with np.column_stack
// (data_processor.py:38,139) and compacts the records with a boolean fancy-index (:114,149,209,224) on the host --
// 248 bytes per splat through a single CPU thread, the dominant non-kernel cost of the cheap filters.  Here the rows
// are uploaded ONCE, the columns the filters read are extracted on the device, the survivors are gathered on the
// device, and the host sees one D2H of the final rows.
//   k_extract_xyz_op : row-major records -> xyz [n,3] + opacity [n]              (column_stack((x,y,z)), v['opacity'])
//   k_gather_rows    : out[j,:] = rows[idx[j],:]                                  (vertices[mask] for ascending idx)
// and the elementwise attribute transforms every writer applies (formats/splat.py:92-147, ksplat.py:464-483,
// spz.py:112-141, data_processor.py:301-333), fused over the resident rows:
//   k_color_dc_u8    : clip((0.5 + C0*f_dc) * 255, 0, 255).astype(uint8) x3 + clip(sigmoid(opacity)*255).astype(uint8)
//                      -> RGBA8 (float32 ops in NumPy's order; the colour channels are bit-exact, the alpha channel
//                      goes through expf and can differ from NumPy's SIMD exp by one count on ~1e-5 of the splats)
//   k_scale_exp      : exp(scale_0..2) -> float32 [n,3]
#include "gsx_common.cuh"
#include "gsx_records.cuh"

namespace gsx {

__global__ void __launch_bounds__(256) k_extract_xyz_op(const float* __restrict__ rows, int64_t n, int F, int cx,
                                                        int cy, int cz, int cop, float* __restrict__ xyz,
                                                        float* __restrict__ opacity) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* r = rows + (size_t)i * F;
    xyz[3 * i] = __ldg(r + cx);
    xyz[3 * i + 1] = __ldg(r + cy);
    xyz[3 * i + 2] = __ldg(r + cz);
    if (opacity) opacity[i] = __ldg(r + cop);
}

// one warp per output row: 32 lanes stride over the F floats of the row (coalesced on both sides)
__global__ void __launch_bounds__(256) k_gather_rows(const float* __restrict__ rows, const int32_t* __restrict__ idx,
                                                     int64_t m, int F, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= m) return;
    const float* src = rows + (size_t)idx[j] * F;
    float* dst = out + (size_t)j * F;
    for (int f = lane; f < F; f += 32) dst[f] = __ldg(src + f);
}

__device__ __forceinline__ uint8_t to_u8_clip(float v) {  // np.clip(v, 0, 255).astype(np.uint8): truncation
    v = fminf(fmaxf(v, 0.f), 255.f);
    return (uint8_t)v;
}

__global__ void __launch_bounds__(256) k_color_dc_u8(const float* __restrict__ rows, int64_t n, int F, int c0, int c1,
                                                     int c2, int cop, float scale, uchar4* __restrict__ rgba) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* r = rows + (size_t)i * F;
    uchar4 o;
    // (0.5 + SH_C0 * f) * 255 : float32 mul, add, mul in NumPy's order (python-float constants are weak scalars)
    o.x = to_u8_clip(__fmul_rn(__fadd_rn(0.5f, __fmul_rn(scale, __ldg(r + c0))), 255.f));
    o.y = to_u8_clip(__fmul_rn(__fadd_rn(0.5f, __fmul_rn(scale, __ldg(r + c1))), 255.f));
    o.z = to_u8_clip(__fmul_rn(__fadd_rn(0.5f, __fmul_rn(scale, __ldg(r + c2))), 255.f));
    // (1 / (1 + exp(-op))) * 255
    const float e = expf(-__ldg(r + cop));
    o.w = to_u8_clip(__fmul_rn(__fdiv_rn(1.0f, __fadd_rn(1.0f, e)), 255.f));
    rgba[i] = o;
}

__global__ void __launch_bounds__(256) k_scale_exp(const float* __restrict__ rows, int64_t n, int F, int s0, int s1,
                                                   int s2, float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* r = rows + (size_t)i * F;
    out[3 * i] = expf(__ldg(r + s0));
    out[3 * i + 1] = expf(__ldg(r + s1));
    out[3 * i + 2] = expf(__ldg(r + s2));
}

static int check_cols(int F, std::initializer_list<int> cols) {
    for (int c : cols) GSX_REQUIRE(c >= 0 && c < F, GSX_ERR_ARG, "records: column %d out of range [0,%d)", c, F);
    return GSX_OK;
}

int records_extract_xyz_opacity(const float* rows, int64_t n, int F, int cx, int cy, int cz, int cop, float* xyz,
                                float* opacity, cudaStream_t st) {
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(F >= 3, GSX_ERR_ARG, "records: bad row width %d", F);
    int rc = check_cols(F, {cx, cy, cz});
    if (rc) return rc;
    if (opacity && (rc = check_cols(F, {cop}))) return rc;
    k_extract_xyz_op<<<(int)((n + 255) / 256), 256, 0, st>>>(rows, n, F, cx, cy, cz, cop, xyz, opacity);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int records_gather_rows(const float* rows, const int32_t* idx, int64_t m, int F, float* out, cudaStream_t st) {
    if (m == 0) return GSX_OK;
    GSX_REQUIRE(F >= 1, GSX_ERR_ARG, "records: bad row width %d", F);
    k_gather_rows<<<(int)((m * 32 + 255) / 256), 256, 0, st>>>(rows, idx, m, F, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int records_color_rgba8(const float* rows, int64_t n, int F, int c0, int c1, int c2, int cop, float scale, uint8_t* rgba,
                        cudaStream_t st) {
    if (n == 0) return GSX_OK;
    int rc = check_cols(F, {c0, c1, c2, cop});
    if (rc) return rc;
    k_color_dc_u8<<<(int)((n + 255) / 256), 256, 0, st>>>(rows, n, F, c0, c1, c2, cop, scale, (uchar4*)rgba);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int records_scale_exp(const float* rows, int64_t n, int F, int s0, int s1, int s2, float* out, cudaStream_t st) {
    if (n == 0) return GSX_OK;
    int rc = check_cols(F, {s0, s1, s2});
    if (rc) return rc;
    k_scale_exp<<<(int)((n + 255) / 256), 256, 0, st>>>(rows, n, F, s0, s1, s2, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // namespace gsx

// gsx_masks.cu -- bbox crop and opacity keep-masks (pure streaming, HBM-bound).
//
// Replaces data_processor.py:215-231 (crop_by_bbox) and :184-213 (apply_alpha_filter); arithmetic
// per SURVEY A.4: bbox = six closed-interval float32 compares (the Python-float bounds are NumPy-2
// weak scalars, i.e. rounded to float32 by the caller); alpha = float64 compare of the float32
// opacity against the float64 logit threshold.
#include "../../include/gsx.h"

#include "gsx_common.cuh"

#include <math.h>

namespace gsx {

// 4 points (48 B = 3 x float4) per thread: fully coalesced 128-bit loads of the AoS xyz rows.
__global__ void __launch_bounds__(256) k_bbox_mask4(const float4* __restrict__ xyz4, int64_t n4, float lx, float ly,
                                                    float lz, float hx, float hy, float hz,
                                                    uchar4* __restrict__ mask4) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n4) return;
    float4 a = ld_stream_f4(xyz4 + 3 * t), b = ld_stream_f4(xyz4 + 3 * t + 1), c = ld_stream_f4(xyz4 + 3 * t + 2);
    // a = x0 y0 z0 x1 | b = y1 z1 x2 y2 | c = z2 x3 y3 z3
    uchar4 o;
    o.x = a.x >= lx && a.x <= hx && a.y >= ly && a.y <= hy && a.z >= lz && a.z <= hz;
    o.y = a.w >= lx && a.w <= hx && b.x >= ly && b.x <= hy && b.y >= lz && b.y <= hz;
    o.z = b.z >= lx && b.z <= hx && b.w >= ly && b.w <= hy && c.x >= lz && c.x <= hz;
    o.w = c.y >= lx && c.y <= hx && c.z >= ly && c.z <= hy && c.w >= lz && c.w <= hz;
    mask4[t] = o;
}

__global__ void __launch_bounds__(256) k_bbox_mask1(const float* __restrict__ xyz, int64_t begin, int64_t n, float lx,
                                                    float ly, float lz, float hx, float hy, float hz,
                                                    uint8_t* __restrict__ mask) {
    int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    mask[i] = x >= lx && x <= hx && y >= ly && y <= hy && z >= lz && z <= hz;
}

__global__ void __launch_bounds__(256) k_alpha_mask(const float* __restrict__ op, int64_t begin, int64_t n, double t,
                                                    uint8_t* __restrict__ mask) {
    int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) mask[i] = (double)op[i] >= t;
}

__global__ void __launch_bounds__(256) k_alpha_mask4(const float4* __restrict__ op4, int64_t n4, double t,
                                                     uchar4* __restrict__ mask4) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 v = ld_stream_f4(op4 + i);
    mask4[i] = make_uchar4((double)v.x >= t, (double)v.y >= t, (double)v.z >= t, (double)v.w >= t);
}

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_bbox_mask(const float* xyz, int64_t n, const float* lohi, uint8_t* mask, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 0, GSX_ERR_ARG, "bbox: n < 0");
    if (n == 0) return GSX_OK;
    int64_t n4 = 0;
    if (((uintptr_t)xyz % 16 == 0) && ((uintptr_t)mask % 4 == 0)) {
        n4 = n / 4;
        if (n4 > 0) {
            k_bbox_mask4<<<(int)((n4 + 255) / 256), 256, 0, st>>>((const float4*)xyz, n4, lohi[0], lohi[1], lohi[2],
                                                                   lohi[3], lohi[4], lohi[5], (uchar4*)mask);
            GSX_KERNEL_CHECK();
        }
    }
    int64_t rest = n - 4 * n4;
    if (rest > 0) {
        k_bbox_mask1<<<(int)((rest + 255) / 256), 256, 0, st>>>(xyz, 4 * n4, n, lohi[0], lohi[1], lohi[2], lohi[3],
                                                                lohi[4], lohi[5], mask);
        GSX_KERNEL_CHECK();
    }
    return GSX_OK;
}

int gsx_alpha_mask(const float* opacity, int64_t n, double logit_thresh, uint8_t* mask, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 0, GSX_ERR_ARG, "alpha: n < 0");
    if (n == 0) return GSX_OK;
    int64_t n4 = 0;
    if (((uintptr_t)opacity % 16 == 0) && ((uintptr_t)mask % 4 == 0)) {
        n4 = n / 4;
        if (n4 > 0) {
            k_alpha_mask4<<<(int)((n4 + 255) / 256), 256, 0, st>>>((const float4*)opacity, n4, logit_thresh,
                                                                    (uchar4*)mask);
            GSX_KERNEL_CHECK();
        }
    }
    if (n - 4 * n4 > 0) {
        k_alpha_mask<<<(int)((n - 4 * n4 + 255) / 256), 256, 0, st>>>(opacity, 4 * n4, n, logit_thresh, mask);
        GSX_KERNEL_CHECK();
    }
    return GSX_OK;
}

double gsx_alpha_logit_threshold(double min_opacity_u8) {
    double a = min_opacity_u8 / 255.0;
    if (a < 1e-6) a = 1e-6;
    if (a > 1.0 - 1e-6) a = 1.0 - 1e-6;
    return log(a / (1.0 - a));
}

}  // extern "C"

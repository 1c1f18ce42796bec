// gsx_numpy_scalar.cuh -- NumPy 2's float32 scalar semantics on x86-64, for the .splat / .ksplat / .spz writers
// (device code only).
//
//   numpy_expf     NumPy's SIMD float32 exp (AVX2 and AVX-512F give the same bytes): Cody-Waite reduction by ln 2,
//                  a [5/2] rational approximation and an exact scaling by 2^q.  It is not correctly rounded (up to 2 ulp
//                  from exp), so expf or a double exp rounded once would not reproduce the writers' raw float32 scales.
//   np_i32         float -> int32 (astype): cvttps2dq, NaN and out-of-range values give INT32_MIN.
//   np_u8, np_u16  float -> uint8 / uint16: the int32 conversion above, truncated to the low bits (NaN -> 0).
//   np_clip        np.clip, which keeps NaN (fminf / fmaxf do not).
//   numpy_f2h      float32 -> float16: round half to even, except NaN: sign | 0x7c00 | mantissa >> 13, a zero result
//                  mantissa becoming 1 (CUDA's __float2half_rn gives 0x7fff for every NaN).
// Every step is an explicit __f*_rn / __fmaf_rn operation, so nothing is contracted whatever the build flags are.
#pragma once
#include <cuda_fp16.h>
#include "gsx_common.cuh"

namespace gsx {

__device__ __forceinline__ float numpy_expf(float x) {
    if (x != x) return __uint_as_float(0x7fc00000u);   // NumPy's output for every NaN input
    if (x > 88.7228394f) return __uint_as_float(0x7f800000u);
    if (x < -103.972084f) return 0.f;
    const float q = rintf(__fmul_rn(x, 1.442695040888963407359924681001892137f));   // round half to even
    float y = __fmaf_rn(q, -6.93145752e-1f, x);
    y = __fmaf_rn(q, -1.42860677e-6f, y);
    float num = 5.082762527590693718096e-04f;
    num = __fmaf_rn(num, y, 6.757896990527504603057e-03f);
    num = __fmaf_rn(num, y, 5.114512081637298353406e-02f);
    num = __fmaf_rn(num, y, 2.473615434895520810817e-01f);
    num = __fmaf_rn(num, y, 7.257664613233124478488e-01f);
    num = __fmaf_rn(num, y, 9.999999999980870924916e-01f);
    float den = 2.159509375685829852307e-02f;
    den = __fmaf_rn(den, y, -2.742335390411667452936e-01f);
    den = __fmaf_rn(den, y, 1.0f);
    // r * 2^q is exact in double (|q| <= 150, r normal), so one rounding gives the correctly rounded scalef result,
    // subnormal and overflowing results included
    const double s = (double)__fdiv_rn(num, den) * __longlong_as_double((long long)(1023 + (int)q) << 52);
    return __double2float_rn(s);
}

__device__ __forceinline__ int32_t np_i32(float v) {
    return (v != v || v >= 2147483648.f || v < -2147483648.f) ? INT32_MIN : (int32_t)v;
}

__device__ __forceinline__ uint8_t np_u8(float v) { return (uint8_t)(uint32_t)np_i32(v); }
__device__ __forceinline__ uint16_t np_u16(float v) { return (uint16_t)(uint32_t)np_i32(v); }

__device__ __forceinline__ float np_clip(float v, float lo, float hi) { return v != v ? v : fminf(fmaxf(v, lo), hi); }

__device__ __forceinline__ uint16_t numpy_f2h(float v) {
    if (v != v) {
        const uint32_t b = __float_as_uint(v);
        const uint32_t m = (b & 0x007fffffu) >> 13;
        return (uint16_t)((b >> 16 & 0x8000u) | 0x7c00u | (m ? m : 1u));
    }
    return __half_as_ushort(__float2half_rn(v));
}

}  // namespace gsx

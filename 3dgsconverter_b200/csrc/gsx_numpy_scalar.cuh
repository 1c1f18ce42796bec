// gsx_numpy_scalar.cuh -- NumPy 2's float32 scalar semantics on x86-64, for the .splat / .ksplat / .spz writers and
// readers, the SOG writer's position log and opacity exp, the compressed PLY alpha and the records' colour alpha and
// scale exp (device code only).
//
//   numpy_expf     NumPy's SIMD float32 exp (AVX2 and AVX-512F give the same bytes): Cody-Waite reduction by ln 2,
//                  a [5/2] rational approximation and an exact scaling by 2^q.  It is not correctly rounded (up to 2 ulp
//                  from exp), so expf or a double exp rounded once would not reproduce the writers' raw float32 scales.
//   numpy_logf     NumPy's SIMD float32 log (AVX-512F), on the .splat reader's domain (which holds the SOG writer's
//                  |v| + 1 >= 1).
//   numpy_h2f      float16 -> float32 as astype(np.float32), NaN payloads kept.
//   x86_*          float / double add, sub, mul, div and conversions with x86's NaN results (first NaN operand quieted,
//                  the negative default NaN for invalid operations), where NaN inputs reach a reader's output.
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

// NumPy's SIMD float32 log (AVX-512F): x = m * 2^e with m in [0.5, 1) (getmant / getexp), m <= sqrt(1/2) doubled,
// a [5/5] rational approximation of log(1 + (m - 1)), then fma(e, ln 2, p).  Not correctly rounded either (about 5 %
// of inputs differ from a correctly rounded log), so logf or a double log would not reproduce the .splat reader's
// scales.  Checked exhaustively against np.log on every float32 >= 1e-6, +inf and NaN: the domain max(s, 1e-6) of the
// reader.  Subnormal inputs are outside it (the exponent is read from the bits).
__device__ __forceinline__ float numpy_logf(float x) {
    if (x != x) return __uint_as_float(0x7fc00000u);   // NumPy's output for every NaN input
    if (x < 0.f) return __uint_as_float(0xffc00000u);
    if (x == 0.f) return __uint_as_float(0xff800000u);
    if (x == __uint_as_float(0x7f800000u)) return x;
    const uint32_t b = __float_as_uint(x);
    float e = (float)((int)(b >> 23) - 126);
    float m = __uint_as_float((b & 0x007fffffu) | 0x3f000000u);   // [0.5, 1)
    if (m <= 0.707106781186547524400844362104849039f) m = __fadd_rn(m, m), e = __fsub_rn(e, 1.f);
    const float y = __fsub_rn(m, 1.f);
    float num = __fmaf_rn(2.589979117907922693523e-02f, y, 3.808837741388407920751e-01f);
    num = __fmaf_rn(num, y, 1.480000633576506585156e+00f);
    num = __fmaf_rn(num, y, 2.112677543073053063722e+00f);
    num = __fmaf_rn(num, y, 9.999999999999998702752e-01f);
    num = __fmaf_rn(num, y, 0.f);
    float den = __fmaf_rn(5.875095403124574342950e-03f, y, 1.546476374983906719538e-01f);
    den = __fmaf_rn(den, y, 9.864942958519418960339e-01f);
    den = __fmaf_rn(den, y, 2.453006071784736363091e+00f);
    den = __fmaf_rn(den, y, 2.612677543073109236779e+00f);
    den = __fmaf_rn(den, y, 1.f);
    return __fmaf_rn(e, 0.693147180559945309417232121458176568f, __fdiv_rn(num, den));
}

// float16 bits -> float32 as NumPy's astype(np.float32): NaN keeps its payload and is NOT quieted (signalling NaN
// patterns stay signalling), which the hardware conversion behind __half2float does not promise.
__device__ __forceinline__ float numpy_h2f(uint16_t h) {
    const uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = h & 0x7c00u, m = h & 0x03ffu;
    if (e == 0x7c00u) return __uint_as_float(s | 0x7f800000u | m << 13);
    if (e) return __uint_as_float(s + (((uint32_t)(h & 0x7fffu) + 0x1c000u) << 13));
    return __uint_as_float(s | __float_as_uint(__fmul_rn((float)m, 5.9604644775390625e-08f)));   // m * 2^-24, exact
}

// x86 SSE arithmetic on NaN: the first NaN operand is returned quieted, an invalid operation (inf - inf, 0 * inf)
// returns the negative "indefinite" NaN.  The GPU returns 0x7fffffff for all of these, and the bytes reach the output.
__device__ __forceinline__ bool x86_isnan(float a) { return a != a; }
__device__ __forceinline__ bool x86_isnan(double a) { return a != a; }
__device__ __forceinline__ float x86_quiet(float a) { return __uint_as_float(__float_as_uint(a) | 0x00400000u); }
__device__ __forceinline__ double x86_quiet(double a) {
    return __longlong_as_double(__double_as_longlong(a) | 0x0008000000000000ll);
}
__device__ __forceinline__ float x86_nan_of(float a, float b, float r) {
    return x86_isnan(a) ? x86_quiet(a) : x86_isnan(b) ? x86_quiet(b) : x86_isnan(r) ? __uint_as_float(0xffc00000u) : r;
}
__device__ __forceinline__ double x86_nan_of(double a, double b, double r) {
    return x86_isnan(a)   ? x86_quiet(a)
           : x86_isnan(b) ? x86_quiet(b)
           : x86_isnan(r) ? __longlong_as_double((long long)0xfff8000000000000ull)
                          : r;
}
__device__ __forceinline__ float x86_add(float a, float b) { return x86_nan_of(a, b, __fadd_rn(a, b)); }
__device__ __forceinline__ float x86_sub(float a, float b) { return x86_nan_of(a, b, __fsub_rn(a, b)); }
__device__ __forceinline__ float x86_mul(float a, float b) { return x86_nan_of(a, b, __fmul_rn(a, b)); }
__device__ __forceinline__ double x86_add(double a, double b) { return x86_nan_of(a, b, __dadd_rn(a, b)); }
__device__ __forceinline__ double x86_sub(double a, double b) { return x86_nan_of(a, b, __dadd_rn(a, -b)); }
__device__ __forceinline__ double x86_mul(double a, double b) { return x86_nan_of(a, b, __dmul_rn(a, b)); }
__device__ __forceinline__ double x86_div(double a, double b) { return x86_nan_of(a, b, __ddiv_rn(a, b)); }
// cvtss2sd / cvtsd2ss: a NaN is quieted and keeps the high bits of its payload
__device__ __forceinline__ double x86_f2d(float a) {
    if (!x86_isnan(a)) return (double)a;
    const uint32_t b = __float_as_uint(a);
    return __longlong_as_double((long long)((uint64_t)(b & 0x80000000u) << 32 | 0x7ff8000000000000ull |
                                            (uint64_t)(b & 0x003fffffu) << 29));
}
__device__ __forceinline__ float x86_d2f(double a) {
    if (!x86_isnan(a)) return __double2float_rn(a);
    const uint64_t b = (uint64_t)__double_as_longlong(a);
    return __uint_as_float((uint32_t)(b >> 32 & 0x80000000u) | 0x7fc00000u | (uint32_t)(b >> 29 & 0x003fffffu));
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

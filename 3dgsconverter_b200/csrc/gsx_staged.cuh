// gsx_staged.cuh -- block-cooperative byte movement between global memory at any alignment and shared memory, for
// the record packers (gsx_splat_codecs.cu) and readers (gsx_readers.cu): whole 16-byte words where they fit.
#pragma once
#include "gsx_common.cuh"

namespace gsx {

// dst[0, nbytes) = s[0, nbytes), block-cooperative: a byte head up to dst's 16-byte boundary, 16-byte words realigned
// from s's 32-bit words with funnel shifts, a byte tail.  s is 4-byte aligned with 4 readable bytes past nbytes.
__device__ __forceinline__ void store_staged(uint8_t* __restrict__ dst, const uint8_t* s, int nbytes) {
    const int a = (int)((uintptr_t)dst & 15);
    const int h = a ? (16 - a < nbytes ? 16 - a : nbytes) : 0;
    for (int i = threadIdx.x; i < h; i += blockDim.x) dst[i] = s[i];
    const int nvec = (nbytes - h) >> 4;
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(s) + (h >> 2);
    const uint32_t sh = (uint32_t)(h & 3) * 8;
    uint4* d4 = reinterpret_cast<uint4*>(dst + h);
    for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
        const uint32_t* p = s32 + 4 * v;
        const uint32_t x0 = p[0], x1 = p[1], x2 = p[2], x3 = p[3], x4 = p[4];
        d4[v] = make_uint4(__funnelshift_r(x0, x1, sh), __funnelshift_r(x1, x2, sh), __funnelshift_r(x2, x3, sh),
                           __funnelshift_r(x3, x4, sh));
    }
    for (int i = h + (nvec << 4) + threadIdx.x; i < nbytes; i += blockDim.x) dst[i] = s[i];
}

// The bytes src[0, nbytes) into shared memory, block-cooperative, as the 16-byte words of global memory that cover
// them: one vector load per word, from the word holding src[0] (inside src's allocation, which is 256-byte aligned);
// a last word that would reach past src[nbytes - 1] is read byte by byte.  `stage` is 16-byte aligned with
// nbytes + 16 bytes of room; returns where src[0] landed.  The caller synchronises before reading.
__device__ __forceinline__ const uint8_t* load_staged(uint8_t* stage, const uint8_t* __restrict__ src, int nbytes) {
    const int a = (int)((uintptr_t)src & 15);
    const uint4* s4 = reinterpret_cast<const uint4*>(src - a);
    uint4* d4 = reinterpret_cast<uint4*>(stage);
    const int full = (a + nbytes) >> 4;
    for (int v = threadIdx.x; v < full; v += blockDim.x) d4[v] = __ldg(s4 + v);
    for (int i = (full << 4) - a + threadIdx.x; i < nbytes; i += blockDim.x) stage[a + i] = __ldg(src + i);
    return stage + a;
}

// Rows of `crow` staged bytes each into rows of `row_bytes` bytes whose bytes [head, head + row_bytes - crow) stay
// as they are (zero-filled by the caller): for layouts too wide to stage whole, such as high SH degrees.
__device__ __forceinline__ void store_rows_gap(uint8_t* __restrict__ dst, const uint8_t* s, int rows, int crow, int head,
                                               int64_t row_bytes) {
    const int64_t gap = row_bytes - crow;
    for (int e = threadIdx.x; e < rows * crow; e += blockDim.x) {
        const int r = e / crow, c = e - r * crow;
        dst[r * row_bytes + c + (c < head ? 0 : gap)] = s[e];
    }
}

}  // namespace gsx

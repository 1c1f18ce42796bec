// gsx_deflate_format.cuh -- the DEFLATE (RFC 1951) code tables that the encoder (gsx_deflate.cu) and the decoder
// (gsx_inflate.cu) share.  The encoder computes a length's code (length_code); the decoder looks codes up in the tables.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gsx {

// the order in which a dynamic block header lists the code lengths of the code-length alphabet (RFC 1951 3.2.7)
static __constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
// length symbols 257..285 and distance symbols 0..29: the base value and the number of extra bits (RFC 1951 3.2.5)
static __constant__ uint16_t kLBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                           31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static __constant__ uint8_t kLExt[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static __constant__ uint16_t kDBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                           193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static __constant__ uint8_t kDExt[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

// length 3..258 -> symbol 257..285, its extra bits and their value: kLBase[sym - 257] + extra == L
__device__ __forceinline__ void length_code(uint32_t L, uint32_t& sym, uint32_t& nextra, uint32_t& extra) {
    if (L == 258) {
        sym = 285, nextra = 0, extra = 0;
        return;
    }
    const uint32_t v = L - 3;
    if (v < 8) {
        sym = 257 + v, nextra = 0, extra = 0;
        return;
    }
    const uint32_t h = 31 - __clz(v);
    nextra = h - 2;
    sym = 257 + 4 * (h - 1) + ((v >> nextra) & 3);
    extra = v & ((1u << nextra) - 1);
}

}  // namespace gsx

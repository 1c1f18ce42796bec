// gsx_sh_mask.cuh -- the SH column mask shared by the compressed PLY and SOG writers (device code only).
#pragma once
#include "gsx_common.cuh"

namespace gsx {

// "SH column k holds a value != 0" bits (the input of the writers' SH-degree rules): OR the 64-bit column masks of the
// 32 lanes and fold the result into *mask with one atomic per warp.  Every lane of the warp must call it.
__device__ __forceinline__ void warp_or_column_mask(unsigned long long bits, unsigned long long* mask) {
    const uint32_t lo = __reduce_or_sync(0xffffffffu, (uint32_t)bits);
    const uint32_t hi = __reduce_or_sync(0xffffffffu, (uint32_t)(bits >> 32));
    if ((threadIdx.x & 31) == 0 && (lo | hi)) atomicOr(mask, (unsigned long long)hi << 32 | lo);
}

}  // namespace gsx

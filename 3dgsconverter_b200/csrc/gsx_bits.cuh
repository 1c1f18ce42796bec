// gsx_bits.cuh -- device helpers for the byte- and bit-level formats: little-endian field access, order-preserving
// float keys and the LSB-first bit reader of DEFLATE and VP8L.  Kept out of gsx_common.cuh, which host-only builds of
// the copy engine (gsx_hostcopy.cu) also include, because these use device intrinsics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gsx {

// Little-endian loads and stores at any byte alignment.  putf advances p past the value.
__device__ __forceinline__ uint16_t get16(const uint8_t* p) { return (uint16_t)(p[0] | p[1] << 8); }
__device__ __forceinline__ uint32_t get32(const uint8_t* p) {
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}
__device__ __forceinline__ float getf(const uint8_t* p) { return __uint_as_float(get32(p)); }
__device__ __forceinline__ void put16(uint8_t* p, uint16_t v) { p[0] = (uint8_t)v, p[1] = (uint8_t)(v >> 8); }
__device__ __forceinline__ void put32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)v, p[1] = (uint8_t)(v >> 8), p[2] = (uint8_t)(v >> 16), p[3] = (uint8_t)(v >> 24);
}
__device__ __forceinline__ void putf(uint8_t*& p, float v) { put32(p, __float_as_uint(v)), p += 4; }

__host__ __device__ __forceinline__ size_t up16(size_t x) { return (x + 15) & ~(size_t)15; }

// Order-preserving float <-> uint32 (for integer min / max and radix keys): unsigned order of the keys is the float
// order, -0 below +0 and +-inf at the extremes of the numbers.  ord_to_float inverts float_to_ord.
__device__ __forceinline__ uint32_t float_to_ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord_to_float(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// The key of np.argsort's float order: -0 equal to +0, and every NaN, whatever its sign and payload, one key above
// +inf, so NaNs sort last and keep their index order in a stable sort.
__device__ __forceinline__ uint32_t numpy_sort_key(float f) {
    return f != f ? 0xffffffffu : float_to_ord(f + 0.0f);   // -0 + 0 = +0
}

// LSB-first bit reader over d[0, nbytes) (DEFLATE and VP8L streams): never reads past the end; need(k) is false when
// fewer than k bits remain.  A start past the end leaves no bits.
struct Reader {
    const uint8_t* d;
    int64_t nbytes, next;
    uint64_t buf;
    int cnt;

    __device__ void init(const uint8_t* d_, int64_t n, int64_t bit) {
        d = d_, nbytes = n, next = bit >> 3, buf = 0, cnt = 0;
        if (next > nbytes) next = nbytes;
        refill();
        drop(min(int(bit & 7), cnt));
    }
    __device__ __forceinline__ void refill() {
        while (cnt <= 56 && next < nbytes) buf |= uint64_t(__ldg(d + next++)) << cnt, cnt += 8;
    }
    __device__ __forceinline__ bool need(int k) {
        if (cnt < k) refill();
        return cnt >= k;
    }
    __device__ __forceinline__ uint32_t peek(int k) const { return uint32_t(buf & ((uint64_t(1) << k) - 1)); }
    __device__ __forceinline__ void drop(int k) { buf >>= k, cnt -= k; }
    __device__ __forceinline__ int64_t pos() const { return next * 8 - cnt; }
    // false when the stream ends first
    __device__ __forceinline__ bool bits(int k, uint32_t& v) {
        if (!need(k)) return false;
        v = peek(k);
        drop(k);
        return true;
    }
};

}  // namespace gsx

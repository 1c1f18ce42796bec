// gsx_vp8l_format.cuh -- the lossless WebP (VP8L, RFC 9649) rules that the encoder (gsx_webp.cu) and the decoder
// (gsx_vp8l.cu) share: the spatial predictors and the prefix coding of LZ77 lengths and distances.
#pragma once
#include "gsx_bits.cuh"

namespace gsx {

// channel k of an ARGB pixel (0 blue, 1 green, 2 red, 3 alpha)
__device__ __forceinline__ uint32_t chan(uint32_t p, int k) { return (p >> (8 * k)) & 0xFF; }

__device__ __forceinline__ uint32_t avg2(uint32_t a, uint32_t b) {
    return (((a ^ b) & 0xFEFEFEFEu) >> 1) + (a & b);
}

__device__ __forceinline__ uint32_t select_pred(uint32_t L, uint32_t T, uint32_t TL) {
    int pl = 0, pt = 0;
    for (int k = 0; k < 4; ++k) {
        pl += abs(int(chan(T, k)) - int(chan(TL, k)));
        pt += abs(int(chan(L, k)) - int(chan(TL, k)));
    }
    return pl < pt ? L : T;
}

__device__ __forceinline__ uint32_t clamp_full(uint32_t L, uint32_t T, uint32_t TL) {
    uint32_t out = 0;
    for (int k = 0; k < 4; ++k) {
        int v = int(chan(L, k)) + int(chan(T, k)) - int(chan(TL, k));
        out |= uint32_t(min(max(v, 0), 255)) << (8 * k);
    }
    return out;
}

__device__ __forceinline__ uint32_t clamp_half(uint32_t a, uint32_t b) {
    uint32_t out = 0;
    for (int k = 0; k < 4; ++k) {
        int ak = int(chan(a, k));
        int v = ak + (ak - int(chan(b, k))) / 2;   // C division: truncation toward zero, as the RFC states it
        out |= uint32_t(min(max(v, 0), 255)) << (8 * k);
    }
    return out;
}

// The prediction of predictor mode 0..13 from the left, top, top-right and top-left pixels.  A stream can also name
// modes 14 and 15; like mode 0 they predict opaque black.
__device__ __forceinline__ uint32_t predict(int mode, uint32_t L, uint32_t T, uint32_t TR, uint32_t TL) {
    switch (mode) {
        case 1: return L;
        case 2: return T;
        case 3: return TR;
        case 4: return TL;
        case 5: return avg2(avg2(L, TR), T);
        case 6: return avg2(L, TL);
        case 7: return avg2(L, T);
        case 8: return avg2(TL, T);
        case 9: return avg2(T, TR);
        case 10: return avg2(avg2(L, TL), avg2(T, TR));
        case 11: return select_pred(L, T, TL);
        case 12: return clamp_full(L, T, TL);
        case 13: return clamp_half(avg2(L, T), TL);
        default: return 0xFF000000u;
    }
}

// A copy length (or distance code) >= 1 as its prefix symbol `code` and `nbits` extra bits of value `extra`;
// prefix_value below is the inverse.
__device__ __forceinline__ void length_prefix(uint32_t length, uint32_t& code, uint32_t& nbits, uint32_t& extra) {
    uint32_t v = length - 1;
    if (v < 4) {
        code = v, nbits = 0, extra = 0;
        return;
    }
    uint32_t h = 31 - __clz(v);
    code = 2 * h + ((v >> (h - 1)) & 1);
    nbits = h - 1;
    extra = v & ((1u << nbits) - 1);
}

// The value of prefix symbol `sym`, its extra bits read from r; false when the stream ends first.
__device__ __forceinline__ bool prefix_value(Reader& r, uint32_t sym, uint32_t& out) {
    if (sym < 4) {
        out = sym + 1;
        return true;
    }
    const int extra = int(sym - 2) >> 1;
    uint32_t v;
    if (!r.bits(extra, v)) return false;
    out = ((2 + (sym & 1)) << extra) + v + 1;
    return true;
}

}  // namespace gsx

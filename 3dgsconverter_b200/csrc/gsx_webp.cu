// gsx_webp.cu -- the device half of the lossless WebP (VP8L) encoder: transforms, run copies, histograms and the
// bit emission of the entropy-coded images.  gsx/webp.py builds the Huffman codes from the histograms, picks the
// candidate and writes the headers; tests/webp_oracle.py restates every decision in NumPy.
//
// Per image the pipeline is:
//   k_webp_clean       RGBA bytes -> ARGB words, RGB cleared where alpha is 0 (image 0)
//   k_webp_predict     one block per 16x16 tile: the cost of the 14 predictors, the cheapest (lowest on a tie), the
//                      residuals (images 1 and 2) and the sub-image pixel (images 3 and 4)
//   k_webp_breaks      break[i] = i is 0 or differs from the pixel before it; exclusive scan -> run index
//   k_webp_run_starts  the first pixel of every run, by run index
//   k_webp_tokens      literal / copy head (length) / inside a copy, and the five histograms
// and for the chosen candidate:
//   k_webp_bits        the bits of each pixel's token; exclusive scan per 2^26 pixels -> bit offsets
//   k_webp_bases       the 64-bit base of each scanned chunk and the image's total
//   k_webp_emit        the LSB-first fields of every token ORed into a zeroed word buffer (a token straddles up to
//                      three 32-bit words)
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_radix.cuh"
#include "gsx_vp8l_format.cuh"

#include <algorithm>

namespace gsx {

constexpr int kWebpMaxSide = 16384;
constexpr int kWebpTreeSyms = 280 + 256 + 256 + 256 + 40;   // green + 24 lengths, red, blue, alpha, distance

namespace {

constexpr int kTile = 16;
constexpr int kModes = 14;
constexpr int kMaxCopy = 4096;
constexpr int kMinCopy = 3;
constexpr int64_t kScanChunk = int64_t(1) << 26;   // 2^26 tokens of at most 60 bits fit a uint32 offset
constexpr int kGreen = 0, kRed = 280, kBlue = 536, kAlpha = 792, kDist = 1048;
constexpr int kLeftDistSymbol = 1;                 // plane code 2 (the left pixel) -> prefix symbol 1, no extra bits

__device__ __forceinline__ uint32_t subtract_green(uint32_t p) {
    uint32_t g = chan(p, 1);
    return (p & 0xFF00FF00u) | (((chan(p, 2) - g) & 0xFF) << 16) | ((chan(p, 0) - g) & 0xFF);
}

// sum over the four channels of |residual as int8|
__device__ __forceinline__ int residual_cost(uint32_t r) {
    int s = 0;
    for (int k = 0; k < 4; ++k) s += abs(int(int8_t(chan(r, k))));
    return s;
}

__global__ void k_webp_clean(const uchar4* __restrict__ rgba, int64_t n, uint32_t* __restrict__ argb,
                             uint32_t* __restrict__ alpha_used) {
    bool used = false;
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        uchar4 p = rgba[i];
        argb[i] = p.w ? (uint32_t(p.w) << 24) | (uint32_t(p.x) << 16) | (uint32_t(p.y) << 8) | p.z : 0u;
        used |= p.w != 255;
    }
    if (__syncthreads_or(used) && threadIdx.x == 0) atomicOr(alpha_used, 1u);
}

template <bool SUBTRACT_GREEN>
__device__ __forceinline__ uint32_t load_src(const uint32_t* src, int64_t i) {
    uint32_t p = src[i];
    return SUBTRACT_GREEN ? subtract_green(p) : p;
}

// one block of 256 threads per 16x16 tile
template <bool SUBTRACT_GREEN>
__global__ void __launch_bounds__(256) k_webp_predict(const uint32_t* __restrict__ src, int W, int H, int tiles_x,
                                                      uint32_t* __restrict__ res, uint32_t* __restrict__ sub,
                                                      uint8_t* __restrict__ modes_out) {
    __shared__ int warp_cost[8][kModes];
    __shared__ int best;
    const int tile = blockIdx.x;
    const int x = (tile % tiles_x) * kTile + (threadIdx.x % kTile);
    const int y = (tile / tiles_x) * kTile + (threadIdx.x / kTile);
    const bool valid = x < W && y < H;
    const bool inner = valid && x > 0 && y > 0;
    const int64_t i = int64_t(y) * W + x;
    uint32_t c = 0, L = 0, T = 0, TR = 0, TL = 0;
    int cost[kModes];
#pragma unroll
    for (int m = 0; m < kModes; ++m) cost[m] = 0;
    if (inner) {
        c = load_src<SUBTRACT_GREEN>(src, i);
        L = load_src<SUBTRACT_GREEN>(src, i - 1);
        T = load_src<SUBTRACT_GREEN>(src, i - W);
        TL = load_src<SUBTRACT_GREEN>(src, i - W - 1);
        TR = load_src<SUBTRACT_GREEN>(src, i - W + 1);   // the rightmost column: the first pixel of this row
#pragma unroll
        for (int m = 0; m < kModes; ++m) cost[m] = residual_cost(__vsub4(c, predict(m, L, T, TR, TL)));
    }
    // edge pixels are predicted the same way under every mode, so they do not move the argmin
#pragma unroll
    for (int m = 0; m < kModes; ++m) {
        int v = cost[m];
        for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
        if ((threadIdx.x & 31) == 0) warp_cost[threadIdx.x >> 5][m] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int bm = 0, bc = 0x7FFFFFFF;
        for (int m = 0; m < kModes; ++m) {
            int s = 0;
            for (int w = 0; w < 8; ++w) s += warp_cost[w][m];
            if (s < bc) bc = s, bm = m;
        }
        best = bm;
        sub[tile] = 0xFF000000u | (uint32_t(bm) << 8);
        if (modes_out) modes_out[tile] = uint8_t(bm);
    }
    __syncthreads();
    if (!valid) return;
    uint32_t pred;
    if (inner) {
        pred = predict(best, L, T, TR, TL);
    } else {
        c = load_src<SUBTRACT_GREEN>(src, i);
        pred = x == 0 && y == 0 ? 0xFF000000u : load_src<SUBTRACT_GREEN>(src, y == 0 ? i - 1 : i - W);
    }
    res[i] = __vsub4(c, pred);
}

__device__ __forceinline__ bool is_break(const uint32_t* sym, int64_t i) { return i == 0 || sym[i] != sym[i - 1]; }

__global__ void k_webp_breaks(const uint32_t* __restrict__ sym, int64_t n, uint32_t* __restrict__ flags) {
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
        flags[i] = is_break(sym, i);
}

__global__ void k_webp_run_starts(const uint32_t* __restrict__ sym, int64_t n, const uint32_t* __restrict__ run,
                                  uint32_t* __restrict__ starts) {
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
        if (is_break(sym, i)) starts[run[i]] = uint32_t(i);
}

// tok: 1 = literal, L >= 3 = the first pixel of a copy of L pixels, 0 = inside a copy
__global__ void __launch_bounds__(256) k_webp_tokens(const uint32_t* __restrict__ sym, int64_t n,
                                                     const uint32_t* __restrict__ run,
                                                     const uint32_t* __restrict__ starts, uint16_t* __restrict__ tok,
                                                     uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[kWebpTreeSyms];
    for (int k = threadIdx.x; k < kWebpTreeSyms; k += blockDim.x) h[k] = 0;
    __syncthreads();
    const int64_t nruns = int64_t(run[n - 1]) + is_break(sym, n - 1);
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const bool b = is_break(sym, i);
        const int64_t r = int64_t(run[i]) + b - 1;
        const int64_t start = starts[r];
        const int64_t end = r + 1 < nruns ? int64_t(starts[r + 1]) : n;
        uint16_t t = 1;
        if (!b) {
            const int64_t k = i - start - 1, followers = end - start - 1;
            const int64_t q = k / kMaxCopy;
            const int64_t chunk = min(int64_t(kMaxCopy), followers - q * kMaxCopy);
            if (chunk >= kMinCopy) t = k % kMaxCopy == 0 ? uint16_t(chunk) : 0;
        }
        tok[i] = t;
        if (t == 1) {
            const uint32_t s = sym[i];
            atomicAdd(&h[kGreen + chan(s, 1)], 1u);
            atomicAdd(&h[kRed + chan(s, 2)], 1u);
            atomicAdd(&h[kBlue + chan(s, 0)], 1u);
            atomicAdd(&h[kAlpha + chan(s, 3)], 1u);
        } else if (t) {
            uint32_t code, nbits, extra;
            length_prefix(t, code, nbits, extra);
            atomicAdd(&h[kGreen + 256 + code], 1u);
            atomicAdd(&h[kDist + kLeftDistSymbol], 1u);
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < kWebpTreeSyms; k += blockDim.x)
        if (h[k]) atomicAdd(&hist[k], h[k]);
}

// table entry: bit-reversed code | length << 16
__device__ __forceinline__ uint32_t token_fields(uint32_t s, uint32_t t, const uint32_t* table, uint64_t& v) {
    uint32_t nb = 0;
    v = 0;
    auto put = [&](uint32_t e) {
        v |= uint64_t(e & 0xFFFF) << nb;
        nb += e >> 16;
    };
    if (t == 1) {
        put(table[kGreen + chan(s, 1)]);
        put(table[kRed + chan(s, 2)]);
        put(table[kBlue + chan(s, 0)]);
        put(table[kAlpha + chan(s, 3)]);
    } else {
        uint32_t code, nbits, extra;
        length_prefix(t, code, nbits, extra);
        put(table[kGreen + 256 + code]);
        put(extra | (nbits << 16));
        put(table[kDist + kLeftDistSymbol]);
    }
    return nb;
}

__global__ void __launch_bounds__(256) k_webp_bits(const uint32_t* __restrict__ sym, const uint16_t* __restrict__ tok,
                                                   int64_t n, const uint32_t* __restrict__ table,
                                                   uint32_t* __restrict__ bits) {
    __shared__ uint32_t tb[kWebpTreeSyms];
    for (int k = threadIdx.x; k < kWebpTreeSyms; k += blockDim.x) tb[k] = table[k];
    __syncthreads();
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        uint64_t v;
        const uint32_t t = tok[i];
        bits[i] = t ? token_fields(sym[i], t, tb, v) : 0u;
    }
}

// one thread: chunk c's offsets start at bases[c]; the last entry of each chunk's scan plus its own bits is its size
__global__ void k_webp_bases(const uint32_t* __restrict__ sym, const uint16_t* __restrict__ tok, int64_t n,
                             const uint32_t* __restrict__ table, const uint32_t* __restrict__ offsets,
                             uint64_t* __restrict__ bases, unsigned long long* __restrict__ total) {
    uint64_t acc = 0;
    for (int64_t c = 0; c * kScanChunk < n; ++c) {
        bases[c] = acc;
        const int64_t last = min(n, (c + 1) * kScanChunk) - 1;
        uint64_t v;
        acc += offsets[last] + (tok[last] ? token_fields(sym[last], tok[last], table, v) : 0u);
    }
    *total = acc;
}

__global__ void __launch_bounds__(256) k_webp_emit(const uint32_t* __restrict__ sym, const uint16_t* __restrict__ tok,
                                                   int64_t n, const uint32_t* __restrict__ table,
                                                   const uint32_t* __restrict__ offsets,
                                                   const uint64_t* __restrict__ bases, uint64_t bit_offset,
                                                   uint32_t* __restrict__ words, int64_t nwords) {
    __shared__ uint32_t tb[kWebpTreeSyms];
    for (int k = threadIdx.x; k < kWebpTreeSyms; k += blockDim.x) tb[k] = table[k];
    __syncthreads();
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const uint32_t t = tok[i];
        if (!t) continue;
        uint64_t v;
        const uint32_t nb = token_fields(sym[i], t, tb, v);
        if (!nb) continue;
        const uint64_t o = bit_offset + bases[i / kScanChunk] + offsets[i];
        const int64_t w = int64_t(o >> 5);
        const uint32_t sh = uint32_t(o & 31);
        const uint64_t rest = v >> (32 - sh);   // the bits past the first word (sh == 0: v >> 32)
        const uint32_t part[3] = {uint32_t(v << sh), uint32_t(rest), uint32_t(rest >> 32)};
        for (int k = 0; k < 3; ++k)
            if (part[k] && w + k < nwords) atomicOr(&words[w + k], part[k]);
    }
}

__global__ void k_webp_patch(uint32_t* __restrict__ words, int64_t nwords, const uint32_t* __restrict__ patches,
                             int64_t npatches) {
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < npatches;
         i += int64_t(gridDim.x) * blockDim.x) {
        const uint32_t w = patches[2 * i];
        if (w < nwords) atomicOr(&words[w], patches[2 * i + 1]);   // two header pieces can share a word
    }
}

struct Layout {
    int64_t n, tiles;
    uint32_t* sym[5];
    uint16_t* tok[5];
    uint32_t *scan, *starts, *scan_ws, *alpha_used;
    uint64_t* bases;
};

int64_t tiles_of(int64_t w, int64_t h) { return ((w + kTile - 1) / kTile) * ((h + kTile - 1) / kTile); }

bool carve(Carver& cv, int64_t width, int64_t height, Layout& L) {
    L.n = width * height;
    L.tiles = tiles_of(width, height);
    for (int k = 0; k < 5; ++k) L.sym[k] = cv.take<uint32_t>(k < 3 ? L.n : L.tiles);
    for (int k = 0; k < 5; ++k) L.tok[k] = cv.take<uint16_t>(k < 3 ? L.n : L.tiles);
    L.scan = cv.take<uint32_t>(L.n);
    L.starts = cv.take<uint32_t>(L.n);
    L.scan_ws = cv.take<uint32_t>(scan_workspace_bytes(L.n) / sizeof(uint32_t) + 1);
    L.bases = cv.take<uint64_t>((L.n + kScanChunk - 1) / kScanChunk);
    L.alpha_used = cv.take<uint32_t>(1);
    return cv.ok();
}

bool side_ok(int64_t width, int64_t height) {
    return width >= 1 && height >= 1 && width <= kWebpMaxSide && height <= kWebpMaxSide;
}

int grid_for(int64_t n) { return int(std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, int64_t(sm_count()) * 8))); }

int tokens_of(const uint32_t* sym, int64_t n, uint16_t* tok, uint32_t* hist, const Layout& L, cudaStream_t st) {
    const int g = grid_for(n);
    k_webp_breaks<<<g, 256, 0, st>>>(sym, n, L.scan);
    GSX_KERNEL_CHECK();
    int rc = exclusive_scan_u32_ws(L.scan, n, L.scan_ws, st);
    if (rc) return rc;
    k_webp_run_starts<<<g, 256, 0, st>>>(sym, n, L.scan, L.starts);
    GSX_KERNEL_CHECK();
    k_webp_tokens<<<g, 256, 0, st>>>(sym, n, L.scan, L.starts, tok, hist);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_webp_workspace_bytes(int64_t width, int64_t height) {
    if (!side_ok(width, height)) return 0;
    Carver cv(nullptr, 0);
    Layout L;
    carve(cv, width, height, L);
    return int64_t(cv.off) + 256;
}

int gsx_webp_analyze(const uint8_t* rgba, int64_t width, int64_t height, void* ws, int64_t ws_bytes, uint32_t* hist,
                     uint8_t* modes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_webp_analyze");
    GSX_REQUIRE(side_ok(width, height), GSX_ERR_ARG, "webp: width and height must be 1..16384 (got %lld x %lld)",
                (long long)width, (long long)height);
    GSX_REQUIRE(rgba && ws && hist, GSX_ERR_ARG, "webp_analyze: null pointer");
    Carver cv(ws, size_t(ws_bytes));
    Layout L;
    GSX_REQUIRE(carve(cv, width, height, L), GSX_ERR_WORKSPACE, "webp_analyze: workspace too small");
    GSX_CUDA_CHECK(cudaMemsetAsync(hist, 0, (5 * kWebpTreeSyms + 1) * sizeof(uint32_t), st));
    GSX_CUDA_CHECK(cudaMemsetAsync(L.alpha_used, 0, sizeof(uint32_t), st));
    k_webp_clean<<<grid_for(L.n), 256, 0, st>>>((const uchar4*)rgba, L.n, L.sym[0], L.alpha_used);
    GSX_KERNEL_CHECK();
    const int tiles_x = int((width + kTile - 1) / kTile);
    k_webp_predict<false><<<int(L.tiles), 256, 0, st>>>(L.sym[0], int(width), int(height), tiles_x, L.sym[1], L.sym[3],
                                                         modes);
    GSX_KERNEL_CHECK();
    k_webp_predict<true><<<int(L.tiles), 256, 0, st>>>(L.sym[0], int(width), int(height), tiles_x, L.sym[2], L.sym[4],
                                                        modes ? modes + L.tiles : nullptr);
    GSX_KERNEL_CHECK();
    for (int k = 0; k < 5; ++k) {
        int rc = tokens_of(L.sym[k], k < 3 ? L.n : L.tiles, L.tok[k], hist + k * kWebpTreeSyms, L, st);
        if (rc) return rc;
    }
    GSX_CUDA_CHECK(cudaMemcpyAsync(hist + 5 * kWebpTreeSyms, L.alpha_used, sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                                   st));
    return GSX_OK;
}

int gsx_webp_emit(int64_t width, int64_t height, int32_t image, const uint32_t* table, uint64_t bit_offset, void* ws,
                  int64_t ws_bytes, uint32_t* words, int64_t nwords, unsigned long long* total_bits, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_webp_emit");
    GSX_REQUIRE(side_ok(width, height), GSX_ERR_ARG, "webp: width and height must be 1..16384 (got %lld x %lld)",
                (long long)width, (long long)height);
    GSX_REQUIRE(image >= 0 && image < 5, GSX_ERR_ARG, "webp_emit: image must be 0..4 (got %d)", image);
    GSX_REQUIRE(table && ws && words && total_bits, GSX_ERR_ARG, "webp_emit: null pointer");
    Carver cv(ws, size_t(ws_bytes));
    Layout L;
    GSX_REQUIRE(carve(cv, width, height, L), GSX_ERR_WORKSPACE, "webp_emit: workspace too small");
    const int64_t n = image < 3 ? L.n : L.tiles;
    const uint32_t* sym = L.sym[image];
    const uint16_t* tok = L.tok[image];
    const int g = grid_for(n);
    k_webp_bits<<<g, 256, 0, st>>>(sym, tok, n, table, L.scan);
    GSX_KERNEL_CHECK();
    for (int64_t c = 0; c < n; c += kScanChunk) {
        int rc = exclusive_scan_u32_ws(L.scan + c, std::min(kScanChunk, n - c), L.scan_ws, st);
        if (rc) return rc;
    }
    k_webp_bases<<<1, 1, 0, st>>>(sym, tok, n, table, L.scan, L.bases, total_bits);
    GSX_KERNEL_CHECK();
    k_webp_emit<<<g, 256, 0, st>>>(sym, tok, n, table, L.scan, L.bases, bit_offset, words, nwords);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_webp_patch(uint32_t* words, int64_t nwords, const uint32_t* patches, int64_t npatches, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(words && (patches || npatches == 0) && npatches >= 0, GSX_ERR_ARG, "webp_patch: bad arguments");
    if (npatches == 0) return GSX_OK;
    k_webp_patch<<<grid_for(npatches), 256, 0, st>>>(words, nwords, patches, npatches);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

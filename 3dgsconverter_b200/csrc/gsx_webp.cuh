#pragma once
#include "gsx_common.cuh"
namespace gsx {
// Lossless WebP (VP8L, RFC 9649) encoder over a device RGBA image; the host side (Huffman codes, headers, candidate
// choice) is gsx/webp.py.  Five entropy-coded images live in the workspace: 0 = the pixels (candidate 0),
// 1 = predictor residuals, 2 = subtract-green + predictor residuals, 3 / 4 = the predictor sub-images of 1 / 2.
constexpr int kWebpMaxSide = 16384;
constexpr int kWebpTreeSyms = 280 + 256 + 256 + 256 + 40;   // green + 24 lengths, red, blue, alpha, distance
int64_t webp_workspace_bytes(int64_t width, int64_t height);
int webp_analyze(const uint8_t* rgba, int64_t width, int64_t height, void* ws, int64_t ws_bytes, uint32_t* hist,
                 uint8_t* modes, cudaStream_t st);
int webp_emit(int64_t width, int64_t height, int image, const uint32_t* table, uint64_t bit_offset, void* ws,
              int64_t ws_bytes, uint32_t* words, int64_t nwords, unsigned long long* total_bits, cudaStream_t st);
int webp_patch(uint32_t* words, int64_t nwords, const uint32_t* patches, int64_t npatches, cudaStream_t st);
}

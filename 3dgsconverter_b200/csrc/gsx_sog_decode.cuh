#pragma once
#include "gsx_common.cuh"
namespace gsx {
// bits of the error word: the index the reference reader rejects with IndexError
constexpr int32_t kSogErrScaleCodebook = 1, kSogErrSh0Codebook = 2, kSogErrShCodebook = 4, kSogErrLabel = 8;

struct SogTextures {   // RGBA pixels, 4-byte aligned; labels null without shN
    const uint8_t *means_l, *means_u, *quats, *scales, *sh0, *labels;
};

int sog_decode_palette(const uint8_t* centroids, int64_t P, int coeffs, const float* codebook, int ncb, float* palette,
                       int32_t* err, cudaStream_t st);
int sog_decode(const SogTextures& tx, int64_t n, const float* pos_tables, const float* tables, int nscb, int nccb,
               const float* palette, int64_t P, int coeffs, uint8_t* rows, int32_t* err, cudaStream_t st);
}  // namespace gsx

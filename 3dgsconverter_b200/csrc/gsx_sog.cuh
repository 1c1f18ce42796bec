#pragma once
#include "gsx_common.cuh"
namespace gsx {
int64_t lexsort_workspace_bytes(int64_t n);
int lexsort_zyx(const float* xyz, int64_t n, int32_t* order_out, void* ws, int64_t ws_bytes, cudaStream_t st);
int quantize_to_codebook(const float* vals, int64_t n, const float* codebook_host, int m, uint8_t* labels, void* ws,
                         int64_t ws_bytes, cudaStream_t st);
int sog_means_minmax(const float* rows, int64_t n, int F, const int32_t* cols3_host, float* ws, int64_t ws_bytes,
                     float* minmax, cudaStream_t st);
int sog_means(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols3_host,
              const float* minmax, int64_t pixels, uint8_t* means_l, uint8_t* means_u, cudaStream_t st);
int sog_quats(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols4_host, int64_t pixels,
              uint8_t* quats, cudaStream_t st);
int sog_gather_values(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols_host, int ncols,
                      const int64_t* sel, int64_t m, float* out, cudaStream_t st);
int sog_scales_sh0(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols7_host,
                   const float* scale_cb, int m_scale, const float* color_cb, int m_color, int64_t pixels,
                   uint8_t* scales, uint8_t* sh0, cudaStream_t st);
int sog_sh_gather(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols_host, int ncols,
                  float* out, unsigned long long* nonzero, cudaStream_t st);
int sog_labels(const int32_t* labels, int64_t n, int64_t chunk_size, int nchunks, const int32_t* offsets_host,
               const int32_t* passthrough_host, int64_t pixels, uint8_t* out, cudaStream_t st);
int sog_centroids(const float* palette, int64_t P, int coeffs, const float* cb, int m, int64_t pixels, uint8_t* out,
                  cudaStream_t st);
}

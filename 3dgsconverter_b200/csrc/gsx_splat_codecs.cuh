#pragma once
#include "gsx_common.cuh"
namespace gsx {
int codec_sh_mask(const float* rows, int64_t n, int F, const int32_t* sh_cols, int nsh, unsigned long long* mask,
                  cudaStream_t st);
int ksplat_record_bytes(int level, int sh_count);
int ksplat_centres(const float* lo, const float* hi, int64_t nbucket, float* centres, cudaStream_t st);
int ksplat_pack(const float* rows, int64_t n, int F, const int32_t* cols14, const int32_t* sh_cols, int sh_count,
                int level, int64_t bucket_size, float sf_inv, const float* centres, uint8_t* out, cudaStream_t st);
int spz_pack(const float* rows, int64_t n, int F, const int32_t* cols14, const int32_t* sh_cols, int sh_dim,
             uint8_t* body, cudaStream_t st);
int splat_sort_keys(const float* rows, int64_t n, int F, const int32_t* cols4, uint64_t* keys, int32_t* vals,
                    cudaStream_t st);
int splat_pack(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols14, uint8_t* out,
               cudaStream_t st);
int records_from_bytes(const uint8_t* src, int64_t n, int64_t row_bytes, const int32_t* offsets, int nf, float* out,
                       cudaStream_t st);
}

#pragma once
#include "gsx_common.cuh"
namespace gsx {
int splat_decode(const uint8_t* data, int64_t n, const float* tables, uint8_t* rows, cudaStream_t st);
int ksplat_decode_section(const uint8_t* rec, int64_t n, int level, int sh_count, float sr, float sf,
                          const uint8_t* centres, int64_t ncentres, int64_t full_buckets, int64_t bucket_size,
                          const int64_t* partial_end, int32_t npartial, const float* tables, int32_t row_bytes,
                          uint8_t* rows, cudaStream_t st);
int spz_decode(const uint8_t* body, int64_t n, int version, int sh_dim, int frac_bits, const float* tables,
               int32_t row_bytes, uint8_t* rows, cudaStream_t st);
int cply_decode(const uint8_t* chunk, int64_t nchunk, int32_t chunk_row, const int32_t* chunk_offs,
                const uint8_t* vertex, int64_t n, int32_t vertex_row, const int32_t* vertex_offs, const uint8_t* sh,
                int32_t sh_row, const int32_t* sh_offs, int32_t nsh, const float* tables, uint8_t* rows,
                cudaStream_t st);
}

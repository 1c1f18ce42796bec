#pragma once
#include "gsx_common.cuh"
namespace gsx {
int cply_pack(const float* rows, int64_t n, int F, const int32_t* order, const int32_t* cols14_host,
              const int32_t* rest_cols_host, int n_rest, const float* lo_pos_dc, const float* hi_pos_dc,
              const float* lo_scale, const float* hi_scale, float* chunk_out, uint32_t* vertex_out, uint8_t* sh_out,
              unsigned long long* rest_nonzero_out, cudaStream_t st);
int cply_narrow_sh(const uint8_t* sh, int64_t n, int width, int keep, uint8_t* out, cudaStream_t st);
}

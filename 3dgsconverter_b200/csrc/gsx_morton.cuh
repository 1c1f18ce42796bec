#pragma once
#include "gsx_common.cuh"
namespace gsx {
int64_t morton_workspace_bytes(int64_t n);
int morton_order(const float* xyz, int64_t n, int32_t* order, int limit, int* levels_out, void* ws, int64_t ws_bytes,
                 cudaStream_t st);
int chunk_minmax(const float* rows, int64_t n, int F, const int32_t* order, int chunk, const int* cols_host, int ncol,
                 float clip_lo, float clip_hi, float* lo_out, float* hi_out, void* ws, int64_t ws_bytes, cudaStream_t st);
}

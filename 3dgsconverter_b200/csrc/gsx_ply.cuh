#pragma once
#include "gsx_common.cuh"
namespace gsx {
int ply_transcode(const uint8_t* src, int64_t n, int32_t src_row, uint8_t* dst, int32_t dst_row, const int32_t* fields,
                  int32_t nf, cudaStream_t st);
}

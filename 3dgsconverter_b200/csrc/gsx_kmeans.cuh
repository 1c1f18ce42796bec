#pragma once
#include "gsx_common.cuh"
#include "../../include/gsx.h"

namespace gsx {

struct KmProb {
    long long row0;      // first row of the problem in X
    long long rows;      // number of rows
    long long tc_tile0;  // first 128-row tile of the problem (tensor-core assign)
    int tile0;           // first assign tile of the problem (CUDA-core assign)
    int sub0;            // first label sub-tile (kSubTile points, one warp each) of the problem
};

// gsx_kmeans_tc.cu
bool kmeans_tc_supported(int K, int D);
int kmeans_assign_tc(const float* X, long long x_floats, const float* C, int* labels, const KmProb* probs_dev, int nprob,
                     int K, int D, long long tiles, int mode, float* dump, unsigned long long* stats,
                     int* err_flag_dev, cudaStream_t st);
}

// gsx_sor.cuh -- internal declarations shared by the SOR translation units.
#pragma once
#include "gsx_common.cuh"

#define GSX_HASH_MODE_I32WRAP 0
#define GSX_HASH_MODE_I64 1

namespace gsx {

struct SorWs {
    int64_t n;
    uint64_t *keys0, *keys1, *keys_sorted;
    float4* spos;   // hash-sorted positions, w = original index
    int2* tab_se;         // per bucket {start, end} in sorted order; {0,0} = empty (cell_start == -1)
    float4* tab_box;      // per bucket {lo.xyz,-},{hi.xyz,-}: exact box of its points (occupied buckets only)
    uint32_t* startbits;  // one bit per sorted position: starts a bucket
    uint32_t* cellbits;   // one bit per sorted position: other grid cell than the position before
    uint32_t* bigbits;    // one bit per sorted position: starts a bucket longer than kSmallBucket (distributed stage C)
    float4* caabb;  // 2 float4 per 32-point chunk: {lo.x,lo.y,lo.z,hi.x},{hi.y,hi.z,-,-}
    float4* saabb;  // same per 1024-point super
    float* partial;
    float* minmax;
    uint32_t* startlist;  // positions of the bucket starts, n/8 + 1024 entries (distributed stage C)
    unsigned int* counters;
    unsigned long long* stats;
    float* meanstd;
    char* sort_ws;
    size_t sort_ws_bytes;
    char* ms_ws;
    size_t ms_bytes;
    size_t total, grid_total;  // whole workspace / the grid part only (a prefix)
    bool ok, grid_ok;
};

SorWs sor_carve(void* ws, int64_t ws_bytes, int64_t n, size_t sort_ws_bytes);
size_t sor_sort_ws_bytes(int64_t n);
int sor_minmax(const float* xyz, int64_t n, float* minmax_dev, float* partial, cudaStream_t st);
int sor_build(const float* xyz, int64_t n, const float* bmin, float cell, SorWs& w, cudaStream_t st);
int sor_mean_dists(SorWs& w, int64_t q_begin, int64_t q_end, int q_stride, int q_phase, int k, int hash_mode,
                   const float* bmin, float cell,
                   float* final_means, unsigned long long* stats, cudaStream_t st);

int sor_dist_local_run(const float* xyz, int64_t n_local, int64_t idx_base, int64_t n_global, int world,
                       const float* bmin, float cell, float4* pos4_out, long long* cuts_dev, SorWs& w,
                       cudaStream_t st);
int sor_dist_merge(const float4* pos4_in, int64_t m, int64_t n_global, int64_t bucket_lo, int64_t bucket_hi,
                   const float* bmin, float cell, float4* pos4_out, uint8_t* flags_out, SorWs& w, cudaStream_t st);
int sor_build_from_sorted(const float4* spos_in, const uint8_t* flags, int64_t n, const float* bmin, float cell, SorWs& w,
                          cudaStream_t st);

const char* sor_build_info();

size_t mean_std_ws_bytes(int64_t n);
int mean_std_f32(const float* a, int64_t n, float* out_dev, void* ws, size_t ws_bytes, cudaStream_t st);
int threshold_mask(const float* a, int64_t n, const float* meanstd_dev, float tf, uint8_t* mask, cudaStream_t st);

}  // namespace gsx

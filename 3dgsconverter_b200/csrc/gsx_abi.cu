// gsx_abi.cu -- library-wide state of libgsx.so (error buffer, launch counter, device queries) and the host-buffer
// convenience entry points, which own device memory for the caller.  Every other entry point of include/gsx.h is
// defined in the module that implements it.
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_hostcopy.cuh"
#include "gsx_sor.cuh"

#include <atomic>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

namespace gsx {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    static int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        cached = v;
        cached_dev = dev;
    }
    return cached;
}

// keep freed blocks in the default memory pool across calls: without this the pool is trimmed at every
// stream synchronisation and each *_host call pays ~20 ms of cudaMalloc for its workspace again
static void keep_pool_warm() {
    static thread_local int done_for = -1;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev == done_for) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long thr = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    done_for = dev;
}

struct DevBuf {  // stream-ordered device allocation for the *_host entry points
    void* p = nullptr;
    cudaStream_t st;
    explicit DevBuf(cudaStream_t s) : st(s) { keep_pool_warm(); }
    int alloc(size_t bytes) {
        cudaError_t e = cudaMallocAsync(&p, bytes ? bytes : 1, st);
        if (e != cudaSuccess) {
            set_error("cudaMallocAsync(%zu) -> %s", bytes, cudaGetErrorString(e));
            p = nullptr;
            return GSX_ERR_CUDA;
        }
        return GSX_OK;
    }
    ~DevBuf() {
        if (p) cudaFreeAsync(p, st);
    }
};

}  // namespace gsx

using namespace gsx;

extern "C" {

const char* gsx_last_error(void) { return g_err; }
int gsx_version(void) { return 100; }
const char* gsx_build_info(void) { return sor_build_info(); }
long long gsx_kernel_launches(void) { return g_launches.load(); }
int gsx_device_sm_count(void) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return GSX_ERR_CUDA;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return GSX_ERR_CUDA;
    return v;
}

/* ------------------------------------------------------------------ whole filters and K-Means on HOST buffers */

int gsx_sor_filter_host(const float* xyz_host, int64_t n, int32_t k, float threshold_factor, int32_t hash_mode,
                        uint8_t* mask_host, float* means_host) {
    GSX_REQUIRE(n >= 1 && n < 2147483584ll, GSX_ERR_ARG, "sor: n=%lld out of range", (long long)n);
    cudaStream_t st = 0;
    int64_t wsb = gsx_sor_workspace_bytes(n);
    DevBuf xyz(st), ws(st), mask(st), means(st);
    int rc;
    if ((rc = xyz.alloc((size_t)n * 12))) return rc;
    if ((rc = ws.alloc((size_t)wsb))) return rc;
    if ((rc = mask.alloc((size_t)n))) return rc;
    if ((rc = means.alloc((size_t)n * 4))) return rc;
    if ((rc = copy_h2d(xyz.p, xyz_host, (size_t)n * 12, st))) return rc;
    if ((rc = gsx_sor_filter_device((const float*)xyz.p, n, k, threshold_factor, hash_mode, (uint8_t*)mask.p,
                                    (float*)means.p, ws.p, wsb, st)))
        return rc;
    // the kernels are queued: make the (usually never touched) destination pages resident while the GPU works
    prefault_host(mask_host, (size_t)n);
    if (means_host) prefault_host(means_host, (size_t)n * 4);
    if ((rc = copy_d2h(mask_host, mask.p, (size_t)n, st))) return rc;
    if (means_host && (rc = copy_d2h(means_host, means.p, (size_t)n * 4, st))) return rc;
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    return GSX_OK;
}

int gsx_sor_ckdtree_filter_host(const float* xyz_host, int64_t n, int32_t k, float threshold_factor, uint8_t* mask_host,
                                float* means_host) {
    GSX_REQUIRE(n >= 1 && n < 2147483584ll, GSX_ERR_ARG, "sor: n=%lld out of range", (long long)n);
    cudaStream_t st = 0;
    int64_t wsb = gsx_knn_exact_workspace_bytes(n);
    int64_t msb = gsx_mean_std_workspace_bytes(n);
    DevBuf xyz(st), ws(st), mask(st), means(st), ms(st), msws(st);
    int rc;
    if ((rc = xyz.alloc((size_t)n * 12))) return rc;
    if ((rc = ws.alloc((size_t)wsb))) return rc;
    if ((rc = mask.alloc((size_t)n))) return rc;
    if ((rc = means.alloc((size_t)n * 4))) return rc;
    if ((rc = ms.alloc(64))) return rc;
    if ((rc = msws.alloc((size_t)msb))) return rc;
    if ((rc = copy_h2d(xyz.p, xyz_host, (size_t)n * 12, st))) return rc;
    if ((rc = gsx_knn_exact_mean_dists((const float*)xyz.p, n, k, (float*)means.p, ws.p, wsb, st))) return rc;
    if ((rc = gsx_mean_std_f32((const float*)means.p, n, (float*)ms.p, msws.p, msb, st))) return rc;
    if ((rc = gsx_threshold_mask((const float*)means.p, n, (const float*)ms.p, threshold_factor, (uint8_t*)mask.p,
                                 st)))
        return rc;
    // the kernels are queued: make the (usually never touched) destination pages resident while the GPU works
    prefault_host(mask_host, (size_t)n);
    if (means_host) prefault_host(means_host, (size_t)n * 4);
    if ((rc = copy_d2h(mask_host, mask.p, (size_t)n, st))) return rc;
    if (means_host && (rc = copy_d2h(means_host, means.p, (size_t)n * 4, st))) return rc;
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    return GSX_OK;
}

int gsx_kmeans_host(const float* X_host, int64_t n, int32_t K, int32_t D, int32_t max_iter, float* C_host_inout,
                    int32_t* labels_host, int32_t assign_mode) {
    const int64_t off[2] = {0, n};
    return gsx_kmeans_host_batched(X_host, off, 1, K, D, max_iter, C_host_inout, labels_host, assign_mode);
}

/* SOG shN schedule in one call on HOST buffers: nprob problems stored back to back in X_host (rows row_off[p] ..
 * row_off[p+1]), each with K centroids; C_host_inout [nprob*K*D] holds the init on entry, the centroids on return. */
int gsx_kmeans_host_batched(const float* X_host, const int64_t* row_off_host, int32_t nprob, int32_t K, int32_t D,
                            int32_t max_iter, float* C_host_inout, int32_t* labels_host, int32_t assign_mode) {
    GSX_REQUIRE(nprob >= 1 && K >= 1 && D >= 1, GSX_ERR_ARG, "kmeans: bad shape");
    GSX_REQUIRE(row_off_host[0] == 0, GSX_ERR_ARG, "kmeans: row_off[0] must be 0");
    const int64_t n = row_off_host[nprob];
    GSX_REQUIRE(n >= 1, GSX_ERR_ARG, "kmeans: no rows");
    cudaStream_t st = 0;
    DevBuf X(st), C(st), L(st), cnt(st), ws(st);
    int rc;
    int64_t wsb = gsx_kmeans_workspace_bytes(n, nprob, K, D);
    if ((rc = X.alloc((size_t)n * D * 4))) return rc;
    if ((rc = C.alloc((size_t)nprob * K * D * 4))) return rc;
    if ((rc = L.alloc((size_t)n * 4))) return rc;
    if ((rc = cnt.alloc((size_t)nprob * K * 4))) return rc;
    if ((rc = ws.alloc((size_t)wsb))) return rc;
    if ((rc = copy_h2d(X.p, X_host, (size_t)n * D * 4, st))) return rc;
    GSX_CUDA_CHECK(cudaMemcpyAsync(C.p, C_host_inout, (size_t)nprob * K * D * 4, cudaMemcpyHostToDevice, st));
    GSX_CUDA_CHECK(cudaMemsetAsync(L.p, 0, (size_t)n * 4, st));
    if ((rc = gsx_kmeans_lloyd_device((const float*)X.p, row_off_host, nprob, K, D, max_iter, (float*)C.p, (int*)L.p,
                                      (int*)cnt.p, ws.p, wsb, assign_mode, nullptr, st)))
        return rc;
    prefault_host(labels_host, (size_t)n * 4);   // while the Lloyd iterations run
    GSX_CUDA_CHECK(cudaMemcpyAsync(C_host_inout, C.p, (size_t)nprob * K * D * 4, cudaMemcpyDeviceToHost, st));
    if ((rc = copy_d2h(labels_host, L.p, (size_t)n * 4, st))) return rc;
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    return GSX_OK;
}

/* free / total device memory of the current device (sizing decisions of the host-buffer entry points) */
int gsx_device_memory(int64_t* free_bytes, int64_t* total_bytes) {
    size_t f = 0, t = 0;
    GSX_CUDA_CHECK(cudaMemGetInfo(&f, &t));
    if (free_bytes) *free_bytes = (int64_t)f;
    if (total_bytes) *total_bytes = (int64_t)t;
    return GSX_OK;
}

}  // extern "C"

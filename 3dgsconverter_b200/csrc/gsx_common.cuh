// gsx_common.cuh -- shared helpers for the gsx sm_90a kernels.
//
// Arithmetic contract (SURVEY.md Appendix A): every float operation that feeds a
// keep-mask is IEEE binary32 round-to-nearest with NO fma contraction.  The whole
// library is compiled with --fmad=false and the parity-critical expressions use the
// explicit __f*_rn intrinsics as well, so the contract survives a flag change.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <nvtx3/nvToolsExt.h>   // header-only (dlopen of the injection library at run time; no link dependency)

#define GSX_OK 0
#define GSX_ERR_CUDA -1
#define GSX_ERR_ARG -2
#define GSX_ERR_WORKSPACE -3
#define GSX_ERR_UNSUPPORTED -4

namespace gsx {

void set_error(const char* fmt, ...);
void count_launch();

#define GSX_CUDA_CHECK(expr)                                                                  \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            gsx::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return GSX_ERR_CUDA;                                                              \
        }                                                                                     \
    } while (0)

// follows every launch of one of OUR kernels: counts it (gsx_kernel_launches) and checks the launch
#define GSX_KERNEL_CHECK()                    \
    do {                                      \
        gsx::count_launch();                  \
        GSX_CUDA_CHECK(cudaGetLastError());   \
    } while (0)

#define GSX_REQUIRE(cond, code, ...)   \
    do {                               \
        if (!(cond)) {                 \
            gsx::set_error(__VA_ARGS__); \
            return (code);             \
        }                              \
    } while (0)

// NVTX range of a host-side stage (visible in nsys / ncu --nvtx): one per C-ABI stage, RAII
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
#define GSX_NVTX(name) gsx::NvtxRange _gsx_nvtx_range(name)

// Device properties cached per process (queried on first use for the current device).
int sm_count();

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace blob.
struct Carver {
    char* base;
    size_t off;
    size_t cap;
    __host__ Carver(void* p, size_t bytes) : base((char*)p), off(0), cap(bytes) {}
    template <typename T>
    __host__ T* take(size_t count) {
        off = align_up(off, 256);
        T* r = (T*)(base + off);
        off += count * sizeof(T);
        return r;
    }
    __host__ bool ok() const { return off <= cap; }
};

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// Lemire fastmod: a % d for 32-bit a, d with M = UINT64_MAX / d + 1.
__device__ __forceinline__ uint32_t fastmod_u32(uint32_t a, uint64_t M, uint32_t d) {
    uint64_t low = M * (uint64_t)a;
    return (uint32_t)__umul64hi(low, (uint64_t)d);
}

// streaming 128-bit load that does not allocate in L1 (read-once data)
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

}  // namespace gsx

// gsx_hostcopy.cu -- host <-> device copies for the *_host entry points when the caller's buffer is PAGEABLE.
//
// The reference's call sites hand libgsx ordinary NumPy arrays (np.column_stack at data_processor.py:139, the
// shN block at sog.py:536-549).  cudaMemcpyAsync from pageable memory is staged by the driver through one
// internal pinned buffer on ONE CPU thread, so the PCIe link idles most of the time and the upload can
// cost more than the whole filter.
//
// Here T host threads each own two pinned chunks and one copy stream: a thread memcpy()s its next chunk of
// the user's buffer into a free pinned chunk and enqueues the DMA itself, so T memcpys and the DMAs of earlier
// chunks overlap.  D2H is the mirror image (DMA into a pinned chunk, memcpy out while the next DMA runs).
// A buffer that is already pinned / registered / managed goes straight to cudaMemcpyAsync.
#include "gsx_hostcopy.cuh"

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <thread>
#include <unistd.h>
#include <vector>

namespace gsx {

namespace {

constexpr size_t kStagedMin = 8u << 20;      // below this the plain path is as fast
constexpr int kMaxThreads = 16;
size_t kChunk = 4u << 20;                    // pinned chunk (GSX_COPY_CHUNK_KB, default 4 MiB; smaller chunks
                                             // measured slower on large uploads)

// The helper threads are created once and parked on a condition variable: creating 7 threads and giving each a CUDA
// context binding cost more than the copy itself for a 120 MB cloud.  Leaked on purpose (no static destruction order
// to get wrong at process exit; the threads only ever wait or copy).
struct Workers {
    std::mutex m;
    std::condition_variable cv_job, cv_done;
    std::function<cudaError_t(int)> job;
    unsigned long long gen = 0;
    int pending = 0, T = 0, dev = -1;
    std::atomic<int> err{0};
    void start(int threads) {
        T = threads;
        for (int t = 1; t < T; ++t)
            std::thread([this, t] {
                unsigned long long seen = 0;
                int bound = -1;
                for (;;) {
                    std::unique_lock<std::mutex> lk(m);
                    cv_job.wait(lk, [&] { return gen != seen; });
                    seen = gen;
                    const int d = dev;
                    lk.unlock();
                    cudaError_t e = cudaSuccess;
                    if (d >= 0 && d != bound) {
                        e = cudaSetDevice(d);
                        bound = d;
                    }
                    if (e == cudaSuccess) e = job(t);
                    if (e != cudaSuccess) {
                        int expect = 0;
                        err.compare_exchange_strong(expect, (int)e);
                    }
                    lk.lock();
                    if (--pending == 0) cv_done.notify_one();
                }
            }).detach();
    }
    // run body(t) for t = 0 .. T-1 (t = 0 on the calling thread); returns the first error
    cudaError_t run(int device, std::function<cudaError_t(int)> body) {
        {
            std::lock_guard<std::mutex> lk(m);
            job = body;
            dev = device;
            err.store(0);
            pending = T - 1;
            ++gen;
        }
        cv_job.notify_all();
        cudaError_t e0 = body(0);
        std::unique_lock<std::mutex> lk(m);
        cv_done.wait(lk, [&] { return pending == 0; });
        return e0 != cudaSuccess ? e0 : (cudaError_t)err.load();
    }
};
Workers* g_workers = nullptr;

struct Pool {
    std::mutex mu;                 // one staged copy at a time (the pinned chunks are shared state)
    int dev = -1;
    int T = 0;
    char* pinned = nullptr;        // 2 * T chunks
    cudaStream_t streams[kMaxThreads] = {};
    cudaEvent_t ev[2 * kMaxThreads] = {};
    cudaEvent_t ev_start = nullptr;
    bool failed = false;           // creation failed once: stay on the plain path
};
Pool g_pool;

int env_int(const char* name, int dflt) {
    const char* s = getenv(name);
    return s && *s ? atoi(s) : dflt;
}

// (re)create the pool for the current device; false -> use the plain path
bool pool_ready(Pool& p, int dev) {
    if (p.failed) return false;
    if (p.pinned && p.dev == dev) return true;
    if (p.pinned && p.dev != dev) {   // another device became current: streams / events belong to a device
        int cur = dev;
        cudaSetDevice(p.dev);
        for (int t = 0; t < p.T; ++t) cudaStreamDestroy(p.streams[t]);
        for (int i = 0; i < 2 * p.T; ++i) cudaEventDestroy(p.ev[i]);
        cudaEventDestroy(p.ev_start);
        cudaSetDevice(cur);
        p.dev = -1;
    }
    if (!p.pinned) {
        unsigned hw = std::thread::hardware_concurrency();
        int T = env_int("GSX_COPY_THREADS", hw >= 16 ? 8 : (hw >= 4 ? (int)hw / 2 : 1));
        p.T = std::max(1, std::min(T, kMaxThreads));
        kChunk = (size_t)std::max(64, std::min(env_int("GSX_COPY_CHUNK_KB", 4096), 16384)) << 10;
        if (cudaHostAlloc((void**)&p.pinned, 2 * (size_t)p.T * kChunk, cudaHostAllocPortable) != cudaSuccess) {
            cudaGetLastError();
            p.pinned = nullptr;
            p.failed = true;
            return false;
        }
    }
    bool ok = true;
    for (int t = 0; t < p.T && ok; ++t) ok = cudaStreamCreateWithFlags(&p.streams[t], cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; i < 2 * p.T && ok; ++i) ok = cudaEventCreateWithFlags(&p.ev[i], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&p.ev_start, cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        p.failed = true;
        return false;
    }
    if (!g_workers) {
        g_workers = new Workers();
        g_workers->start(p.T);
    }
    p.dev = dev;
    return true;
}

// pageable (unregistered) host memory?  Anything the driver already knows (pinned, registered, managed) and any
// failure to tell take the plain path.
bool is_pageable(const void* host) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, host) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeUnregistered;
}

bool staged_enabled() {
    static int v = -1;
    if (v < 0) v = env_int("GSX_STAGED_COPY", 1) != 0;
    return v != 0;
}

template <typename F>
cudaError_t run_workers(Pool& p, F&& body) {
    return g_workers->run(p.dev, std::function<cudaError_t(int)>(body));
}

}  // namespace

int copy_h2d(void* dst_dev, const void* src_host, size_t bytes, cudaStream_t st) {
    if (bytes == 0) return GSX_OK;
    int dev = 0;
    GSX_CUDA_CHECK(cudaGetDevice(&dev));
    if (bytes < kStagedMin || !staged_enabled() || !is_pageable(src_host)) {
        GSX_CUDA_CHECK(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, st));
        return GSX_OK;
    }
    Pool& p = g_pool;
    std::lock_guard<std::mutex> lock(p.mu);
    if (!pool_ready(p, dev)) {
        GSX_CUDA_CHECK(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, st));
        return GSX_OK;
    }
    GSX_NVTX("gsx_copy_h2d_staged");
    // dst may be a stream-ordered allocation of `st`: the copy streams start after everything queued on st so far
    GSX_CUDA_CHECK(cudaEventRecord(p.ev_start, st));
    const size_t nchunks = (bytes + kChunk - 1) / kChunk;
    const char* src = (const char*)src_host;
    char* dst = (char*)dst_dev;
    cudaError_t e = run_workers(p, [&](int t) -> cudaError_t {
        cudaError_t r = cudaStreamWaitEvent(p.streams[t], p.ev_start, 0);
        if (r != cudaSuccess) return r;
        int flip = 0;
        for (size_t c = (size_t)t; c < nchunks; c += (size_t)p.T, flip ^= 1) {
            const int slot = 2 * t + flip;
            char* stage = p.pinned + (size_t)slot * kChunk;
            if ((r = cudaEventSynchronize(p.ev[slot])) != cudaSuccess) return r;   // the chunk's previous DMA has drained
            const size_t off = c * kChunk, len = std::min(kChunk, bytes - off);
            memcpy(stage, src + off, len);
            if ((r = cudaMemcpyAsync(dst + off, stage, len, cudaMemcpyHostToDevice, p.streams[t])) != cudaSuccess) return r;
            if ((r = cudaEventRecord(p.ev[slot], p.streams[t])) != cudaSuccess) return r;
        }
        return cudaSuccess;
    });
    if (e != cudaSuccess) {
        set_error("staged H2D copy of %zu bytes -> %s", bytes, cudaGetErrorString(e));
        return GSX_ERR_CUDA;
    }
    // st continues once every chunk has landed (the last event of a stream covers its earlier copies)
    for (int i = 0; i < 2 * p.T; ++i) GSX_CUDA_CHECK(cudaStreamWaitEvent(st, p.ev[i], 0));
    return GSX_OK;
}

// Make the pages of a (typically fresh, never touched) host destination resident BEFORE the download needs them: a
// first touch of a 4 KiB page costs a page fault, which slows a staged D2H into np.empty far below a copy into
// touched memory, and the caller has nothing else to do while the GPU computes.  Content is preserved.
int prefault_host(void* dst_host, size_t bytes) {
    if (bytes < (1u << 20) || !staged_enabled()) return GSX_OK;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || !is_pageable(dst_host)) return GSX_OK;
    Pool& p = g_pool;
    std::lock_guard<std::mutex> lock(p.mu);
    if (!pool_ready(p, dev)) return GSX_OK;
    const size_t page = (size_t)sysconf(_SC_PAGESIZE);
    char* base = (char*)dst_host;
    char* lo = (char*)(((uintptr_t)base + page - 1) / page * page);
    char* hi = (char*)(((uintptr_t)base + bytes) / page * page);
    if (hi <= lo) return GSX_OK;
    const size_t npages = (size_t)(hi - lo) / page;
    run_workers(p, [&](int t) -> cudaError_t {
        const size_t a = npages * (size_t)t / (size_t)p.T, b = npages * (size_t)(t + 1) / (size_t)p.T;
        if (b <= a) return cudaSuccess;
#ifdef MADV_POPULATE_WRITE
        if (madvise(lo + a * page, (b - a) * page, MADV_POPULATE_WRITE) == 0) return cudaSuccess;
#endif
        for (size_t i = a; i < b; ++i) {   // read-modify-write of one byte: a write fault that changes nothing
            volatile char* q = (volatile char*)(lo + i * page);
            *q = *q;
        }
        return cudaSuccess;
    });
    return GSX_OK;
}

int copy_d2h(void* dst_host, const void* src_dev, size_t bytes, cudaStream_t st) {
    if (bytes == 0) return GSX_OK;
    int dev = 0;
    GSX_CUDA_CHECK(cudaGetDevice(&dev));
    if (bytes < kStagedMin || !staged_enabled() || !is_pageable(dst_host)) {
        GSX_CUDA_CHECK(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, st));
        GSX_CUDA_CHECK(cudaStreamSynchronize(st));
        return GSX_OK;
    }
    Pool& p = g_pool;
    std::lock_guard<std::mutex> lock(p.mu);
    if (!pool_ready(p, dev)) {
        GSX_CUDA_CHECK(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, st));
        GSX_CUDA_CHECK(cudaStreamSynchronize(st));
        return GSX_OK;
    }
    GSX_NVTX("gsx_copy_d2h_staged");
    GSX_CUDA_CHECK(cudaEventRecord(p.ev_start, st));   // the producer of src_dev
    const size_t nchunks = (bytes + kChunk - 1) / kChunk;
    const char* src = (const char*)src_dev;
    char* dst = (char*)dst_host;
    cudaError_t e = run_workers(p, [&](int t) -> cudaError_t {
        cudaError_t r = cudaStreamWaitEvent(p.streams[t], p.ev_start, 0);
        if (r != cudaSuccess) return r;
        int flip = 0;
        long long prev = -1;      // chunk whose DMA is in flight in slot 2t + (flip ^ 1)
        for (size_t c = (size_t)t; c < nchunks; c += (size_t)p.T, flip ^= 1) {
            const int slot = 2 * t + flip;
            const size_t off = c * kChunk, len = std::min(kChunk, bytes - off);
            if ((r = cudaEventSynchronize(p.ev[slot])) != cudaSuccess) return r;   // left over from an earlier call
            if ((r = cudaMemcpyAsync(p.pinned + (size_t)slot * kChunk, src + off, len, cudaMemcpyDeviceToHost,
                                     p.streams[t])) != cudaSuccess) return r;
            if ((r = cudaEventRecord(p.ev[slot], p.streams[t])) != cudaSuccess) return r;
            if (prev >= 0) {       // while that DMA runs, hand the previous chunk to the caller
                const int pslot = 2 * t + (flip ^ 1);
                const size_t poff = (size_t)prev * kChunk, plen = std::min(kChunk, bytes - poff);
                if ((r = cudaEventSynchronize(p.ev[pslot])) != cudaSuccess) return r;
                memcpy(dst + poff, p.pinned + (size_t)pslot * kChunk, plen);
            }
            prev = (long long)c;
        }
        if (prev >= 0) {
            const int pslot = 2 * t + (flip ^ 1);
            const size_t poff = (size_t)prev * kChunk, plen = std::min(kChunk, bytes - poff);
            if ((r = cudaEventSynchronize(p.ev[pslot])) != cudaSuccess) return r;
            memcpy(dst + poff, p.pinned + (size_t)pslot * kChunk, plen);
        }
        return cudaSuccess;
    });
    if (e != cudaSuccess) {
        set_error("staged D2H copy of %zu bytes -> %s", bytes, cudaGetErrorString(e));
        return GSX_ERR_CUDA;
    }
    return GSX_OK;
}

}  // namespace gsx

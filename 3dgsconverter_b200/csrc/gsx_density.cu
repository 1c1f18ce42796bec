// gsx_density.cu -- voxel histogram and voxel-membership mask of the density filter.
//
// Replaces data_processor.py:38-52 (quantise, np.unique(axis=0) with counts, dense = counts >=
// min_points) and :111-114 (per-point membership of the kept voxels).  The connected-component
// step in between (:59-106) stays on the host: it runs over at most N/min_points dense voxels
// and its tie-breaking depends on CPython set iteration order (SURVEY A.3).
//
// Instead of the reference's lexicographic sort of N int64 triples, voxels are counted with
// atomics: on a dense int32 grid over the voxel bounding box when that fits the workspace,
// otherwise in an open-addressing hash table keyed by the packed relative voxel coordinate.
// The thread whose increment makes a voxel reach the density threshold appends it to the
// dense list, so no pass over the grid is needed.  q = floor(x / f32(voxel)) uses the float32
// division of the reference (NumPy-2 weak-scalar semantics).
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_sor.cuh"

#include <limits.h>
#include <math.h>
#include <vector>

namespace gsx {

constexpr int kAxisBits = 21;
constexpr long long kAxisLim = 1ll << kAxisBits;

// Slots of the counter array of the dense-voxel extraction.
enum : int { kDense = 0, kDistinct = 1, kOutside = 2 };

// A NaN quotient, or one outside the int64 range, gives INT64_MIN on host and device alike: what the reference's
// np.floor(...).astype(np.int64) gives on x86.  (The device conversion alone saturates +inf to INT64_MAX, and the
// host one is undefined there.)
__host__ __device__ __forceinline__ long long voxel_of(float v, float voxel) {
#ifdef __CUDA_ARCH__
    const float f = floorf(__fdiv_rn(v, voxel));
#else
    const float f = floorf(v / voxel);
#endif
    return fabsf(f) < 9.2233720368547758e18f ? (long long)f : LLONG_MIN;   // -2^63 itself maps to INT64_MIN too
}

// Hash of the device tables and of the keep sets the host builds.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

// Key of a voxel relative to the box origin when every extent is < 2^21: three 21-bit fields, + 1 (0 = empty slot).
__host__ __device__ __forceinline__ uint64_t pack_rel(long long rx, long long ry, long long rz) {
    return (((uint64_t)rx << (2 * kAxisBits)) | ((uint64_t)ry << kAxisBits) | (uint64_t)rz) + 1ull;
}

// Two-word key for boxes that span 2^21 or more voxels on some axis (one far-away flyer with a small voxel):
// a = (rx << 32 | ry) + 1, b = rz + 1, exact for any extent < 2^31.
__host__ __device__ __forceinline__ void wide_key(long long rx, long long ry, long long rz, unsigned long long& a,
                                                  unsigned long long& b) {
    a = (((unsigned long long)rx << 32) | (unsigned long long)ry) + 1ull;
    b = (unsigned long long)rz + 1ull;
}

__host__ __device__ __forceinline__ uint64_t wide_slot(unsigned long long a, unsigned long long b) {
    return mix64(a ^ mix64(b));
}

struct Vox {
    long long x, y, z;
};

struct VoxGrid {
    long long q0[3];   // voxel-space origin
    long long dim[3];  // extent in voxels

    // Row-major cell index (z fastest) of a voxel in the box.
    __device__ __forceinline__ size_t cell(long long qx, long long qy, long long qz) const {
        return ((size_t)(qx - q0[0]) * dim[1] + (size_t)(qy - q0[1])) * dim[2] + (size_t)(qz - q0[2]);
    }
    __device__ __forceinline__ Vox voxel(size_t c) const {
        const size_t z = c % (size_t)dim[2], y = (c / (size_t)dim[2]) % (size_t)dim[1],
                     x = c / ((size_t)dim[2] * (size_t)dim[1]);
        return {(long long)x + q0[0], (long long)y + q0[1], (long long)z + q0[2]};
    }
};

// Whether voxel q lies in the box.  Compares before subtracting, so INT64_MIN - q0 is never formed.  Only rows with a
// NaN coordinate fall outside the box of the one-shot path (the box is the finite min/max of the cloud).
__device__ __forceinline__ bool in_box(long long qx, long long qy, long long qz, const VoxGrid& g) {
    return qx >= g.q0[0] && qx <= g.q0[0] + (g.dim[0] - 1) && qy >= g.q0[1] && qy <= g.q0[1] + (g.dim[1] - 1) &&
           qz >= g.q0[2] && qz <= g.q0[2] + (g.dim[2] - 1);
}

// Appends a voxel to the dense list: every append takes a slot of counters[kDense], the first `cap` are stored.
// `voxel()` is called only for a stored slot.  Returns the slot.
template <class VoxelOf>
__device__ __forceinline__ unsigned long long dense_append(unsigned long long* counters, long long* dense_vox,
                                                           int64_t cap, VoxelOf voxel) {
    const unsigned long long slot = atomicAdd(counters + kDense, 1ull);
    if ((int64_t)slot < cap) {
        const Vox q = voxel();
        dense_vox[3 * slot] = q.x;
        dense_vox[3 * slot + 1] = q.y;
        dense_vox[3 * slot + 2] = q.z;
    }
    return slot;
}

// The dense-voxel rule of one counting add of c rows to a voxel whose counter held `old`: the first add counts a
// distinct voxel, and the add that carries the count across thr (old < thr <= old + c: exactly one add does) appends
// the voxel to the dense list.
template <class VoxelOf>
__device__ __forceinline__ void dense_rule(int old, int c, int thr, unsigned long long* counters,
                                           long long* dense_vox, int64_t cap, VoxelOf voxel) {
    if (old == 0) atomicAdd(counters + kDistinct, 1ull);
    if (old < thr && old + c >= thr) dense_append(counters, dense_vox, cap, voxel);
}

// ---------------------------------------------------------------- counter tables
// at() returns the counter of an in-box voxel, claiming its slot on first sight; find() returns the count of a voxel.

struct GridTable {   // dense int32 grid over the voxel box
    int* cnt;
    __device__ __forceinline__ int* at(const VoxGrid& g, long long qx, long long qy, long long qz) const {
        return cnt + g.cell(qx, qy, qz);
    }
    __device__ __forceinline__ int find(const VoxGrid& g, long long qx, long long qy, long long qz) const {
        return cnt[g.cell(qx, qy, qz)];
    }
};

struct HashTable {   // 3 x 21-bit keys: key at keys[s], count at cnt[s]
    unsigned long long* keys;
    int* cnt;
    uint64_t slot_mask;
    __device__ __forceinline__ int* at(const VoxGrid& g, long long qx, long long qy, long long qz) const {
        const uint64_t key = pack_rel(qx - g.q0[0], qy - g.q0[1], qz - g.q0[2]);
        uint64_t s = mix64(key) & slot_mask;
        for (;;) {
            unsigned long long cur = keys[s];
            if (cur == 0ull) {
                unsigned long long prev = atomicCAS(keys + s, 0ull, (unsigned long long)key);
                cur = prev == 0ull ? (unsigned long long)key : prev;
            }
            if (cur == key) break;
            s = (s + 1) & slot_mask;
        }
        return cnt + s;
    }
    __device__ __forceinline__ int find(const VoxGrid& g, long long qx, long long qy, long long qz) const {
        const uint64_t key = pack_rel(qx - g.q0[0], qy - g.q0[1], qz - g.q0[2]);
        uint64_t s = mix64(key) & slot_mask;
        while (keys[s] != key) s = (s + 1) & slot_mask;
        return cnt[s];
    }
};

// Two-word keys {a, b} at ha[s], hb[s].  A slot is claimed by a CAS on `a`; the owner then publishes `b`; a thread
// that finds its own `a` waits for `b` (independent thread scheduling makes the intra-warp wait safe) and moves on if
// it differs (same x,y column, other z).
struct WideHashTable {
    unsigned long long* ha;
    unsigned long long* hb;
    int* cnt;
    uint64_t slot_mask;
    __device__ __forceinline__ uint64_t slot(const VoxGrid& g, long long qx, long long qy, long long qz,
                                             bool insert) const {
        unsigned long long a, b;
        wide_key(qx - g.q0[0], qy - g.q0[1], qz - g.q0[2], a, b);
        uint64_t s = wide_slot(a, b) & slot_mask;
        for (;;) {
            unsigned long long cur = *((volatile unsigned long long*)(ha + s));
            if (cur == 0ull) {
                if (!insert) return ~0ull;
                unsigned long long prev = atomicCAS(ha + s, 0ull, a);
                if (prev == 0ull) {
                    atomicExch(hb + s, b);
                    return s;
                }
                cur = prev;
            }
            if (cur == a) {
                unsigned long long bv;
                do {
                    bv = *((volatile unsigned long long*)(hb + s));
                } while (bv == 0ull);
                if (bv == b) return s;
            }
            s = (s + 1) & slot_mask;
        }
    }
    __device__ __forceinline__ int* at(const VoxGrid& g, long long qx, long long qy, long long qz) const {
        return cnt + slot(g, qx, qy, qz, true);
    }
    __device__ __forceinline__ int find(const VoxGrid& g, long long qx, long long qy, long long qz) const {
        const uint64_t s = slot(g, qx, qy, qz, false);
        return s == ~0ull ? 0 : cnt[s];
    }
};

// ---------------------------------------------------------------- histogram kernels
// One row per thread into any table.  DENSE: with the dense-voxel rule of the one-shot path.  Without it (the staged
// grid) the add's old value is unused and the add compiles to a reduction, which does not wait for a reply; a run-time
// switch would not do, as the compiler merges the two adds into one that returns the old value.
template <bool DENSE, class Table>
__global__ void __launch_bounds__(256) k_vox_count(const float* __restrict__ xyz, int64_t n, float voxel, VoxGrid g,
                                                   Table tab, int thr, unsigned long long* __restrict__ counters,
                                                   long long* __restrict__ dense_vox, int64_t cap,
                                                   unsigned long long* __restrict__ oob) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long qx = voxel_of(xyz[3 * i], voxel), qy = voxel_of(xyz[3 * i + 1], voxel),
                    qz = voxel_of(xyz[3 * i + 2], voxel);
    if (!in_box(qx, qy, qz, g)) {
        atomicAdd(oob, 1ull);  // rows dropped (non-finite coordinates)
        return;
    }
    const int old = atomicAdd(tab.at(g, qx, qy, qz), 1);
    if (DENSE) dense_rule(old, 1, thr, counters, dense_vox, cap, [&] { return Vox{qx, qy, qz}; });
}

// Dense-grid histogram with per-block aggregation: clustered clouds put 10^5..10^6 points into a handful of voxels and
// same-address global atomics serialise in L2.  Each block first counts its 2048 points in a 1024-slot shared-memory
// hash (cell index -> count) and then issues ONE global atomicAdd per distinct cell; the increment may be > 1, so the
// threshold crossing is detected as old < thr <= old + c (still exactly one block sees it).
constexpr int kAggItems = 8, kAggSlots = 1024;
__global__ void __launch_bounds__(256) k_vox_count_grid_agg(const float* __restrict__ xyz, int64_t n, float voxel,
                                                            VoxGrid g, int thr, int* __restrict__ grid,
                                                            unsigned long long* __restrict__ counters,
                                                            long long* __restrict__ dense_vox, int64_t cap) {
    __shared__ unsigned int skey[kAggSlots];
    __shared__ int sval[kAggSlots];
    for (int t = threadIdx.x; t < kAggSlots; t += 256) {
        skey[t] = 0xffffffffu;
        sval[t] = 0;
    }
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * (256 * kAggItems);
    unsigned long long bad = 0;   // rows dropped (non-finite coordinates)
    auto commit = [&](unsigned int idx, int c) {
        dense_rule(atomicAdd(grid + idx, c), c, thr, counters, dense_vox, cap, [&] { return g.voxel(idx); });
    };
#pragma unroll 2
    for (int e = 0; e < kAggItems; ++e) {
        const int64_t i = base + (int64_t)e * 256 + threadIdx.x;
        if (i >= n) break;
        long long qx = voxel_of(xyz[3 * i], voxel), qy = voxel_of(xyz[3 * i + 1], voxel),
                  qz = voxel_of(xyz[3 * i + 2], voxel);
        if (!in_box(qx, qy, qz, g)) {
            ++bad;
            continue;
        }
        const unsigned int idx = (unsigned int)g.cell(qx, qy, qz);
        unsigned int slot = (idx * 2654435761u) >> 22;  // 10 bits
        bool placed = false;
#pragma unroll 1
        for (int probe = 0; probe < 8 && !placed; ++probe) {
            unsigned int cur = atomicCAS(&skey[slot], 0xffffffffu, idx);
            if (cur == 0xffffffffu || cur == idx) {
                atomicAdd(&sval[slot], 1);
                placed = true;
            }
            slot = (slot + 1) & (kAggSlots - 1);
        }
        if (!placed) commit(idx, 1);
    }
    if (bad) atomicAdd(counters + kOutside, bad);
    __syncthreads();
    for (int t = threadIdx.x; t < kAggSlots; t += 256)
        if (sval[t] > 0) commit(skey[t], sval[t]);
}

// Small voxel boxes (<= kSmemCells cells: --density_sensitivity 0.5 over a 24-unit cloud is 22^3 = 10.6 k): the whole
// histogram lives in shared memory.  Persistent CTAs count a contiguous slice of the cloud with shared-memory atomics
// (4 splats = three 128-bit streaming loads per thread) and flush their non-zero bins with ONE global atomicAdd each:
// <= cells per CTA instead of one same-address global atomic per splat (clustered clouds put 10^5..10^6 splats into a
// handful of voxels).  thr > 0: also the dense-voxel detection of the one-shot path (the CTA whose add crosses thr).
constexpr int kSmemCells = 24 * 1024;
__global__ void __launch_bounds__(512)
    k_vox_count_smem(const float* __restrict__ xyz, int64_t n, float voxel, VoxGrid g, int ncell, int thr,
                     int* __restrict__ grid, unsigned long long* __restrict__ counters,
                     long long* __restrict__ dense_vox, int64_t cap, unsigned long long* __restrict__ oob) {
    extern __shared__ int sh_hist[];
    for (int t = threadIdx.x; t < ncell; t += blockDim.x) sh_hist[t] = 0;
    __syncthreads();
    const int64_t n4 = n / 4;                       // groups of 4 splats = 3 float4
    const int64_t per = (n4 + gridDim.x - 1) / gridDim.x;
    const int64_t g0 = (int64_t)blockIdx.x * per, g1 = g0 + per < n4 ? g0 + per : n4;
    const bool vec = (reinterpret_cast<uintptr_t>(xyz) & 15) == 0;
    unsigned long long bad = 0;
    auto add = [&](float x, float y, float z) {
        const long long qx = voxel_of(x, voxel), qy = voxel_of(y, voxel), qz = voxel_of(z, voxel);
        if (!in_box(qx, qy, qz, g)) {
            ++bad;
            return;
        }
        atomicAdd(&sh_hist[(int)g.cell(qx, qy, qz)], 1);
    };
    for (int64_t t = g0 + threadIdx.x; t < g1; t += blockDim.x) {
        if (vec) {
            const float4* p4 = reinterpret_cast<const float4*>(xyz) + 3 * t;
            const float4 a = ld_stream_f4(p4), b = ld_stream_f4(p4 + 1), c = ld_stream_f4(p4 + 2);
            add(a.x, a.y, a.z);
            add(a.w, b.x, b.y);
            add(b.z, b.w, c.x);
            add(c.y, c.z, c.w);
        } else {
            for (int e = 0; e < 4; ++e) add(xyz[12 * t + 3 * e], xyz[12 * t + 3 * e + 1], xyz[12 * t + 3 * e + 2]);
        }
    }
    if (blockIdx.x == 0)   // ragged tail (< 4 splats)
        for (int64_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) add(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    if (bad && oob) atomicAdd(oob, bad);
    __syncthreads();
    for (int t = threadIdx.x; t < ncell; t += blockDim.x) {
        const int c = sh_hist[t];
        if (c == 0) continue;
        const int old = atomicAdd(grid + t, c);
        if (thr > 0) dense_rule(old, c, thr, counters, dense_vox, cap, [&] { return g.voxel(t); });
    }
}

static int launch_vox_count_smem(const float* xyz, int64_t n, float voxel, const VoxGrid& g, size_t ncell, int thr, int* grid,
                                 unsigned long long* counters, long long* dvox, int64_t cap, unsigned long long* oob,
                                 cudaStream_t st) {
    const size_t smem = ncell * sizeof(int);
    static bool attr_done = false;
    if (!attr_done) {
        GSX_CUDA_CHECK(cudaFuncSetAttribute(k_vox_count_smem, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)(kSmemCells * sizeof(int))));
        attr_done = true;
    }
    int blocks = sm_count() * 2;
    const int64_t n4 = n / 4;
    if ((int64_t)blocks > (n4 + 511) / 512) blocks = (int)((n4 + 511) / 512);
    if (blocks < 1) blocks = 1;
    k_vox_count_smem<<<blocks, 512, smem, st>>>(xyz, n, voxel, g, (int)ncell, thr, grid, counters, dvox, cap, oob);
    return GSX_OK;
}

template <class Table>
__global__ void k_vox_dense_counts(const long long* __restrict__ dense_vox, int64_t nd, VoxGrid g, Table tab,
                                   int* __restrict__ dense_cnt) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nd) return;
    dense_cnt[t] = tab.find(g, dense_vox[3 * t], dense_vox[3 * t + 1], dense_vox[3 * t + 2]);
}

// ---------------------------------------------------------------- staged dense-grid API (multi-GPU)
// Rank-local histogram into a caller-owned int32 grid over a caller-chosen voxel box (the global one);
// the caller all-reduces the grid and then extracts the dense voxels.
__global__ void __launch_bounds__(256) k_vox_grid_dense(const int* __restrict__ grid, size_t ncell, VoxGrid g, int thr,
                                                        unsigned long long* __restrict__ counters,
                                                        long long* __restrict__ dense_vox,
                                                        int* __restrict__ dense_cnt, int64_t cap) {
    size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncell) return;
    int v = grid[c];
    if (v > 0) atomicAdd(counters + kDistinct, 1ull);
    if (v >= thr) {
        const unsigned long long slot = dense_append(counters, dense_vox, cap, [&] { return g.voxel(c); });
        if ((int64_t)slot < cap) dense_cnt[slot] = v;
    }
}

static int make_grid(const int64_t* q0, const int64_t* dim, VoxGrid& g, size_t& ncell) {
    double cells = 1.0;
    for (int a = 0; a < 3; ++a) {
        g.q0[a] = q0[a];
        g.dim[a] = dim[a];
        GSX_REQUIRE(dim[a] >= 1, GSX_ERR_ARG, "density: bad grid extent on axis %d", a);
        cells *= (double)dim[a];
    }
    GSX_REQUIRE(cells < 4.0e9, GSX_ERR_UNSUPPORTED, "density: grid too large for the dense path");
    ncell = (size_t)dim[0] * dim[1] * dim[2];
    return GSX_OK;
}

// ---------------------------------------------------------------- membership mask
// Keep sets: contains() tells whether a voxel is one of the kept voxels.  The host builds the set in the workspace.

// Bitmap form: when the bounding box of the kept voxels is small (the usual case -- a few clusters of voxels of one
// scene unit) one bit per voxel of that box replaces the hash probe: the whole set is a few KiB that stay in L1, and
// the kernel streams at the speed of the bbox mask instead of waiting on dependent table reads.
struct VoxBits {
    long long ox, oy, oz;
    unsigned long long dx, dy, dz;
    const uint32_t* bits;
    __device__ __forceinline__ uint8_t contains(long long qx, long long qy, long long qz) const {
        const unsigned long long rx = (unsigned long long)(qx - ox), ry = (unsigned long long)(qy - oy),
                                 rz = (unsigned long long)(qz - oz);
        if (rx >= dx || ry >= dy || rz >= dz) return 0;    // (negative differences wrap to huge values)
        const uint32_t idx = (uint32_t)((rx * dy + ry) * dz + rz);
        return (uint8_t)((__ldg(bits + (idx >> 5)) >> (idx & 31u)) & 1u);
    }
};

// Hash form: the keys of HashTable (one word per slot), or for kept voxels that span >= 2^21 on some axis the
// two-word keys of WideHashTable with {a, b} at set[2s], set[2s+1].
template <bool WIDE>
struct KeepHash {
    long long ox, oy, oz;
    const unsigned long long* set;
    uint64_t slot_mask;
    __device__ __forceinline__ uint8_t contains(long long qx, long long qy, long long qz) const {
        const long long rx = qx - ox, ry = qy - oy, rz = qz - oz;
        if (WIDE) {
            if (rx < 0 || ry < 0 || rz < 0 || rx >= (1ll << 31) || ry >= (1ll << 31) || rz >= (1ll << 31)) return 0;
            unsigned long long a, b;
            wide_key(rx, ry, rz, a, b);
            uint64_t s = wide_slot(a, b) & slot_mask;
            for (;;) {
                unsigned long long ca = __ldg(set + 2 * s);
                if (ca == 0ull) return 0;
                if (ca == a && __ldg(set + 2 * s + 1) == b) return 1;
                s = (s + 1) & slot_mask;
            }
        }
        if (rx < 0 || ry < 0 || rz < 0 || rx >= kAxisLim || ry >= kAxisLim || rz >= kAxisLim) return 0;
        uint64_t key = pack_rel(rx, ry, rz);
        uint64_t s = mix64(key) & slot_mask;
        for (;;) {
            unsigned long long cur = __ldg(set + s);
            if (cur == key) return 1;
            if (cur == 0ull) return 0;
            s = (s + 1) & slot_mask;
        }
    }
};

template <class Set>
__device__ __forceinline__ uint8_t vox_member(const Set& set, float x, float y, float z, float voxel) {
    return set.contains(voxel_of(x, voxel), voxel_of(y, voxel), voxel_of(z, voxel));
}

template <class Set>
__global__ void __launch_bounds__(256) k_vox_member(const float* __restrict__ xyz, int64_t begin, int64_t n,
                                                    float voxel, Set set, uint8_t* __restrict__ mask) {
    int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    mask[i] = vox_member(set, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], voxel);
}

// 4 points (3 x 128-bit loads) per thread, uchar4 store
template <class Set>
__global__ void __launch_bounds__(256) k_vox_member4(const float4* __restrict__ xyz4, int64_t n4, float voxel, Set set,
                                                     uchar4* __restrict__ mask4) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n4) return;
    float4 a = ld_stream_f4(xyz4 + 3 * t), b = ld_stream_f4(xyz4 + 3 * t + 1), c = ld_stream_f4(xyz4 + 3 * t + 2);
    uchar4 o;
    o.x = vox_member(set, a.x, a.y, a.z, voxel);
    o.y = vox_member(set, a.w, b.x, b.y, voxel);
    o.z = vox_member(set, b.z, b.w, c.x, voxel);
    o.w = vox_member(set, c.y, c.z, c.w, voxel);
    mask4[t] = o;
}

// The 4-wide kernel over whole groups of 4 rows when xyz is 16-byte and the mask 4-byte aligned, the scalar one over
// the rest.
template <class Set>
static int launch_member(const float* xyz, int64_t n, float voxel, const Set& set, uint8_t* mask, cudaStream_t st) {
    int64_t n4 = 0;
    if (((uintptr_t)xyz % 16 == 0) && ((uintptr_t)mask % 4 == 0)) {
        n4 = n / 4;
        if (n4 > 0) {
            k_vox_member4<<<(int)((n4 + 255) / 256), 256, 0, st>>>((const float4*)xyz, n4, voxel, set, (uchar4*)mask);
            GSX_KERNEL_CHECK();
        }
    }
    if (n - 4 * n4 > 0) {
        k_vox_member<<<(int)((n - 4 * n4 + 255) / 256), 256, 0, st>>>(xyz, 4 * n4, n, voxel, set, mask);
        GSX_KERNEL_CHECK();
    }
    return GSX_OK;
}

constexpr unsigned long long kMaxKeepBits = 1ull << 27;   // 16 MiB of bitmap at most; larger boxes use the hash set

}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_density_workspace_bytes(int64_t n, int64_t cap) {
    if (n < 1) n = 1;
    if (cap < 1) cap = 1;
    // hash path: table of >= 2n slots (power of two), 8-byte key + 4-byte count; plus minmax scratch
    size_t slots = 64;
    while (slots < (size_t)2 * n) slots <<= 1;
    return (int64_t)(slots * 12 + 6 * 1024 * 4 + (size_t)cap * 28 + 8192);
}

int gsx_density_voxel_count(const float* xyz, int64_t n, float voxel, int64_t min_points, int64_t* dense_vox_host,
                            int32_t* dense_cnt_host, int64_t cap, int64_t* n_dense_host, int64_t* n_voxels_host,
                            void* ws, int64_t ws_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::density_voxel_count");
    GSX_REQUIRE(n >= 1, GSX_ERR_ARG, "density: n must be >= 1");
    GSX_REQUIRE(voxel > 0.f, GSX_ERR_ARG, "density: voxel size must be > 0");
    GSX_REQUIRE(ws_bytes >= gsx_density_workspace_bytes(n, cap), GSX_ERR_WORKSPACE, "density: workspace too small");
    GSX_REQUIRE(cap >= 1, GSX_ERR_ARG, "density: cap must be >= 1");
    Carver c(ws, (size_t)ws_bytes);
    float* partial = c.take<float>(6 * 1024);
    float* minmax = c.take<float>(8);
    unsigned long long* counters = c.take<unsigned long long>(4);
    long long* dvox = c.take<long long>(3 * (size_t)cap);
    int* dcnt = c.take<int>((size_t)cap);
    size_t used = align_up(c.off, 256);
    GSX_REQUIRE(c.ok() && used < (size_t)ws_bytes, GSX_ERR_WORKSPACE, "density: workspace too small for cap=%lld",
                (long long)cap);
    char* blob = (char*)ws + used;
    size_t blob_bytes = (size_t)ws_bytes - used;

    int rc = sor_minmax(xyz, n, minmax, partial, st);
    if (rc) return rc;
    float mm[6];
    GSX_CUDA_CHECK(cudaMemcpyAsync(mm, minmax, sizeof(mm), cudaMemcpyDeviceToHost, st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    VoxGrid g;
    double cells = 1.0;
    bool wide = false;
    for (int a = 0; a < 3; ++a) {
        g.q0[a] = voxel_of(mm[a], voxel);  // floor(x/voxel) is monotone in x: min/max commute with it
        long long q1 = voxel_of(mm[3 + a], voxel);
        GSX_REQUIRE(g.q0[a] != LLONG_MIN && q1 != LLONG_MIN, GSX_ERR_UNSUPPORTED,
                    "density: non-finite or out-of-range coordinates on axis %d", a);
        // q1 >= q0; the unsigned difference is exact where the signed one could overflow
        GSX_REQUIRE((unsigned long long)q1 - (unsigned long long)g.q0[a] < (1ull << 31) - 1, GSX_ERR_UNSUPPORTED,
                    "density: voxel grid extent on axis %d exceeds 2^31 voxels", a);
        g.dim[a] = q1 - g.q0[a] + 1;
        if (g.dim[a] >= kAxisLim) wide = true;  // the packed 3 x 21-bit key does not fit: two-word keys
        cells *= (double)g.dim[a];
    }
    long long thr_ll = min_points < 1 ? 1 : min_points;
    GSX_REQUIRE(thr_ll < 2147483647ll, GSX_ERR_ARG, "density: min_points too large");
    int thr = (int)thr_ll;
    GSX_CUDA_CHECK(cudaMemsetAsync(counters, 0, 4 * sizeof(unsigned long long), st));
    auto count_rows = [&](const auto& tab) {
        k_vox_count<true><<<(int)((n + 255) / 256), 256, 0, st>>>(xyz, n, voxel, g, tab, thr, counters, dvox, cap,
                                                                  counters + kOutside);
    };
    // After the histogram: the refusals, then the counts of the dense voxels looked up in `tab`.
    auto read_dense = [&](const auto& tab) -> int {
        GSX_KERNEL_CHECK();
        unsigned long long hc[3];   // counters[kDense], [kDistinct], [kOutside]
        GSX_CUDA_CHECK(cudaMemcpyAsync(hc, counters, sizeof(hc), cudaMemcpyDeviceToHost, st));
        GSX_CUDA_CHECK(cudaStreamSynchronize(st));
        *n_dense_host = (int64_t)hc[kDense];
        if (n_voxels_host) *n_voxels_host = (int64_t)hc[kDistinct];
        // The reference puts a NaN row in a voxel outside the finite box.  Fewer than thr such rows make no dense
        // voxel, so dropping them is exact; with thr or more, one of those voxels may be dense, and that is refused.
        GSX_REQUIRE(hc[kOutside] < (unsigned long long)thr, GSX_ERR_UNSUPPORTED,
                    "density: %llu points have non-finite (NaN) coordinates, at least min_points = %d", hc[kOutside],
                    thr);
        GSX_REQUIRE((int64_t)hc[kDense] <= cap, GSX_ERR_WORKSPACE, "density: %llu dense voxels exceed cap %lld",
                    hc[kDense], (long long)cap);
        const int64_t nd = (int64_t)hc[kDense];
        if (nd > 0) {
            k_vox_dense_counts<<<(int)((nd + 127) / 128), 128, 0, st>>>(dvox, nd, g, tab, dcnt);
            GSX_KERNEL_CHECK();
            GSX_CUDA_CHECK(cudaMemcpyAsync(dense_vox_host, dvox, (size_t)nd * 24, cudaMemcpyDeviceToHost, st));
            GSX_CUDA_CHECK(cudaMemcpyAsync(dense_cnt_host, dcnt, (size_t)nd * 4, cudaMemcpyDeviceToHost, st));
            GSX_CUDA_CHECK(cudaStreamSynchronize(st));
        }
        return GSX_OK;
    };

    if (cells * 4.0 <= (double)blob_bytes) {
        const GridTable tab{(int*)blob};
        const size_t ncell = (size_t)g.dim[0] * g.dim[1] * g.dim[2];
        GSX_CUDA_CHECK(cudaMemsetAsync(blob, 0, ncell * 4, st));
        if (ncell <= (size_t)kSmemCells) {
            rc = launch_vox_count_smem(xyz, n, voxel, g, ncell, thr, tab.cnt, counters, dvox, cap, counters + kOutside,
                                       st);
            if (rc) return rc;
        } else if (ncell < 0xfffffff0ull) {
            const int ablocks = (int)((n + 256 * kAggItems - 1) / (256 * kAggItems));
            k_vox_count_grid_agg<<<ablocks, 256, 0, st>>>(xyz, n, voxel, g, thr, tab.cnt, counters, dvox, cap);
        } else {
            count_rows(tab);
        }
        return read_dense(tab);
    }
    size_t slots = 64;
    while (slots < (size_t)2 * n) slots <<= 1;
    GSX_REQUIRE(slots * 12 <= blob_bytes, GSX_ERR_WORKSPACE, "density: workspace too small for the hash table");
    if (!wide) {
        const HashTable tab{(unsigned long long*)blob, (int*)(blob + slots * 8), slots - 1};
        GSX_CUDA_CHECK(cudaMemsetAsync(blob, 0, slots * 12, st));
        count_rows(tab);
        return read_dense(tab);
    }
    slots >>= 1;   // two-word keys in the same budget: half the slots (still >= n), 20 bytes each
    const WideHashTable tab{(unsigned long long*)blob, (unsigned long long*)blob + slots, (int*)(blob + slots * 16),
                            slots - 1};
    GSX_CUDA_CHECK(cudaMemsetAsync(blob, 0, slots * 20, st));
    count_rows(tab);
    return read_dense(tab);
}

void gsx_density_voxel_range(const float* minmax_host, float voxel, int64_t* q0, int64_t* dim) {
    for (int a = 0; a < 3; ++a) {
        q0[a] = voxel_of(minmax_host[a], voxel);
        dim[a] = voxel_of(minmax_host[3 + a], voxel) - q0[a] + 1;
    }
}

int gsx_density_grid_count(const float* xyz, int64_t n, float voxel, const int64_t* q0, const int64_t* dim,
                           int32_t* grid_dev, unsigned long long* oob_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(voxel > 0.f, GSX_ERR_ARG, "density: voxel size must be > 0");
    VoxGrid g;
    size_t ncell;
    int rc = make_grid(q0, dim, g, ncell);
    if (rc) return rc;
    if (ncell <= (size_t)kSmemCells) {
        rc = launch_vox_count_smem(xyz, n, voxel, g, ncell, 0, grid_dev, nullptr, nullptr, 0, oob_dev, st);
        if (rc) return rc;
    } else {
        k_vox_count<false><<<(int)((n + 255) / 256), 256, 0, st>>>(xyz, n, voxel, g, GridTable{grid_dev}, 0, nullptr,
                                                                   nullptr, 0, oob_dev);
    }
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_density_grid_dense(const int32_t* grid_dev, const int64_t* q0, const int64_t* dim, int64_t min_points,
                           int64_t* dense_vox_host, int32_t* dense_cnt_host, int64_t cap, int64_t* n_dense_host,
                           int64_t* n_voxels_host, void* ws, int64_t ws_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    VoxGrid g;
    size_t ncell;
    int rc = make_grid(q0, dim, g, ncell);
    if (rc) return rc;
    GSX_REQUIRE(cap >= 1, GSX_ERR_ARG, "density: cap must be >= 1");
    Carver c(ws, (size_t)ws_bytes);
    unsigned long long* counters = c.take<unsigned long long>(4);
    long long* dvox = c.take<long long>(3 * (size_t)cap);
    int* dcnt = c.take<int>((size_t)cap);
    GSX_REQUIRE(c.ok(), GSX_ERR_WORKSPACE, "density: workspace too small for cap=%lld", (long long)cap);
    long long thr_ll = min_points < 1 ? 1 : min_points;
    GSX_REQUIRE(thr_ll < 2147483647ll, GSX_ERR_ARG, "density: min_points too large");
    GSX_CUDA_CHECK(cudaMemsetAsync(counters, 0, 4 * sizeof(unsigned long long), st));
    k_vox_grid_dense<<<(unsigned)((ncell + 255) / 256), 256, 0, st>>>(grid_dev, ncell, g, (int)thr_ll, counters, dvox,
                                                                      dcnt, cap);
    GSX_KERNEL_CHECK();
    unsigned long long hc[2];   // counters[kDense], [kDistinct]
    GSX_CUDA_CHECK(cudaMemcpyAsync(hc, counters, sizeof(hc), cudaMemcpyDeviceToHost, st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    *n_dense_host = (int64_t)hc[kDense];
    if (n_voxels_host) *n_voxels_host = (int64_t)hc[kDistinct];
    GSX_REQUIRE((int64_t)hc[kDense] <= cap, GSX_ERR_WORKSPACE, "density: %llu dense voxels exceed cap %lld",
                hc[kDense], (long long)cap);
    if (hc[kDense] > 0) {
        GSX_CUDA_CHECK(cudaMemcpyAsync(dense_vox_host, dvox, (size_t)hc[kDense] * 24, cudaMemcpyDeviceToHost, st));
        GSX_CUDA_CHECK(cudaMemcpyAsync(dense_cnt_host, dcnt, (size_t)hc[kDense] * 4, cudaMemcpyDeviceToHost, st));
        GSX_CUDA_CHECK(cudaStreamSynchronize(st));
    }
    return GSX_OK;
}

int gsx_density_member_mask(const float* xyz, int64_t n, float voxel, const int64_t* keep, int64_t n_keep,
                            uint8_t* mask, void* ws, int64_t ws_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx::density_member_mask");
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(voxel > 0.f, GSX_ERR_ARG, "density: voxel size must be > 0");
    if (n_keep == 0) {
        GSX_CUDA_CHECK(cudaMemsetAsync(mask, 0, (size_t)n, st));
        return GSX_OK;
    }
    long long o[3] = {keep[0], keep[1], keep[2]}, hi[3] = {keep[0], keep[1], keep[2]};
    for (int64_t t = 1; t < n_keep; ++t)
        for (int a = 0; a < 3; ++a) {
            if (keep[3 * t + a] < o[a]) o[a] = keep[3 * t + a];
            if (keep[3 * t + a] > hi[a]) hi[a] = keep[3 * t + a];
        }
    bool wide = false;
    for (int a = 0; a < 3; ++a) {
        GSX_REQUIRE(hi[a] - o[a] < (1ll << 31), GSX_ERR_UNSUPPORTED, "density: kept voxels span more than 2^31 on axis %d", a);
        if (hi[a] - o[a] >= kAxisLim) wide = true;
    }
    {   // bitmap over the bounding box of the kept voxels, when that box is small enough
        const unsigned long long dx = (unsigned long long)(hi[0] - o[0] + 1), dy = (unsigned long long)(hi[1] - o[1] + 1),
                                 dz = (unsigned long long)(hi[2] - o[2] + 1);
        // (each factor < 2^31: the products below cannot overflow before the comparisons reject them)
        const bool small = dx <= kMaxKeepBits && dy <= kMaxKeepBits && dx * dy <= kMaxKeepBits &&
                           dx * dy * dz <= kMaxKeepBits;
        const size_t nwords = small ? (size_t)((dx * dy * dz + 31) / 32) : 0;
        if (small && nwords * 4 <= (size_t)ws_bytes) {
            std::vector<uint32_t> bm(nwords, 0u);
            for (int64_t t = 0; t < n_keep; ++t) {
                const unsigned long long idx = ((unsigned long long)(keep[3 * t] - o[0]) * dy +
                                                (unsigned long long)(keep[3 * t + 1] - o[1])) * dz +
                                               (unsigned long long)(keep[3 * t + 2] - o[2]);
                bm[idx >> 5] |= 1u << (idx & 31);
            }
            GSX_CUDA_CHECK(cudaMemcpyAsync(ws, bm.data(), nwords * 4, cudaMemcpyHostToDevice, st));
            GSX_CUDA_CHECK(cudaStreamSynchronize(st));  // bm is a stack-owned pageable buffer
            return launch_member(xyz, n, voxel, VoxBits{o[0], o[1], o[2], dx, dy, dz, (const uint32_t*)ws}, mask, st);
        }
    }
    size_t slots = 64;
    while (slots < (size_t)2 * n_keep) slots <<= 1;
    const size_t words = wide ? 2 : 1;
    GSX_REQUIRE(slots * 8 * words <= (size_t)ws_bytes, GSX_ERR_WORKSPACE, "density: workspace too small for the keep set");
    std::vector<unsigned long long> tab(slots * words, 0ull);
    for (int64_t t = 0; t < n_keep; ++t) {
        const long long rx = keep[3 * t] - o[0], ry = keep[3 * t + 1] - o[1], rz = keep[3 * t + 2] - o[2];
        if (!wide) {
            const uint64_t key = pack_rel(rx, ry, rz);
            uint64_t s = mix64(key) & (slots - 1);
            while (tab[s] != 0ull && tab[s] != key) s = (s + 1) & (slots - 1);
            tab[s] = key;
        } else {
            unsigned long long a, b;
            wide_key(rx, ry, rz, a, b);
            uint64_t s = wide_slot(a, b) & (slots - 1);
            while (tab[2 * s] != 0ull && !(tab[2 * s] == a && tab[2 * s + 1] == b)) s = (s + 1) & (slots - 1);
            tab[2 * s] = a;
            tab[2 * s + 1] = b;
        }
    }
    GSX_CUDA_CHECK(cudaMemcpyAsync(ws, tab.data(), slots * 8 * words, cudaMemcpyHostToDevice, st));
    GSX_CUDA_CHECK(cudaStreamSynchronize(st));  // tab is a stack-owned pageable buffer
    const unsigned long long* set = (const unsigned long long*)ws;
    if (wide) return launch_member(xyz, n, voxel, KeepHash<true>{o[0], o[1], o[2], set, slots - 1}, mask, st);
    return launch_member(xyz, n, voxel, KeepHash<false>{o[0], o[1], o[2], set, slots - 1}, mask, st);
}

}  // extern "C"

// gsx_parquet.cu -- the Parquet writer's kernels for sm_90a (H100): ParquetFormat.write (formats/parquet.py:59-112)
// hands the renamed frame to pandas' to_parquet; gsx builds the same table's file from device rows (gsx/parquet.py).
//
//   k_pq_split       a CTA owns a 2048-row tile (one page holds 128 of them): it stages 64 rows at a time in shared
//                    memory, writes every column's 32-bit patterns column-major (uint8 widened), and counts the tile's
//                    nulls (NaN) per column; min and max keys (order-preserving, NaN excluded) go to the column chunk
//                    with one atomicMin / atomicMax per CTA and column.  Min and max do not depend on the order.
//   k_pq_insert      every non-null pattern of a column chunk into the chunk's open-addressing table in HBM (64-bit
//                    slots: 1 << 32 | pattern, 0 empty); a chunk stops inserting once it holds more than 262 144.
//   k_pq_collect     the patterns of the tables of the chunks that take a dictionary, as (job << 32 | pattern) keys;
//                    gsx::radix_sort_keys orders them, so the dictionary is ascending and independent of scheduling.
//   k_pq_rank        each sorted pattern's rank into its table slot (the slot's high word becomes rank + 1) and into
//                    the dictionary values.
//   k_pq_index       every non-null value of a dictionary chunk replaced by its rank; per page the least and greatest
//                    rank (a page whose ranks are all equal is written as one RLE run).
//   k_pq_data_pages  a CTA per 2048-row tile of a data page: the page's definition levels (one RLE run, or one
//                    bit-packed run when it has nulls), then the non-null values compacted (a block scan plus the
//                    counts of the tiles before it in the page), PLAIN or bit-packed indices ORed into 32-bit words.
//   k_pq_dict_pages  the dictionary pages: the sorted values, PLAIN.
//   k_pq_snappy      a CTA per 64 KiB piece of a page body: Snappy elements with copies of distance 1 (byte runs) or 4
//                    (repeated 32-bit values) of >= 8 bytes inside the piece, taken greedily from the left (the longer
//                    of the two: they never tie), and literals.  The candidates come from two ballots and an AND of 8
//                    shifted words; warp 0 walks them.
//   k_pq_assemble    the host's page headers and footer and the compressed pieces into the file buffer.
#include "../../include/gsx.h"

#include "gsx_bits.cuh"
#include "gsx_common.cuh"
#include "gsx_radix.cuh"
#include "gsx_staged.cuh"

namespace gsx {

namespace {

constexpr int kThreads = 256;
constexpr int64_t kRowGroup = 1 << 20;
constexpr int64_t kPage = 1 << 18;
constexpr int kTile = 2048;              // rows per split / page-body CTA; a page is 128 tiles
constexpr int kStage = 64;               // rows staged in shared memory at a time
constexpr int kMaxCols = 1024;
constexpr int kRowMax = 1024;
constexpr uint32_t kDictMax = 1u << 18;  // pyarrow's 1 MiB dictionary page limit, in float32 values
// Least table size: k_pq_insert stops a chunk only once a thread reads its count above kDictMax, so every thread past
// that check (up to one resident grid, 132 SMs x 2048 threads on an H100) may still insert.  2^19 slots < 2^18 + 132 *
// 2048 could fill, and a full table's failing threads could wrap the count back below the limit.
constexpr int kSlotsMin = 20;
constexpr int kPiece = 1 << 16;
constexpr int kPieceCap = kPiece + 16;   // a piece's elements never exceed its literal-only encoding (3 tag bytes)
constexpr int kJobs = 1024;              // literal copies per walk round

__device__ __forceinline__ bool is_null(uint32_t v) { return (v & 0x7FFFFFFFu) > 0x7F800000u; }

__device__ __forceinline__ uint32_t order_key(uint32_t v, int kind) {
    return kind ? v : float_to_ord(__uint_as_float(v));
}

__device__ __forceinline__ uint32_t mix(uint32_t h) {   // murmur3's finaliser
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    return h ^ (h >> 16);
}

__device__ __forceinline__ int varint_put(uint8_t* p, uint32_t v) {
    int k = 0;
    while (v >= 0x80) {
        p[k++] = (uint8_t)(v | 0x80);
        v >>= 7;
    }
    p[k++] = (uint8_t)v;
    return k;
}
__host__ __device__ __forceinline__ int varint_len(uint32_t v) {
    int k = 1;
    while (v >= 0x80) {
        v >>= 7;
        ++k;
    }
    return k;
}

// ------------------------------------------------------------------------------------------------------------ split
__global__ void __launch_bounds__(kThreads) k_pq_split(const uint8_t* __restrict__ rows, int64_t n, int row_bytes,
                                                       const int2* __restrict__ cols, int ncols,
                                                       uint32_t* __restrict__ out, uint32_t* __restrict__ tile_nulls,
                                                       uint32_t* __restrict__ kmin, uint32_t* __restrict__ kmax,
                                                       int ngroups) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t* s_null = reinterpret_cast<uint32_t*>(smem);
    uint32_t* s_min = s_null + ncols;
    uint32_t* s_max = s_min + ncols;
    int2* s_col = reinterpret_cast<int2*>(s_max + ncols + (ncols & 1));
    uint8_t* stage = reinterpret_cast<uint8_t*>(s_col + ncols);
    stage += (16 - ((uintptr_t)stage & 15)) & 15;
    for (int c = threadIdx.x; c < ncols; c += kThreads) {
        s_null[c] = 0;
        s_min[c] = 0xFFFFFFFFu;
        s_max[c] = 0;
        s_col[c] = cols[c];
    }
    const int64_t base = (int64_t)blockIdx.x * kTile;
    const int tile_rows = (int)(n - base < kTile ? n - base : kTile);
    const int r = threadIdx.x % kStage, h = threadIdx.x / kStage;
    for (int s0 = 0; s0 < tile_rows; s0 += kStage) {
        const int nr = tile_rows - s0 < kStage ? tile_rows - s0 : kStage;
        __syncthreads();
        const uint8_t* in = load_staged(stage, rows + (base + s0) * row_bytes, nr * row_bytes);
        __syncthreads();
        for (int c = h; c < ncols; c += kThreads / kStage) {
            const int2 cd = s_col[c];
            uint32_t v = 0;
            bool nul = false;
            if (r < nr) {
                const uint8_t* p = in + r * row_bytes + cd.x;
                v = cd.y ? p[0] : (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
                out[(int64_t)c * n + base + s0 + r] = v;
                nul = !cd.y && is_null(v);
            }
            const bool val = r < nr && !nul;
            const uint32_t k = order_key(v, cd.y);
            const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, nul));
            const uint32_t lo = __reduce_min_sync(0xFFFFFFFFu, val ? k : 0xFFFFFFFFu);
            const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, val ? k : 0u);
            const bool any = __any_sync(0xFFFFFFFFu, val);
            if ((threadIdx.x & 31) == 0) {
                if (cnt) atomicAdd(&s_null[c], cnt);
                if (any) {
                    atomicMin(&s_min[c], lo);
                    atomicMax(&s_max[c], hi);
                }
            }
        }
    }
    __syncthreads();
    const int64_t ntiles = (n + kTile - 1) / kTile;
    const int g = (int)(base / kRowGroup);
    for (int c = threadIdx.x; c < ncols; c += kThreads) {
        tile_nulls[(int64_t)c * ntiles + blockIdx.x] = s_null[c];
        if (s_min[c] <= s_max[c] && s_null[c] < (uint32_t)tile_rows) {
            atomicMin(&kmin[(int64_t)c * ngroups + g], s_min[c]);
            atomicMax(&kmax[(int64_t)c * ngroups + g], s_max[c]);
        }
    }
}

// ----------------------------------------------------------------------------------------------------- dictionaries
// Row r of the batch's row groups [g0, g0 + ng): blockIdx.y is the column.
__global__ void __launch_bounds__(kThreads) k_pq_insert(const uint32_t* __restrict__ cols, int64_t n, int g0, int ng,
                                                        int ngroups, unsigned long long* __restrict__ table,
                                                        int slots_log2, uint32_t* __restrict__ distinct) {
    const int64_t r = g0 * kRowGroup + (int64_t)blockIdx.x * kThreads + threadIdx.x;
    const int c = blockIdx.y;
    if (r >= n || r >= (int64_t)(g0 + ng) * kRowGroup) return;
    const int g = (int)(r / kRowGroup);
    uint32_t* cnt = &distinct[(int64_t)c * ngroups + g];
    if (*(volatile uint32_t*)cnt > kDictMax) return;
    const uint32_t v = cols[(int64_t)c * n + r];
    if (is_null(v)) return;
    const uint32_t mask = (1u << slots_log2) - 1;
    unsigned long long* t = table + (((int64_t)(g - g0) * gridDim.y + c) << slots_log2);
    const unsigned long long want = (1ull << 32) | v;
    uint32_t s = mix(v) & mask;
    for (uint32_t probe = 0; probe <= mask; ++probe, s = (s + 1) & mask) {
        const unsigned long long prev = atomicCAS(&t[s], 0ull, want);
        if (prev == 0ull) {
            atomicAdd(cnt, 1u);
            return;
        }
        if (prev == want) return;
        if (*(volatile uint32_t*)cnt > kDictMax) return;
    }
    atomicAdd(cnt, kDictMax + 1);   // table full: no dictionary for this chunk
}

// jobs int64 [njobs][3]: (table index in the batch, first key in the sort array, first dictionary value)
__global__ void __launch_bounds__(kThreads) k_pq_collect(const unsigned long long* __restrict__ table, int slots_log2,
                                                         const int64_t* __restrict__ jobs,
                                                         unsigned int* __restrict__ fill,
                                                         unsigned long long* __restrict__ keys) {
    const int j = blockIdx.y;
    const unsigned long long* t = table + (jobs[3 * j] << slots_log2);
    for (int64_t s = (int64_t)blockIdx.x * kThreads + threadIdx.x; s < (1ll << slots_log2);
         s += (int64_t)gridDim.x * kThreads) {
        const unsigned long long e = t[s];
        if (e) keys[jobs[3 * j + 1] + atomicAdd(&fill[j], 1u)] = ((unsigned long long)j << 32) | (e & 0xFFFFFFFFull);
    }
}

__global__ void __launch_bounds__(kThreads) k_pq_rank(unsigned long long* __restrict__ table, int slots_log2,
                                                      const int64_t* __restrict__ jobs,
                                                      const unsigned long long* __restrict__ keys, int64_t m,
                                                      uint32_t* __restrict__ dict_vals) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= m) return;
    const unsigned long long k = keys[i];
    const int j = (int)(k >> 32);
    const uint32_t v = (uint32_t)k;
    const uint32_t rank = (uint32_t)(i - jobs[3 * j + 1]);
    dict_vals[jobs[3 * j + 2] + rank] = v;
    unsigned long long* t = table + (jobs[3 * j] << slots_log2);
    const uint32_t mask = (1u << slots_log2) - 1;
    for (uint32_t s = mix(v) & mask;; s = (s + 1) & mask) {
        if ((uint32_t)t[s] == v && (t[s] >> 32)) {
            t[s] = ((unsigned long long)(rank + 1) << 32) | v;
            return;
        }
    }
}

// dict_chunk int32 [ncols][ng]: 1 where the chunk takes its dictionary.  page_idx uint32 [2][ncols][npages].
__global__ void __launch_bounds__(kThreads) k_pq_index(uint32_t* __restrict__ cols, int64_t n, int g0, int ng,
                                                       const unsigned long long* __restrict__ table, int slots_log2,
                                                       const int32_t* __restrict__ dict_chunk,
                                                       uint32_t* __restrict__ page_idx, int64_t npages) {
    const int64_t rb = g0 * kRowGroup + (int64_t)blockIdx.x * kThreads, r = rb + threadIdx.x;
    const int c = blockIdx.y;
    const bool in = r < n && r < (int64_t)(g0 + ng) * kRowGroup;
    const int g = (int)(rb / kRowGroup);          // 256 rows never straddle a row group
    if (!dict_chunk[c * ng + (g - g0)]) return;   // uniform over the CTA
    uint32_t rank = 0;
    bool val = false;
    if (in) {
        const uint32_t v = cols[(int64_t)c * n + r];
        if (!is_null(v)) {
            const unsigned long long* t = table + (((int64_t)(g - g0) * gridDim.y + c) << slots_log2);
            const uint32_t mask = (1u << slots_log2) - 1;
            for (uint32_t s = mix(v) & mask;; s = (s + 1) & mask) {
                const unsigned long long e = t[s];
                if ((uint32_t)e == v && (e >> 32)) {
                    rank = (uint32_t)(e >> 32) - 1;
                    break;
                }
            }
            cols[(int64_t)c * n + r] = rank;
            val = true;
        }
    }
    const uint32_t lo = __reduce_min_sync(0xFFFFFFFFu, val ? rank : 0xFFFFFFFFu);
    const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, val ? rank : 0u);
    if ((threadIdx.x & 31) == 0 && lo != 0xFFFFFFFFu) {   // a warp's 32 rows lie in one page
        const int64_t p = r / kPage;
        atomicMin(&page_idx[(int64_t)c * npages + p], lo);
        atomicMax(&page_idx[((int64_t)gridDim.y + c) * npages + p], hi);
    }
}

// ------------------------------------------------------------------------------------------------------- page bodies
// info int64 [ncols][npages][4]: body offset, nulls, bit width (0 = PLAIN), all ranks equal
__global__ void __launch_bounds__(kThreads) k_pq_data_pages(const uint32_t* __restrict__ cols, int64_t n,
                                                            const uint32_t* __restrict__ tile_nulls, int64_t ntiles,
                                                            const int64_t* __restrict__ info, int64_t npages,
                                                            uint32_t* __restrict__ body) {
    __shared__ uint32_t s_warp[kThreads / 32];
    __shared__ uint32_t s_before;
    const int c = blockIdx.y;
    const int64_t tile = blockIdx.x;
    const int64_t p = tile * kTile / kPage;
    const int64_t t0 = p * (kPage / kTile);
    const int64_t* in = info + ((int64_t)c * npages + p) * 4;
    const int64_t off = in[0];
    const int nulls = (int)in[1], w = (int)in[2];
    const bool equal = in[3] != 0;
    const int64_t prow0 = p * kPage;
    const int rows = (int)(n - prow0 < kPage ? n - prow0 : kPage);
    const int nn = rows - nulls;
    const int gbytes = (rows + 7) / 8;
    const int defs = nulls ? varint_len(2 * gbytes + 1) + gbytes : varint_len(2 * rows) + 1;
    const int64_t vstart = off + 4 + defs;
    const int64_t pstart = vstart + 1 + varint_len(2 * ((nn + 7) / 8) + 1);
    uint8_t* b = reinterpret_cast<uint8_t*>(body);
    // non-null values in the page's tiles before this one
    uint32_t acc = 0;
    for (int64_t t = t0 + threadIdx.x; t < tile; t += kThreads) acc += kTile - tile_nulls[(int64_t)c * ntiles + t];
    acc = __reduce_add_sync(0xFFFFFFFFu, acc);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int k = 0; k < kThreads / 32; ++k) s += s_warp[k];
        s_before = s;
    }
    __syncthreads();
    // this thread's 8 rows
    const int64_t r0 = tile * kTile + threadIdx.x * 8;
    uint32_t v[8];
    uint32_t bits = 0;   // non-null rows (dictionary chunks hold ranks, which never look like NaN, and their nulls)
    for (int k = 0; k < 8; ++k) {
        const int64_t r = r0 + k;
        v[k] = r < n ? cols[(int64_t)c * n + r] : 0;
        if (r < n && !is_null(v[k])) bits |= 1u << k;
    }
    const uint32_t cnt = __popc(bits);
    uint32_t incl = cnt;
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if ((threadIdx.x & 31) >= d) incl += y;
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (int k = 0; k < (int)(threadIdx.x >> 5); ++k) wbase += s_warp[k];
    uint32_t ord = s_before + wbase + incl - cnt;   // ordinal of this thread's first non-null value in the page
    const int prow = (int)(r0 - prow0);
    if (tile == t0 && threadIdx.x == 0) {
        uint8_t* h = b + off;
        h[0] = (uint8_t)defs;
        h[1] = (uint8_t)(defs >> 8);
        h[2] = (uint8_t)(defs >> 16);
        h[3] = (uint8_t)(defs >> 24);
        if (nulls) {
            varint_put(h + 4, 2 * gbytes + 1);
        } else {
            h[4 + varint_put(h + 4, 2 * rows)] = 1;
        }
        if (w) {
            b[vstart] = (uint8_t)w;
            if (nn > 0) varint_put(b + vstart + 1, equal ? 2 * nn : 2 * ((nn + 7) / 8) + 1);
        }
    }
    if (nulls && prow < rows) b[off + 4 + varint_len(2 * gbytes + 1) + prow / 8] = (uint8_t)bits;
    if (r0 >= n || !cnt) return;
    if (w && !equal) {   // the thread's ranks are consecutive in the run: pack them, then OR the words they cover
        const uint64_t pos = (uint64_t)pstart * 8 + (uint64_t)ord * w;
        const uint32_t sh = (uint32_t)(pos & 31);
        uint32_t acc[6] = {0u, 0u, 0u, 0u, 0u, 0u};
        uint32_t bit = sh;
        for (int k = 0; k < 8; ++k) {
            if (!(bits >> k & 1)) continue;
            const uint64_t x = (uint64_t)v[k] << (bit & 31);
            acc[bit >> 5] |= (uint32_t)x;
            if ((bit & 31) + w > 32) acc[(bit >> 5) + 1] |= (uint32_t)(x >> 32);
            bit += w;
        }
        for (uint32_t q = 0; q <= (bit - 1) >> 5; ++q)
            if (acc[q]) atomicOr(&body[(pos >> 5) + q], acc[q]);
        return;
    }
    for (int k = 0; k < 8; ++k) {
        if (!(bits >> k & 1)) continue;
        const uint32_t x = v[k];
        if (w == 0) {
            uint8_t* d = b + vstart + 4 * (int64_t)ord;
            d[0] = (uint8_t)x;
            d[1] = (uint8_t)(x >> 8);
            d[2] = (uint8_t)(x >> 16);
            d[3] = (uint8_t)(x >> 24);
        } else if (ord == 0) {   // all ranks equal: the RLE run's value
            uint8_t* d = b + vstart + 1 + varint_len(2 * nn);
            for (int q = 0; q < (w + 7) / 8; ++q) d[q] = (uint8_t)(x >> (8 * q));
        }
        ++ord;
    }
}

// jobs int64 [njobs][3]: first dictionary value, body offset, entries
__global__ void __launch_bounds__(kThreads) k_pq_dict_pages(const uint32_t* __restrict__ dict_vals,
                                                            const int64_t* __restrict__ jobs,
                                                            int64_t njobs, uint32_t* __restrict__ body) {
    for (int64_t jb = blockIdx.y; jb < njobs; jb += gridDim.y) {
        const int64_t* j = jobs + 3 * jb;
        const int64_t first = j[0], cnt = j[2];
        uint32_t* d = body + j[1] / 4;   // body offsets are 16-byte aligned
        for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < cnt; i += (int64_t)gridDim.x * kThreads)
            d[i] = dict_vals[first + i];
    }
}

// ----------------------------------------------------------------------------------------------------------- snappy
struct LitJob {
    uint32_t src, dst, len;
};
constexpr int kWords = kPiece / 32 + 1;
constexpr size_t kSnappySmem = kPiece + 16 + 3 * kWords * 4 + kJobs * sizeof(LitJob);

__device__ __forceinline__ uint32_t run_from(const uint32_t* e, int i, int len) {   // consecutive set bits from i
    int k = i;
    while (k < len) {
        const uint32_t y = e[k >> 5] >> (k & 31);
        if (~y == 0u) {
            k += 32;
            continue;
        }
        const int f = __ffs(~y) - 1, avail = 32 - (k & 31);
        k += f;
        if (f < avail) break;
    }
    return (uint32_t)((k < len ? k : len) - i);
}

__device__ __forceinline__ int literal_tag(uint8_t* d, uint32_t L) {
    const uint32_t m = L - 1;
    if (m < 60) {
        d[0] = (uint8_t)(m << 2);
        return 1;
    }
    if (m < 256) {
        d[0] = 60 << 2;
        d[1] = (uint8_t)m;
        return 2;
    }
    d[0] = 61 << 2;
    d[1] = (uint8_t)m;
    d[2] = (uint8_t)(m >> 8);
    return 3;
}

__device__ __forceinline__ int copy_elems(uint8_t* d, uint32_t d1, uint32_t L) {
    int k = 0;
    while (L > 64) {
        d[k++] = (63 << 2) | 2;
        d[k++] = (uint8_t)d1;
        d[k++] = 0;
        L -= 64;
    }
    if (L >= 4 && L <= 11) {
        d[k++] = (uint8_t)(((L - 4) << 2) | 1);
        d[k++] = (uint8_t)d1;
    } else {
        d[k++] = (uint8_t)(((L - 1) << 2) | 2);
        d[k++] = (uint8_t)d1;
        d[k++] = 0;
    }
    return k;
}

// pieces int64 [m][3]: page, body offset, bytes
__global__ void __launch_bounds__(kThreads) k_pq_snappy(const uint8_t* __restrict__ body,
                                                        const int64_t* __restrict__ pieces,
                                                        uint8_t* __restrict__ scratch, uint32_t* __restrict__ sizes,
                                                        uint32_t* __restrict__ page_csize) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* s_b = smem;
    uint32_t* s_e1 = reinterpret_cast<uint32_t*>(smem + kPiece + 16);
    uint32_t* s_e4 = s_e1 + kWords;
    uint32_t* s_c = s_e4 + kWords;
    LitJob* s_job = reinterpret_cast<LitJob*>(s_c + kWords);
    __shared__ int s_njobs, s_done;
    const int64_t* pc = pieces + 3 * (int64_t)blockIdx.x;
    const int len = (int)pc[2];
    const uint4* src = reinterpret_cast<const uint4*>(body + pc[1]);
    for (int i = threadIdx.x; i < (len + 15) / 16; i += kThreads) reinterpret_cast<uint4*>(s_b)[i] = src[i];
    __syncthreads();
    const int nw = (len + 31) / 32;
    for (int wd = threadIdx.x >> 5; wd < kWords; wd += kThreads / 32) {
        const int i = wd * 32 + (threadIdx.x & 31);
        const bool e1 = i < len && i >= 1 && s_b[i] == s_b[i - 1];
        const bool e4 = i < len && i >= 4 && s_b[i] == s_b[i - 4];
        const uint32_t b1 = __ballot_sync(0xFFFFFFFFu, e1), b4 = __ballot_sync(0xFFFFFFFFu, e4);
        if ((threadIdx.x & 31) == 0) {
            s_e1[wd] = b1;
            s_e4[wd] = b4;
        }
    }
    __syncthreads();
    for (int wd = threadIdx.x; wd < nw; wd += kThreads) {
        const uint64_t x1 = s_e1[wd] | (uint64_t)s_e1[wd + 1] << 32, x4 = s_e4[wd] | (uint64_t)s_e4[wd + 1] << 32;
        uint64_t a1 = x1, a4 = x4;
        for (int k = 1; k < 8; ++k) {
            a1 &= x1 >> k;
            a4 &= x4 >> k;
        }
        s_c[wd] = (uint32_t)(a1 | a4);
    }
    if (threadIdx.x == 0) s_done = 0;
    __syncthreads();
    uint8_t* out = scratch + (int64_t)blockIdx.x * kPieceCap;
    // warp 0 walks with uniform state; lane 0 writes tags and copies
    int i = 0, lit = 0;
    uint32_t o = 0;
    while (true) {
        if (threadIdx.x < 32) {
            int nj = 0;
            bool done = false;
            while (nj < kJobs) {
                // next candidate at or after i
                int j = len;
                for (int w0 = i >> 5; w0 < nw; w0 += 32) {
                    const int wd = w0 + (int)threadIdx.x;
                    uint32_t x = wd < nw ? s_c[wd] : 0u;
                    if (wd == (i >> 5)) x &= 0xFFFFFFFFu << (i & 31);
                    const uint32_t hit = __ballot_sync(0xFFFFFFFFu, x != 0);
                    if (hit) {
                        const int lane = __ffs(hit) - 1;
                        const uint32_t xl = __shfl_sync(0xFFFFFFFFu, x, lane);
                        j = (w0 + lane) * 32 + __ffs(xl) - 1;
                        break;
                    }
                }
                if (j >= len) {
                    if (len > lit) {
                        if (threadIdx.x == 0) {
                            const int t = literal_tag(out + o, (uint32_t)(len - lit));
                            s_job[nj] = LitJob{(uint32_t)lit, o + t, (uint32_t)(len - lit)};
                        }
                        o += (uint32_t)(len - lit) + (len - lit <= 60 ? 1 : len - lit <= 256 ? 2 : 3);
                        ++nj;
                    }
                    done = true;
                    break;
                }
                // L1 == L4 cannot happen: e1[j - 1] and e4[j - 1] are clear at a chosen start (else j - 1 was the
                // candidate, or the previous copy went on), so b[j - 2] != b[j - 1]: beside a distance-1 run of >= 8
                // (b[j - 1 .. j + 7] equal) the distance-4 run is <= 2 bytes
                const uint32_t L1 = run_from(s_e1, j, len), L4 = run_from(s_e4, j, len);
                const uint32_t L = L1 >= L4 ? L1 : L4;
                const uint32_t d = L1 >= L4 ? 1 : 4;
                if (j > lit) {
                    const uint32_t ll = (uint32_t)(j - lit);
                    if (threadIdx.x == 0) {
                        const int t = literal_tag(out + o, ll);
                        s_job[nj] = LitJob{(uint32_t)lit, o + t, ll};
                    }
                    o += ll + (ll <= 60 ? 1 : ll <= 256 ? 2 : 3);
                    ++nj;
                }
                uint32_t ce = 0;
                if (threadIdx.x == 0) ce = copy_elems(out + o, d, L);
                o += __shfl_sync(0xFFFFFFFFu, ce, 0);
                i = lit = j + (int)L;
            }
            if (threadIdx.x == 0) {
                s_njobs = nj;
                s_done = done;
            }
        }
        __syncthreads();
        const int nj = s_njobs;
        for (int k = 0; k < nj; ++k) {
            const LitJob jb = s_job[k];
            for (uint32_t q = threadIdx.x; q < jb.len; q += kThreads) out[jb.dst + q] = s_b[jb.src + q];
        }
        const int done = s_done;
        __syncthreads();
        if (done) break;
    }
    if (threadIdx.x == 0) {
        sizes[blockIdx.x] = o;
        atomicAdd(&page_csize[pc[0]], o);
    }
}

// --------------------------------------------------------------------------------------------------------- assembly
// blocks [0, npieces): one piece each; blocks [npieces, ...): heads jobs int64 [nh][3] (blob offset, file offset, bytes)
__global__ void __launch_bounds__(kThreads) k_pq_assemble(const uint8_t* __restrict__ scratch,
                                                          const int64_t* __restrict__ pieces, int64_t npieces,
                                                          const uint32_t* __restrict__ sizes,
                                                          const int64_t* __restrict__ page_first,
                                                          const int64_t* __restrict__ page_dst,
                                                          const uint8_t* __restrict__ heads,
                                                          const int64_t* __restrict__ hjobs, int64_t nh,
                                                          uint8_t* __restrict__ file) {
    if ((int64_t)blockIdx.x < npieces) {
        const int64_t i = blockIdx.x, p = pieces[3 * i];
        __shared__ int64_t s_dst;
        if (threadIdx.x == 0) {
            int64_t d = page_dst[p];
            for (int64_t k = page_first[p]; k < i; ++k) d += sizes[k];
            s_dst = d;
        }
        __syncthreads();
        const uint8_t* s = scratch + i * kPieceCap;
        uint8_t* d = file + s_dst;
        for (uint32_t q = threadIdx.x; q < sizes[i]; q += kThreads) d[q] = s[q];
        return;
    }
    for (int64_t h = blockIdx.x - npieces; h < nh; h += gridDim.x - npieces) {
        const int64_t* j = hjobs + 3 * h;
        for (int64_t q = threadIdx.x; q < j[2]; q += kThreads) file[j[1] + q] = heads[j[0] + q];
    }
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_parquet_split(const uint8_t* rows_dev, int64_t n, int32_t row_bytes, const int32_t* cols_host, int32_t ncols,
                      uint32_t* out_dev, uint32_t* tile_nulls_dev, uint32_t* keys_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_split");
    GSX_REQUIRE(n >= 0 && n <= (1ll << 31), GSX_ERR_ARG, "parquet_split: n=%lld outside 0 .. 2^31", (long long)n);
    GSX_REQUIRE(row_bytes >= 1 && row_bytes <= kRowMax, GSX_ERR_ARG, "parquet_split: rows of %d bytes (1 .. %d)",
                row_bytes, kRowMax);
    GSX_REQUIRE(ncols >= 1 && ncols <= kMaxCols && cols_host, GSX_ERR_ARG, "parquet_split: %d columns (1 .. %d)", ncols,
                kMaxCols);
    int2 cols[kMaxCols];
    for (int c = 0; c < ncols; ++c) {
        const int off = cols_host[2 * c], kind = cols_host[2 * c + 1];
        GSX_REQUIRE((kind == 0 || kind == 1) && off >= 0 && off + (kind ? 1 : 4) <= row_bytes, GSX_ERR_ARG,
                    "parquet_split: column %d (offset %d, kind %d) outside the rows", c, off, kind);
        cols[c] = make_int2(off, kind);
    }
    const int64_t ngroups = n ? (n + kRowGroup - 1) / kRowGroup : 1;
    GSX_CUDA_CHECK(cudaMemsetAsync(keys_dev, 0xFF, (size_t)ncols * ngroups * 4, st));
    GSX_CUDA_CHECK(cudaMemsetAsync(keys_dev + ncols * ngroups, 0, (size_t)ncols * ngroups * 4, st));
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(rows_dev && out_dev && tile_nulls_dev, GSX_ERR_ARG, "parquet_split: null device pointer");
    int2* cols_dev = nullptr;
    GSX_CUDA_CHECK(cudaMallocAsync((void**)&cols_dev, sizeof(int2) * ncols, st));
    GSX_CUDA_CHECK(cudaMemcpyAsync(cols_dev, cols, sizeof(int2) * ncols, cudaMemcpyHostToDevice, st));
    const size_t smem = (size_t)ncols * 12 + 4 + (size_t)ncols * 8 + 16 + (size_t)kStage * row_bytes + 16;
    if (smem > 48 * 1024)
        GSX_CUDA_CHECK(cudaFuncSetAttribute(k_pq_split, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_pq_split<<<(unsigned)((n + kTile - 1) / kTile), kThreads, smem, st>>>(
        rows_dev, n, row_bytes, cols_dev, ncols, out_dev, tile_nulls_dev, keys_dev, keys_dev + ncols * ngroups,
        (int)ngroups);
    GSX_KERNEL_CHECK();
    GSX_CUDA_CHECK(cudaFreeAsync(cols_dev, st));
    return GSX_OK;
}

int gsx_parquet_dict_insert(const uint32_t* cols_dev, int64_t n, int32_t ncols, int32_t g0, int32_t ng,
                            unsigned long long* table_dev, int32_t slots_log2, uint32_t* distinct_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_dict_insert");
    GSX_REQUIRE(n > 0 && n <= (1ll << 31) && ncols >= 1 && ncols <= kMaxCols, GSX_ERR_ARG,
                "parquet_dict_insert: n=%lld, %d columns", (long long)n, ncols);
    const int64_t ngroups = (n + kRowGroup - 1) / kRowGroup;
    GSX_REQUIRE(g0 >= 0 && ng >= 1 && g0 + ng <= ngroups && slots_log2 >= kSlotsMin && slots_log2 <= 24, GSX_ERR_ARG,
                "parquet_dict_insert: row groups %d + %d of %lld, 2^%d slots", g0, ng, (long long)ngroups, slots_log2);
    const int64_t rows = (g0 + ng) * kRowGroup < n ? (int64_t)ng * kRowGroup : n - g0 * kRowGroup;
    k_pq_insert<<<dim3((unsigned)((rows + kThreads - 1) / kThreads), ncols), kThreads, 0, st>>>(
        cols_dev, n, g0, ng, (int)ngroups, table_dev, slots_log2, distinct_dev);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int64_t gsx_parquet_dictionary_workspace_bytes(int64_t nkeys) {
    if (nkeys < 1) nkeys = 1;
    return (int64_t)(2 * align_up((size_t)nkeys * 8, 256) + radix_ws_bytes(nkeys) + 4096);
}

int gsx_parquet_dictionary(unsigned long long* table_dev, int32_t slots_log2, const int64_t* jobs_dev, int32_t njobs,
                           int64_t nkeys, void* ws_dev, int64_t ws_bytes, uint32_t* dict_vals_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_dictionary");
    GSX_REQUIRE(njobs >= 0 && njobs <= 65535 && nkeys >= 0 && slots_log2 >= kSlotsMin && slots_log2 <= 24, GSX_ERR_ARG,
                "parquet_dictionary: %d jobs, %lld keys, 2^%d slots", njobs, (long long)nkeys, slots_log2);
    if (njobs == 0 || nkeys == 0) return GSX_OK;
    GSX_REQUIRE(ws_bytes >= gsx_parquet_dictionary_workspace_bytes(nkeys), GSX_ERR_WORKSPACE,
                "parquet_dictionary: workspace too small");
    Carver cv(ws_dev, (size_t)ws_bytes);
    unsigned long long* k0 = cv.take<unsigned long long>((size_t)nkeys);
    unsigned long long* k1 = cv.take<unsigned long long>((size_t)nkeys);
    unsigned int* fill = cv.take<unsigned int>((size_t)njobs);
    char* rws = cv.take<char>(radix_ws_bytes(nkeys));
    GSX_REQUIRE(cv.ok(), GSX_ERR_WORKSPACE, "parquet_dictionary: workspace too small for %d jobs", njobs);
    GSX_CUDA_CHECK(cudaMemsetAsync(fill, 0, (size_t)njobs * 4, st));
    k_pq_collect<<<dim3(64, njobs), kThreads, 0, st>>>(table_dev, slots_log2, jobs_dev, fill, k0);
    GSX_KERNEL_CHECK();
    int end_bit = 33;
    while ((1ll << (end_bit - 32)) < njobs) ++end_bit;
    uint64_t* sorted = nullptr;
    int rc = radix_sort_keys((uint64_t*)k0, (uint64_t*)k1, nkeys, 0, end_bit, rws, radix_ws_bytes(nkeys), &sorted, st);
    if (rc) return rc;
    k_pq_rank<<<(unsigned)((nkeys + kThreads - 1) / kThreads), kThreads, 0, st>>>(
        table_dev, slots_log2, jobs_dev, (const unsigned long long*)sorted, nkeys, dict_vals_dev);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_parquet_dict_index(uint32_t* cols_dev, int64_t n, int32_t ncols, int32_t g0, int32_t ng,
                           const unsigned long long* table_dev, int32_t slots_log2, const int32_t* dict_chunk_dev,
                           uint32_t* page_idx_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_dict_index");
    GSX_REQUIRE(n > 0 && n <= (1ll << 31) && ncols >= 1 && ncols <= kMaxCols, GSX_ERR_ARG,
                "parquet_dict_index: n=%lld, %d columns", (long long)n, ncols);
    const int64_t ngroups = (n + kRowGroup - 1) / kRowGroup;
    GSX_REQUIRE(g0 >= 0 && ng >= 1 && g0 + ng <= ngroups && slots_log2 >= kSlotsMin && slots_log2 <= 24, GSX_ERR_ARG,
                "parquet_dict_index: row groups %d + %d of %lld, 2^%d slots", g0, ng, (long long)ngroups, slots_log2);
    const int64_t rows = (g0 + ng) * kRowGroup < n ? (int64_t)ng * kRowGroup : n - g0 * kRowGroup;
    k_pq_index<<<dim3((unsigned)((rows + kThreads - 1) / kThreads), ncols), kThreads, 0, st>>>(
        cols_dev, n, g0, ng, table_dev, slots_log2, dict_chunk_dev, page_idx_dev, (n + kPage - 1) / kPage);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_parquet_pages(const uint32_t* cols_dev, int64_t n, int32_t ncols, const uint32_t* tile_nulls_dev,
                      const int64_t* info_dev, const uint32_t* dict_vals_dev, const int64_t* dict_jobs_dev,
                      int32_t ndict, int64_t max_dict, uint32_t* body_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_pages");
    GSX_REQUIRE(n > 0 && n <= (1ll << 31) && ncols >= 1 && ncols <= kMaxCols && ndict >= 0, GSX_ERR_ARG,
                "parquet_pages: n=%lld, %d columns, %d dictionaries", (long long)n, ncols, ndict);
    const int64_t ntiles = (n + kTile - 1) / kTile;
    k_pq_data_pages<<<dim3((unsigned)ntiles, ncols), kThreads, 0, st>>>(cols_dev, n, tile_nulls_dev, ntiles, info_dev,
                                                                      (n + kPage - 1) / kPage, body_dev);
    GSX_KERNEL_CHECK();
    if (ndict) {
        const unsigned gy = (unsigned)(ndict < 65535 ? ndict : 65535);
        k_pq_dict_pages<<<dim3((unsigned)((max_dict + kThreads * 4 - 1) / (kThreads * 4)), gy), kThreads, 0, st>>>(
            dict_vals_dev, dict_jobs_dev, ndict, body_dev);
        GSX_KERNEL_CHECK();
    }
    return GSX_OK;
}

int64_t gsx_parquet_piece_bytes(void) { return kPieceCap; }

int gsx_parquet_snappy(const uint8_t* body_dev, const int64_t* pieces_dev, int64_t npieces, uint8_t* scratch_dev,
                       uint32_t* sizes_dev, uint32_t* page_csize_dev, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_snappy");
    GSX_REQUIRE(npieces >= 0 && npieces < (1ll << 31), GSX_ERR_ARG, "parquet_snappy: %lld pieces", (long long)npieces);
    if (npieces == 0) return GSX_OK;
    GSX_CUDA_CHECK(cudaFuncSetAttribute(k_pq_snappy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSnappySmem));
    k_pq_snappy<<<(unsigned)npieces, kThreads, kSnappySmem, st>>>(body_dev, pieces_dev, scratch_dev, sizes_dev, page_csize_dev);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_parquet_assemble(const uint8_t* scratch_dev, const int64_t* pieces_dev, int64_t npieces,
                         const uint32_t* sizes_dev, const int64_t* page_first_dev, const int64_t* page_dst_dev,
                         const uint8_t* heads_dev, const int64_t* hjobs_dev, int64_t nh, uint8_t* file_dev,
                         void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_parquet_assemble");
    GSX_REQUIRE(npieces >= 0 && nh >= 1 && npieces + 1024 < (1ll << 31), GSX_ERR_ARG,
                "parquet_assemble: %lld pieces, %lld heads", (long long)npieces, (long long)nh);
    const int64_t hb = nh < 1024 ? nh : 1024;
    k_pq_assemble<<<(unsigned)(npieces + hb), kThreads, 0, st>>>(scratch_dev, pieces_dev, npieces, sizes_dev,
                                                                 page_first_dev, page_dst_dev, heads_dev, hjobs_dev, nh,
                                                                 file_dev);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

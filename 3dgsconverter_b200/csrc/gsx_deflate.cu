// gsx_deflate.cu -- raw DEFLATE (RFC 1951) and CRC-32 over a device byte buffer: the body and trailer of the .gz
// files gsx/deflate.py writes.  tests/deflate_oracle.py restates every decision in NumPy, byte for byte.
//
// The caller splits the input into blocks of at most 1 MiB (gsx/deflate.py: at every break offset and every 1 MiB
// inside each span).  Per block, one CTA:
//   k_deflate_plan   histograms of two candidates -- literals only, and literals plus distance-1 copies of the runs
//                    of >= 4 equal bytes -- their length-limited Huffman codes, run-length-coded code lengths and
//                    block headers; keeps the one with fewer bits (literals on a tie) and stores its header bits and
//                    code table in the block's BlockPlan
//   k_deflate_bases  one CTA: exclusive scan of the blocks' bit counts -> 64-bit bit offsets, and the stream's total
//   k_deflate_emit   the block's header, then its tokens tile by tile (a block scan of the bits per thread), each
//                    tile assembled in shared memory; the tile's two edge words are ORed into the zeroed output
//                    (shared with the neighbouring tiles or blocks), the words between them are stored
// Stored blocks (level 0) are k_deflate_stored.  The CRC is k_crc_chunks (the CRC of each 4 KiB chunk, shifted by
// x^(8 * bytes after it) mod P, XORed per CTA) and k_crc_finish (the init / final XOR of zlib's crc32).
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_deflate_format.cuh"

#include <algorithm>
#include <climits>

namespace gsx {
namespace {

constexpr int64_t kDeflateStoredBlock = 65535;
constexpr int kThreads = 512;
constexpr int kPer = 8;                             // consecutive bytes per thread in a tile
constexpr int kTile = kThreads * kPer;              // 4096 bytes
constexpr int kTileWords = kTile * 15 / 32 + 4;     // a literal is <= 15 bits, a copy (>= 3 bytes) <= 35 bits
constexpr int kLitSyms = 286, kDistSyms = 30, kClSyms = 19;
constexpr int kHeadWords = 80;                      // 17 + 19 * 3 + 316 * 7 bits at most
constexpr int kMaxCopy = 258;
constexpr int64_t kCrcChunk = 4096;
constexpr int kCrcParts = 1024;
constexpr uint32_t kPoly = 0xEDB88320u;

struct BlockPlan {
    uint32_t lit[kLitSyms];     // bit-reversed code | length << 16
    uint32_t dist[kDistSyms];
    uint32_t head[kHeadWords];  // the block header, LSB-first
    uint32_t head_bits, copies;
    unsigned long long bits;    // header + data + end-of-block
    unsigned long long base;    // bit offset of the block in the output words
};

struct MaxOp {
    template <typename T> __device__ T operator()(T a, T b) const { return a > b ? a : b; }
};
struct MinOp {
    template <typename T> __device__ T operator()(T a, T b) const { return a < b ? a : b; }
};
struct AddOp {
    template <typename T> __device__ T operator()(T a, T b) const { return a + b; }
};

// exclusive scan over the CTA's threads in thread order (REV: from the last thread down); `total` over all threads
template <bool REV, typename T, typename Op>
__device__ __forceinline__ T block_scan(T v, T ident, Op op, T* sh, T& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = REV ? __shfl_down_sync(0xFFFFFFFFu, x, o) : __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (REV ? lane + o < 32 : lane >= o) x = op(x, y);
    }
    if (lane == (REV ? 0 : 31)) sh[warp] = x;
    T prev = REV ? __shfl_down_sync(0xFFFFFFFFu, x, 1) : __shfl_up_sync(0xFFFFFFFFu, x, 1);
    if (lane == (REV ? 31 : 0)) prev = ident;
    __syncthreads();
    T w = ident, t = ident;
    for (int k = 0; k < kThreads / 32; ++k) {
        const T s = sh[k];
        if (REV ? k > warp : k < warp) w = op(w, s);
        t = op(t, s);
    }
    __syncthreads();
    total = t;
    return op(w, prev);
}

// ORs the bits of v at bit o of words (up to three words; bits past nwords are dropped)
template <bool SHARED>
__device__ __forceinline__ void or_bits(uint32_t* words, int64_t nwords, uint64_t o, uint64_t v) {
    const int64_t w = int64_t(o >> 5);
    const uint32_t sh = uint32_t(o & 31);
    const uint64_t rest = v >> (32 - sh);
    const uint32_t part[3] = {uint32_t(v << sh), uint32_t(rest), uint32_t(rest >> 32)};
#pragma unroll
    for (int k = 0; k < 3; ++k)
        if (part[k] && (SHARED || w + k < nwords)) atomicOr(&words[w + k], part[k]);
}

struct HuffScratch {
    uint64_t w[2 * kLitSyms];   // leaf weights by symbol, then the joined nodes' by creation
    uint16_t order[kLitSyms];   // the used symbols by (weight, symbol)
    uint16_t parent[2 * kLitSyms];
    uint16_t depth[2 * kLitSyms];
    uint64_t floor;
    int done;
};

// Code lengths of cnt[0..m), none above `limit` (the whole CTA calls this): join the two lightest nodes by
// (weight, id) -- the merge of the leaves sorted by (weight, symbol) with the joined nodes in creation order pops the
// same nodes as a heap -- and while a length exceeds the limit, raise every used weight to a floor of 1, 2, 4, ...
// A lone used symbol gets length 1.
__device__ void huffman(const uint32_t* cnt, int m, int limit, uint8_t* len, HuffScratch& h) {
    if (threadIdx.x == 0) h.floor = 1, h.done = 0;
    for (int i = threadIdx.x; i < m; i += kThreads) len[i] = 0;
    __syncthreads();
    for (;;) {
        for (int i = threadIdx.x; i < m; i += kThreads) h.w[i] = cnt[i] ? max(uint64_t(cnt[i]), h.floor) : 0;
        __syncthreads();
        for (int i = threadIdx.x; i < m; i += kThreads) {
            if (!cnt[i]) continue;
            const uint64_t wi = h.w[i];
            int r = 0;
            for (int j = 0; j < m; ++j) r += cnt[j] && (h.w[j] < wi || (h.w[j] == wi && j < i));
            h.order[r] = uint16_t(i);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int nu = 0;
            for (int i = 0; i < m; ++i) nu += cnt[i] != 0;
            if (nu <= 1) {
                if (nu == 1) len[h.order[0]] = 1;
                h.done = 1;
            } else {
                int li = 0, ih = 0;
                for (int k = 0; k < nu - 1; ++k) {
                    int pick[2];
                    for (int t = 0; t < 2; ++t)
                        pick[t] = li < nu && (ih == k || h.w[h.order[li]] <= h.w[m + ih]) ? h.order[li++] : m + ih++;
                    h.w[m + k] = h.w[pick[0]] + h.w[pick[1]];
                    h.parent[pick[0]] = h.parent[pick[1]] = uint16_t(m + k);
                }
                h.depth[m + nu - 2] = 0;
                for (int k = nu - 3; k >= 0; --k) h.depth[m + k] = h.depth[h.parent[m + k]] + 1;
                int deepest = 0;
                for (int k = 0; k < nu; ++k) deepest = max(deepest, h.depth[h.parent[h.order[k]]] + 1);
                if (deepest <= limit) {
                    for (int k = 0; k < nu; ++k) len[h.order[k]] = uint8_t(h.depth[h.parent[h.order[k]]] + 1);
                    h.done = 1;
                } else {
                    h.floor *= 2;
                }
            }
        }
        __syncthreads();
        if (h.done) break;
    }
    __syncthreads();
}

// canonical codes (by length, then symbol), bit-reversed for the LSB-first stream: code | length << 16
__device__ void canonical(const uint8_t* len, int m, uint32_t* table) {
    int count[16] = {0};
    for (int s = 0; s < m; ++s) count[len[s]]++;
    count[0] = 0;
    uint32_t next[16], code = 0;
    for (int b = 1; b < 16; ++b) next[b] = code = (code + count[b - 1]) << 1;
    for (int s = 0; s < m; ++s) {
        const uint32_t l = len[s];
        table[s] = l ? (__brev(next[l]++) >> (32 - l)) | (l << 16) : 0u;
    }
}

// the code lengths of one block, HLIT then HDIST of them, run-length coded: 16 = repeat the previous 3..6 times,
// 17 = 3..10 zeros, 18 = 11..138 zeros, greedy from the left
__device__ int rle(const uint8_t* lit, int hlit, const uint8_t* dist, int hdist, uint8_t* sym, uint8_t* ext) {
    const int N = hlit + hdist;
    auto at = [&](int i) { return i < hlit ? lit[i] : dist[i - hlit]; };
    int i = 0, k = 0;
    while (i < N) {
        const int v = at(i);
        int r = 1;
        while (i + r < N && at(i + r) == v) ++r;
        if (v == 0) {
            const int c = r >= 11 ? min(r, 138) : r >= 3 ? r : 1;
            sym[k] = c >= 11 ? 18 : c >= 3 ? 17 : 0;
            ext[k++] = uint8_t(c >= 11 ? c - 11 : c >= 3 ? c - 3 : 0);
            i += c;
        } else {
            sym[k] = uint8_t(v), ext[k++] = 0;
            ++i;
            for (int rem = r - 1; rem >= 3;) {
                const int c = min(rem, 6);
                sym[k] = 16, ext[k++] = uint8_t(c - 3);
                i += c, rem -= c;
            }
        }
    }
    return k;
}

__device__ __forceinline__ int rle_extra_bits(int sym) { return sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0; }

__device__ __forceinline__ int trimmed(const uint8_t* len, int m, int least) {
    int t = least;
    for (int s = 0; s < m; ++s)
        if (len[s]) t = max(t, s + 1);
    return t;
}

__device__ __forceinline__ int hclen_of(const uint8_t* cl) {
    int t = 4;
    for (int i = 0; i < kClSyms; ++i)
        if (cl[kClOrder[i]]) t = max(t, i + 1);
    return t;
}

// the run starts of one thread's kPer bytes of the tile at t0 (len bytes in tb, tb[len] the next byte when inside
// the block); carry_s is the start of the run holding the byte before t0.  Returns the last run start in the tile.
__device__ __forceinline__ long long tile_starts(const uint8_t* tb, int64_t t0, int len, int64_t b0, uint8_t prev_last,
                                                 long long carry_s, long long* sh, long long* S) {
    const int base = threadIdx.x * kPer;
    long long lb = -1;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
        if (base + j >= len) break;
        const int64_t p = t0 + base + j;
        const uint8_t before = base + j ? tb[base + j - 1] : prev_last;
        if (p == b0 || tb[base + j] != before) lb = p;
    }
    long long last;
    long long s = max(block_scan<false>(lb, -1LL, MaxOp(), sh, last), carry_s);
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
        if (base + j >= len) break;
        const int64_t p = t0 + base + j;
        const uint8_t before = base + j ? tb[base + j - 1] : prev_last;
        if (p == b0 || tb[base + j] != before) s = p;
        S[j] = s;
    }
    return max(last, carry_s);
}

__device__ __forceinline__ bool run_end_at(const uint8_t* tb, int k, int64_t p, int64_t b1) {
    return p == b1 - 1 || tb[k + 1] != tb[k];
}

// the first position in [q, b1) whose byte is not v, or b1 (the whole CTA calls this)
__device__ long long run_end_after(const uint8_t* d, int64_t q, int64_t b1, uint8_t v, long long* sh) {
    for (; q < b1; q += kTile) {
        long long f = LLONG_MAX;
        const int64_t hi = min(q + kTile, b1);
        for (int64_t x = q + threadIdx.x; x < hi; x += kThreads)
            if (d[x] != v) {
                f = x;
                break;
            }
        long long first;
        block_scan<false>(f, LLONG_MAX, MinOp(), sh, first);
        if (first != LLONG_MAX) return first;
    }
    return b1;
}

__device__ __forceinline__ void load_tile(const uint8_t* d, int64_t t0, int len, int64_t b1, uint8_t* tb) {
    const int m = len + (t0 + len < b1);
    for (int k = threadIdx.x; k < m; k += kThreads) tb[k] = d[t0 + k];
}

__global__ void __launch_bounds__(kThreads) k_deflate_plan(const uint8_t* __restrict__ d, int64_t n,
                                                           const int64_t* __restrict__ starts, int64_t nblocks,
                                                           BlockPlan* __restrict__ plans) {
    __shared__ uint8_t tb[kTile + 1];
    __shared__ uint32_t lit[256], covered[256], lenc[kLitSyms - 257];
    __shared__ uint32_t ncopies, xbits;
    __shared__ long long sh[kThreads / 32];
    __shared__ uint32_t cnt[2][kLitSyms], dcnt[kDistSyms], clcnt[2][kClSyms];
    __shared__ uint8_t len[2][kLitSyms], dlen[2][kDistSyms], cllen[2][kClSyms];
    __shared__ uint8_t rsym[2][kLitSyms + kDistSyms], rext[2][kLitSyms + kDistSyms];
    __shared__ int nrle[2], hlit[2], hdist[2];
    __shared__ HuffScratch hs;
    const int64_t b = blockIdx.x;
    const int64_t b0 = starts[b], b1 = b + 1 < nblocks ? starts[b + 1] : n;
    for (int k = threadIdx.x; k < 256; k += kThreads) lit[k] = covered[k] = 0;
    for (int k = threadIdx.x; k < kLitSyms - 257; k += kThreads) lenc[k] = 0;
    if (threadIdx.x == 0) ncopies = xbits = 0;
    long long carry_s = b0;
    uint8_t prev_last = 0;
    const int base = threadIdx.x * kPer;
    for (int64_t t0 = b0; t0 < b1; t0 += kTile) {
        const int len_t = int(min(int64_t(kTile), b1 - t0));
        __syncthreads();
        load_tile(d, t0, len_t, b1, tb);
        __syncthreads();
        long long S[kPer];
        const long long next_s = tile_starts(tb, t0, len_t, b0, prev_last, carry_s, sh, S);
        uint32_t acc = 0;
        int accv = -1;
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            if (base + j >= len_t) break;
            const int64_t p = t0 + base + j;
            const uint32_t v = tb[base + j];
            if (int(v) != accv) {
                if (acc) atomicAdd(&lit[accv], acc);
                accv = int(v), acc = 0;
            }
            ++acc;
            if (!run_end_at(tb, base + j, p, b1)) continue;
            const int64_t r = p + 1 - S[j];
            if (r < 4) continue;
            const uint32_t full = uint32_t((r - 1) / kMaxCopy), rem = uint32_t((r - 1) % kMaxCopy);
            atomicAdd(&covered[v], uint32_t(r - 1) - (rem < 3 ? rem : 0));
            if (full) atomicAdd(&lenc[285 - 257], full);
            if (rem >= 3) {
                uint32_t sym, nx, ex;
                length_code(rem, sym, nx, ex);
                atomicAdd(&lenc[sym - 257], 1u);
                if (nx) atomicAdd(&xbits, nx);
            }
            atomicAdd(&ncopies, full + (rem >= 3));
        }
        if (acc) atomicAdd(&lit[accv], acc);
        carry_s = next_s;
        prev_last = tb[len_t - 1];
    }
    __syncthreads();
    const bool copies = ncopies != 0;
    for (int s = threadIdx.x; s < kLitSyms; s += kThreads) {
        cnt[0][s] = s < 256 ? lit[s] : s == 256 ? 1u : 0u;
        cnt[1][s] = s < 256 ? lit[s] - covered[s] : s == 256 ? 1u : lenc[s - 257];
    }
    for (int s = threadIdx.x; s < kDistSyms; s += kThreads) {
        dcnt[s] = s == 0 ? ncopies : 0u;
        dlen[0][s] = 0;
    }
    __syncthreads();
    huffman(cnt[0], kLitSyms, 15, len[0], hs);
    if (copies) {
        huffman(cnt[1], kLitSyms, 15, len[1], hs);
        huffman(dcnt, kDistSyms, 15, dlen[1], hs);
    }
    const int ncand = copies ? 2 : 1;
    if (threadIdx.x == 0) {
        for (int c = 0; c < ncand; ++c) {
            hlit[c] = trimmed(len[c], kLitSyms, 257);
            hdist[c] = trimmed(dlen[c], kDistSyms, 1);
            nrle[c] = rle(len[c], hlit[c], dlen[c], hdist[c], rsym[c], rext[c]);
            for (int s = 0; s < kClSyms; ++s) clcnt[c][s] = 0;
            for (int k = 0; k < nrle[c]; ++k) clcnt[c][rsym[c][k]]++;
        }
    }
    __syncthreads();
    for (int c = 0; c < ncand; ++c) huffman(clcnt[c], kClSyms, 7, cllen[c], hs);
    if (threadIdx.x != 0) return;
    unsigned long long cost[2] = {0, 0};
    for (int c = 0; c < ncand; ++c) {
        unsigned long long bits = 17 + 3 * hclen_of(cllen[c]);
        for (int k = 0; k < nrle[c]; ++k) bits += cllen[c][rsym[c][k]] + rle_extra_bits(rsym[c][k]);
        for (int s = 0; s < kLitSyms; ++s) bits += (unsigned long long)cnt[c][s] * len[c][s];
        if (c == 1) bits += (unsigned long long)ncopies * dlen[1][0] + xbits;
        cost[c] = bits;
    }
    const int c = copies && cost[1] < cost[0] ? 1 : 0;
    BlockPlan& P = plans[b];
    P.copies = c;
    P.bits = cost[c];
    canonical(len[c], kLitSyms, P.lit);
    canonical(dlen[c], kDistSyms, P.dist);
    uint32_t clcode[kClSyms];
    canonical(cllen[c], kClSyms, clcode);
    uint64_t acc = 0;
    int na = 0, nw = 0;
    uint32_t total = 0;
    auto put = [&](uint32_t v, int nbits) {
        acc |= uint64_t(v) << na;
        na += nbits, total += nbits;
        for (; na >= 32; na -= 32, acc >>= 32) P.head[nw++] = uint32_t(acc);
    };
    put(b == nblocks - 1, 1);
    put(2, 2);
    put(hlit[c] - 257, 5);
    put(hdist[c] - 1, 5);
    const int ncl = hclen_of(cllen[c]);
    put(ncl - 4, 4);
    for (int i = 0; i < ncl; ++i) put(cllen[c][kClOrder[i]], 3);
    for (int k = 0; k < nrle[c]; ++k) {
        const int s = rsym[c][k];
        put(clcode[s] & 0xFFFF, clcode[s] >> 16);
        put(rext[c][k], rle_extra_bits(s));
    }
    if (na) P.head[nw++] = uint32_t(acc);
    P.head_bits = total;
}

__global__ void __launch_bounds__(kThreads) k_deflate_bases(BlockPlan* __restrict__ plans, int64_t nblocks,
                                                            uint64_t bit_offset, unsigned long long* __restrict__ total) {
    __shared__ unsigned long long sh[kThreads / 32];
    const int64_t per = (nblocks + kThreads - 1) / kThreads;
    const int64_t lo = min(nblocks, threadIdx.x * per), hi = min(nblocks, lo + per);
    unsigned long long s = 0;
    for (int64_t i = lo; i < hi; ++i) s += plans[i].bits;
    unsigned long long all;
    unsigned long long at = block_scan<false>(s, 0ull, AddOp(), sh, all) + bit_offset;
    for (int64_t i = lo; i < hi; ++i) {
        plans[i].base = at;
        at += plans[i].bits;
    }
    if (threadIdx.x == 0) *total = all;
}

__global__ void __launch_bounds__(kThreads) k_deflate_emit(const uint8_t* __restrict__ d, int64_t n,
                                                           const int64_t* __restrict__ starts, int64_t nblocks,
                                                           const BlockPlan* __restrict__ plans,
                                                           uint32_t* __restrict__ out, int64_t nwords,
                                                           unsigned long long* __restrict__ mismatches) {
    __shared__ uint8_t tb[kTile + 1];
    __shared__ uint32_t ob[kTileWords];
    __shared__ uint32_t lit[kLitSyms];
    __shared__ long long sh[kThreads / 32];
    __shared__ uint32_t shu[kThreads / 32];
    const int64_t b = blockIdx.x;
    const BlockPlan& P = plans[b];
    const int64_t b0 = starts[b], b1 = b + 1 < nblocks ? starts[b + 1] : n;
    for (int k = threadIdx.x; k < kLitSyms; k += kThreads) lit[k] = P.lit[k];
    const uint32_t dist = P.dist[0], head_bits = P.head_bits;
    const bool copies = P.copies;
    for (uint32_t w = threadIdx.x; w * 32 < head_bits; w += kThreads)
        or_bits<false>(out, nwords, P.base + 32 * uint64_t(w), P.head[w]);
    uint64_t pos = P.base + head_bits;
    long long carry_s = b0, e_cache = b0;
    uint8_t prev_last = 0;
    const int base = threadIdx.x * kPer;
    for (int64_t t0 = b0; t0 < b1; t0 += kTile) {
        const int len_t = int(min(int64_t(kTile), b1 - t0));
        __syncthreads();
        load_tile(d, t0, len_t, b1, tb);
        for (int k = threadIdx.x; k < kTileWords; k += kThreads) ob[k] = 0;
        __syncthreads();
        uint64_t v[kPer];
        uint32_t nb[kPer], mine = 0;
        if (!copies) {
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const uint32_t e = base + j < len_t ? lit[tb[base + j]] : 0u;
                v[j] = e & 0xFFFF, nb[j] = e >> 16, mine += nb[j];
            }
        } else {
            long long S[kPer], E[kPer];
            const long long next_s = tile_starts(tb, t0, len_t, b0, prev_last, carry_s, sh, S);
            long long first_end = LLONG_MAX;
#pragma unroll
            for (int j = kPer - 1; j >= 0; --j)
                if (base + j < len_t && run_end_at(tb, base + j, t0 + base + j, b1)) first_end = t0 + base + j + 1;
            long long unused;
            long long e = block_scan<true>(first_end, LLONG_MAX, MinOp(), sh, unused);
            const int64_t last = t0 + len_t - 1;
            if (!run_end_at(tb, len_t - 1, last, b1)) {   // the tile's last run goes on past the tile
                if (e_cache <= last) e_cache = run_end_after(d, last + 1, b1, tb[len_t - 1], sh);
                e = min(e, e_cache);
            }
#pragma unroll
            for (int j = kPer - 1; j >= 0; --j) {
                if (base + j >= len_t) continue;
                if (run_end_at(tb, base + j, t0 + base + j, b1)) e = t0 + base + j + 1;
                E[j] = e;
            }
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                v[j] = 0, nb[j] = 0;
                if (base + j >= len_t) continue;
                const int64_t p = t0 + base + j;
                const int64_t r = E[j] - S[j], k = p - S[j];
                uint32_t L = 0;   // 0: a literal, 1: inside a copy, else the length of the copy starting here
                if (r >= 4 && k > 0) {
                    const int64_t q = (k - 1) / kMaxCopy, jj = (k - 1) % kMaxCopy;
                    const int64_t full = (r - 1) / kMaxCopy, rem = (r - 1) % kMaxCopy;
                    if (q < full) L = jj ? 1 : kMaxCopy;
                    else if (rem >= 3) L = jj ? 1 : uint32_t(rem);
                }
                if (L == 0) {
                    const uint32_t t = lit[tb[base + j]];
                    v[j] = t & 0xFFFF, nb[j] = t >> 16;
                } else if (L > 1) {
                    uint32_t sym, nx, ex;
                    length_code(L, sym, nx, ex);
                    const uint32_t t = lit[sym], lt = t >> 16;
                    v[j] = (t & 0xFFFF) | (uint64_t(ex) << lt) | (uint64_t(dist & 0xFFFF) << (lt + nx));
                    nb[j] = lt + nx + (dist >> 16);
                }
                mine += nb[j];
            }
            carry_s = next_s;
        }
        uint32_t tile_bits;
        const uint32_t sh0 = uint32_t(pos & 31);
        uint64_t o = sh0 + block_scan<false>(mine, 0u, AddOp(), shu, tile_bits);
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
            if (nb[j]) or_bits<true>(ob, kTileWords, o, v[j]);
            o += nb[j];
        }
        __syncthreads();
        const int64_t w0 = int64_t(pos >> 5);
        const int nw = int((sh0 + tile_bits + 31) / 32);
        for (int k = threadIdx.x; k < nw; k += kThreads) {
            const int64_t gw = w0 + k;
            if (gw >= nwords) continue;
            if (k == 0 || k == nw - 1) {
                if (ob[k]) atomicOr(&out[gw], ob[k]);
            } else {
                out[gw] = ob[k];
            }
        }
        pos += tile_bits;
        prev_last = tb[len_t - 1];
    }
    if (threadIdx.x == 0) {
        const uint32_t eob = lit[256];
        or_bits<false>(out, nwords, pos, eob & 0xFFFF);
        if (pos + (eob >> 16) != P.base + P.bits) atomicAdd(mismatches, 1ull);
    }
}

__global__ void k_deflate_stored(const uint8_t* __restrict__ d, int64_t n, int64_t nb, uint8_t* __restrict__ out) {
    for (int64_t k = blockIdx.x; k < nb; k += gridDim.x) {
        const int64_t at = k * kDeflateStoredBlock;
        const uint32_t len = uint32_t(min(kDeflateStoredBlock, n - at));
        uint8_t* o = out + k * (kDeflateStoredBlock + 5);
        if (threadIdx.x == 0) {
            o[0] = k == nb - 1;
            o[1] = len & 0xFF, o[2] = len >> 8, o[3] = ~len & 0xFF, o[4] = (~len >> 8) & 0xFF;
        }
        for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) o[5 + i] = d[at + i];
    }
}

// ------------------------------------------------------------------------------------------------------- CRC-32
// zlib's representation: bit 31 is x^0.  multmodp(a, b) = a * b mod P; x2n[k] = x^(2^k) mod P.
struct CrcPowers {
    uint32_t x2n[64];
};

__host__ __device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; ++i) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = b & 1 ? (b >> 1) ^ kPoly : b >> 1;
    }
    return p;
}

// x^(8 * nbytes) mod P
__host__ __device__ __forceinline__ uint32_t x8nmodp(uint64_t nbytes, const CrcPowers& pw) {
    uint32_t p = 0x80000000u;
    for (int k = 3; nbytes; nbytes >>= 1, ++k)
        if (nbytes & 1) p = multmodp(pw.x2n[k], p);
    return p;
}

const CrcPowers& crc_powers() {
    static const CrcPowers pw = [] {
        CrcPowers q;
        q.x2n[0] = 0x40000000u;   // x^1
        for (int k = 1; k < 64; ++k) q.x2n[k] = multmodp(q.x2n[k - 1], q.x2n[k - 1]);
        return q;
    }();
    return pw;
}

__global__ void __launch_bounds__(256) k_crc_chunks(const uint8_t* __restrict__ d, int64_t n, CrcPowers pw,
                                                    uint32_t* __restrict__ partial) {
    __shared__ uint32_t T[4][256];
    __shared__ uint32_t red[8];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i;
        for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ kPoly : c >> 1;
        T[0][i] = c;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        for (int t = 1; t < 4; ++t) T[t][i] = (T[t - 1][i] >> 8) ^ T[0][T[t - 1][i] & 0xFF];
    __syncthreads();
    auto word = [&](uint32_t c) {
        return T[3][c & 0xFF] ^ T[2][(c >> 8) & 0xFF] ^ T[1][(c >> 16) & 0xFF] ^ T[0][c >> 24];
    };
    const bool aligned = (reinterpret_cast<uintptr_t>(d) & 15) == 0;
    const int64_t nchunks = (n + kCrcChunk - 1) / kCrcChunk;
    uint32_t acc = 0;
    for (int64_t c = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; c < nchunks; c += int64_t(gridDim.x) * blockDim.x) {
        const uint8_t* p = d + c * kCrcChunk;
        const int64_t len = min(kCrcChunk, n - c * kCrcChunk);
        uint32_t crc = 0;
        int64_t i = 0;
        if (aligned)
            for (; i + 16 <= len; i += 16) {
                const uint4 q = __ldg(reinterpret_cast<const uint4*>(p + i));
                crc = word(crc ^ q.x);
                crc = word(crc ^ q.y);
                crc = word(crc ^ q.z);
                crc = word(crc ^ q.w);
            }
        for (; i < len; ++i) crc = T[0][(crc ^ p[i]) & 0xFF] ^ (crc >> 8);
        acc ^= multmodp(x8nmodp(uint64_t(n - c * kCrcChunk - len), pw), crc);
    }
    for (int o = 16; o; o >>= 1) acc ^= __shfl_down_sync(0xFFFFFFFFu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t x = 0;
        for (int w = 0; w < int(blockDim.x / 32); ++w) x ^= red[w];
        partial[blockIdx.x] = x;
    }
}

__global__ void k_crc_finish(const uint32_t* __restrict__ partial, int nparts, int64_t n, CrcPowers pw,
                             uint8_t* __restrict__ trailer) {
    if (threadIdx.x != 0) return;
    uint32_t x = 0;
    for (int i = 0; i < nparts; ++i) x ^= partial[i];
    const uint32_t crc = x ^ multmodp(x8nmodp(uint64_t(n), pw), 0xFFFFFFFFu) ^ 0xFFFFFFFFu;
    const uint32_t isize = uint32_t(uint64_t(n) & 0xFFFFFFFFu);
    for (int k = 0; k < 4; ++k) trailer[k] = uint8_t(crc >> (8 * k)), trailer[4 + k] = uint8_t(isize >> (8 * k));
}

struct Layout {
    uint32_t* partial;
    BlockPlan* plans;
};

bool carve(Carver& cv, int64_t nblocks, Layout& L) {
    L.partial = cv.take<uint32_t>(kCrcParts);
    L.plans = cv.take<BlockPlan>(size_t(std::max<int64_t>(nblocks, 0)));
    return cv.ok();
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_deflate_workspace_bytes(int64_t nblocks) {
    if (nblocks < 0) return 0;
    Carver cv(nullptr, 0);
    Layout L;
    carve(cv, nblocks, L);
    return int64_t(cv.off) + 256;
}

int gsx_crc32(const uint8_t* data, int64_t n, void* ws, int64_t ws_bytes, uint8_t* trailer, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_crc32");
    GSX_REQUIRE(n >= 0 && (data || n == 0) && ws && trailer, GSX_ERR_ARG, "crc32: bad arguments");
    Carver cv(ws, size_t(ws_bytes));
    Layout L;
    GSX_REQUIRE(carve(cv, 0, L), GSX_ERR_WORKSPACE, "crc32: workspace too small");
    const int64_t nchunks = (n + kCrcChunk - 1) / kCrcChunk;
    const int parts = int(std::max<int64_t>(1, std::min<int64_t>((nchunks + 255) / 256, kCrcParts)));
    const CrcPowers& pw = crc_powers();
    k_crc_chunks<<<parts, 256, 0, st>>>(data, n, pw, L.partial);
    GSX_KERNEL_CHECK();
    k_crc_finish<<<1, 32, 0, st>>>(L.partial, parts, n, pw, trailer);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_deflate_stored(const uint8_t* data, int64_t n, uint8_t* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_deflate_stored");
    GSX_REQUIRE(n >= 0 && (data || n == 0) && out, GSX_ERR_ARG, "deflate_stored: bad arguments");
    const int64_t nb = std::max<int64_t>(1, (n + kDeflateStoredBlock - 1) / kDeflateStoredBlock);
    const int grid = int(std::min<int64_t>(nb, int64_t(sm_count()) * 16));
    k_deflate_stored<<<grid, 256, 0, st>>>(data, n, nb, out);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_deflate_plan(const uint8_t* data, int64_t n, const int64_t* starts, int64_t nblocks, void* ws, int64_t ws_bytes,
                     uint64_t bit_offset, unsigned long long* total_bits, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_deflate_plan");
    GSX_REQUIRE(n >= 0 && (data || n == 0) && starts && ws && total_bits, GSX_ERR_ARG, "deflate_plan: bad arguments");
    GSX_REQUIRE(nblocks >= 1 && nblocks < (int64_t(1) << 31), GSX_ERR_ARG,
                "deflate_plan: nblocks must be 1..2^31-1 (got %lld)", (long long)nblocks);
    Carver cv(ws, size_t(ws_bytes));
    Layout L;
    GSX_REQUIRE(carve(cv, nblocks, L), GSX_ERR_WORKSPACE, "deflate_plan: workspace too small");
    k_deflate_plan<<<unsigned(nblocks), kThreads, 0, st>>>(data, n, starts, nblocks, L.plans);
    GSX_KERNEL_CHECK();
    k_deflate_bases<<<1, kThreads, 0, st>>>(L.plans, nblocks, bit_offset, total_bits);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_deflate_emit(const uint8_t* data, int64_t n, const int64_t* starts, int64_t nblocks, void* ws, int64_t ws_bytes,
                     uint32_t* words, int64_t nwords, unsigned long long* mismatches, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_deflate_emit");
    GSX_REQUIRE(n >= 0 && (data || n == 0) && starts && ws && words && mismatches, GSX_ERR_ARG,
                "deflate_emit: bad arguments");
    GSX_REQUIRE(nblocks >= 1 && nblocks < (int64_t(1) << 31), GSX_ERR_ARG,
                "deflate_emit: nblocks must be 1..2^31-1 (got %lld)", (long long)nblocks);
    Carver cv(ws, size_t(ws_bytes));
    Layout L;
    GSX_REQUIRE(carve(cv, nblocks, L), GSX_ERR_WORKSPACE, "deflate_emit: workspace too small");
    k_deflate_emit<<<unsigned(nblocks), kThreads, 0, st>>>(data, n, starts, nblocks, L.plans, words, nwords,
                                                             mismatches);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

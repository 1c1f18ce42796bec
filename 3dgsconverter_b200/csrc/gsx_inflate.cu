// gsx_inflate.cu -- raw DEFLATE (RFC 1951) decoding of a device byte buffer in parallel: the body of each gzip member
// gsx/deflate.py's gunzip reads.  tests/inflate_model.py restates every stage in Python.
//
// A DEFLATE stream has no index, so the body is cut into chunks of compressed bits and each chunk is decoded
// speculatively; the host walks the chain and re-decodes where a guess was wrong.  Per job, one thread:
//   k_inflate_run      with FIND, the first plausible block start in the chunk's span of bits (a dynamic block whose
//                      header passes zlib's checks and whose trial decode reaches its end-of-block, or a stored block
//                      with zero padding and LEN = ~NLEN, not one inside the byte before another); then decodes blocks from that start until one ends at or past
//                      the job's target bit, or the final block ends.  Output is 16-bit symbols in the workspace: a
//                      byte, or kMark | w, byte w of the 32 KiB window before the start, unknown until the chain is
//                      known.  A job at a member's start has no window: a distance past its first byte is an error.
// Then over the verified chain's pieces, each at its output offset (an exclusive scan of their lengths):
//   k_inflate_bytes    every byte symbol to the output, in parallel
//   k_inflate_window   one CTA, the pieces in chain order: the markers of each piece's last 32 KiB (the next piece's
//                      window), from the first position there to its last marker
//   k_inflate_markers  every other marker, in parallel (every window is final by then)
// A marker that lands before the member's first byte is zlib's "invalid distance too far back".
#include "../../include/gsx.h"

#include "gsx_bits.cuh"
#include "gsx_common.cuh"
#include "gsx_deflate_format.cuh"

#include <algorithm>

namespace gsx {
namespace {

constexpr int kWindow = 32768;
constexpr uint16_t kMark = 0x8000;
constexpr int kLitFast = 10, kDistFast = 8;
constexpr int kRunThreads = 64;
enum : int64_t { kOk = 0, kFinal = 1, kEof = 2, kData = 3, kOverflow = 4, kNone = 5, kBadJob = 6 };
enum : int64_t { kFind = 1, kFirst = 2 };

// Canonical Huffman code: counts and symbols sorted by (length, symbol), and a FAST-bit table of the codes that fit
// (symbol | length << 9; 0 = look further).
template <int NSYM, int FAST>
struct Huff {
    uint16_t count[16];
    uint16_t sym[NSYM];
    uint16_t fast[1 << FAST];
    int max;
    bool over, incomplete;

    __device__ void build(const uint8_t* len, int n) {
        for (int i = 0; i < 16; ++i) count[i] = 0;
        for (int i = 0; i < n; ++i) ++count[len[i]];
        count[0] = 0;
        max = 0;
        int left = 1;
        over = false;
        for (int b = 1; b < 16; ++b) {
            if (count[b]) max = b;
            left = 2 * left - count[b];
            if (left < 0) over = true;
        }
        incomplete = !over && left > 0;
        if (over || (incomplete && max > 1)) return;   // no set zlib accepts: the caller refuses it, no table needed
        uint16_t offs[16], code[16];
        offs[1] = 0, code[1] = 0;
        for (int b = 1; b < 15; ++b) offs[b + 1] = offs[b] + count[b], code[b + 1] = (code[b] + count[b]) << 1;
        for (int i = 0; i < (1 << FAST); ++i) fast[i] = 0;
        for (int s = 0; s < n; ++s) {
            const int b = len[s];
            if (!b) continue;
            sym[offs[b]++] = uint16_t(s);
            const uint32_t c = code[b]++;
            if (b > FAST) continue;
            const uint32_t rev = __brev(c) >> (32 - b);
            for (uint32_t r = rev; r < (1u << FAST); r += 1u << b) fast[r] = uint16_t(s | b << 9);
        }
    }

    // kOk with the symbol, kEof when the input ends inside the code, kData for a code the set does not have (zlib
    // reads max(1, longest length) bits of such a code)
    __device__ __forceinline__ int64_t decode(Reader& r, int& out) const {
        if (r.need(FAST)) {
            const uint16_t e = fast[r.peek(FAST)];
            if (e) {
                r.drop(e >> 9);
                out = e & 511;
                return kOk;
            }
        }
        int code = 0, first = 0, index = 0;
        for (int b = 1; b < 16; ++b) {
            if (!r.need(b)) return kEof;
            code |= int((r.buf >> (b - 1)) & 1);
            const int c = count[b];
            if (code - c < first) {
                r.drop(b);
                out = sym[index + code - first];
                return kOk;
            }
            if (b >= max) return kData;
            index += c;
            first = (first + c) << 1;
            code <<= 1;
        }
        return kData;
    }
};

struct Codes {
    Huff<19, 7> cl;
    Huff<288, kLitFast> lit;
    Huff<32, kDistFast> dist;
    uint8_t lens[316];   // literal/length then distance code lengths
};

__device__ int64_t fixed_codes(Codes& c) {
    for (int i = 0; i < 288; ++i) c.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
    c.lit.build(c.lens, 288);
    for (int i = 0; i < 32; ++i) c.lens[i] = 5;
    c.dist.build(c.lens, 32);
    return kOk;
}

// A dynamic block's header after BTYPE, with zlib's checks in zlib's order.
__device__ int64_t dynamic_codes(Reader& r, Codes& c) {
    if (!r.need(14)) return kEof;
    const int nlen = int(r.peek(5)) + 257, ndist = int((r.buf >> 5) & 31) + 1, ncode = int((r.buf >> 10) & 15) + 4;
    r.drop(14);
    if (nlen > 286 || ndist > 30) return kData;
    uint8_t cl[19];
    for (int i = 0; i < 19; ++i) cl[i] = 0;
    for (int i = 0; i < ncode; ++i) {
        if (!r.need(3)) return kEof;
        cl[kClOrder[i]] = uint8_t(r.peek(3));
        r.drop(3);
    }
    c.cl.build(cl, 19);
    if (c.cl.over || (c.cl.incomplete && c.cl.max > 0)) return kData;
    const bool empty = c.cl.max == 0;   // zlib reads 1 bit per length, as length 0
    int have = 0;
    while (have < nlen + ndist) {
        int s = 0;
        if (empty) {
            if (!r.need(1)) return kEof;
            r.drop(1);
        } else {
            const int64_t st = c.cl.decode(r, s);
            if (st != kOk) return st;
        }
        if (s < 16) {
            c.lens[have++] = uint8_t(s);
            continue;
        }
        int copy, val = 0;
        if (s == 16) {
            if (!r.need(2)) return kEof;
            copy = 3 + int(r.peek(2));
            r.drop(2);
            if (have == 0) return kData;
            val = c.lens[have - 1];
        } else if (s == 17) {
            if (!r.need(3)) return kEof;
            copy = 3 + int(r.peek(3));
            r.drop(3);
        } else {
            if (!r.need(7)) return kEof;
            copy = 11 + int(r.peek(7));
            r.drop(7);
        }
        if (have + copy > nlen + ndist) return kData;
        while (copy--) c.lens[have++] = uint8_t(val);
    }
    if (c.lens[256] == 0) return kData;
    c.lit.build(c.lens, nlen);
    if (c.lit.over || (c.lit.incomplete && c.lit.max > 1)) return kData;
    c.dist.build(c.lens + nlen, ndist);
    if (c.dist.over || (c.dist.incomplete && c.dist.max > 1)) return kData;
    return kOk;
}

struct Sink {
    uint16_t* out;
    int64_t cap, count, last_marker;
};

// One block at r.  TRIAL keeps no symbols and checks no distance against the output.  kOk / kFinal at its end.
template <bool TRIAL>
__device__ int64_t block(Reader& r, Codes& c, Sink& o, bool first) {
    if (!r.need(3)) return kEof;
    const bool final = r.peek(1);
    const int kind = int((r.buf >> 1) & 3);
    r.drop(3);
    const int64_t done = final ? kFinal : kOk;
    if (kind == 3) return kData;
    if (kind == 0) {
        r.drop(r.cnt & 7);
        if (!r.need(32)) return kEof;
        const uint32_t len = r.peek(16), nlen = uint32_t(r.buf >> 16) & 0xFFFF;
        r.drop(32);
        if (len != (nlen ^ 0xFFFF)) return kData;
        // byte-aligned: the bytes still in the bit buffer, then straight from the input
        uint32_t i = 0;
        for (; i < len && r.cnt >= 8; ++i) {
            if (!TRIAL) {
                if (o.count >= o.cap) return kOverflow;
                o.out[o.count++] = uint16_t(r.peek(8));
            }
            r.drop(8);
        }
        const int64_t rest = int64_t(len - i);
        if (rest > r.nbytes - r.next) return kEof;
        if (!TRIAL) {
            if (rest > o.cap - o.count) return kOverflow;
            const uint8_t* src = r.d + r.next;
            for (int64_t k = 0; k < rest; ++k) o.out[o.count + k] = __ldg(src + k);
            o.count += rest;
        }
        r.next += rest;
        return done;
    }
    const int64_t hs = kind == 1 ? fixed_codes(c) : dynamic_codes(r, c);
    if (hs != kOk) return hs;
    for (;;) {
        int s;
        int64_t st = c.lit.decode(r, s);
        if (st != kOk) return st;
        if (s < 256) {
            if (!TRIAL) {
                if (o.count >= o.cap) return kOverflow;
                o.out[o.count++] = uint16_t(s);
            }
            continue;
        }
        if (s == 256) return done;
        if (s > 285) return kData;
        const int li = s - 257;
        if (!r.need(kLExt[li])) return kEof;
        const int len = kLBase[li] + int(r.peek(kLExt[li]));
        r.drop(kLExt[li]);
        int ds;
        st = c.dist.decode(r, ds);
        if (st != kOk) return st;
        if (ds > 29) return kData;
        if (!r.need(kDExt[ds])) return kEof;
        const int dist = kDBase[ds] + int(r.peek(kDExt[ds]));
        r.drop(kDExt[ds]);
        if (TRIAL) continue;
        if (first && dist > o.count) return kData;
        if (o.count + len > o.cap) return kOverflow;
        for (int i = 0; i < len; ++i) {
            const int64_t src = o.count - dist;
            const uint16_t v = src >= 0 ? o.out[src] : uint16_t(kMark | (kWindow + src));
            if (v & kMark) o.last_marker = o.count;
            o.out[o.count++] = v;
        }
    }
}

// A stored block header at bit b: BTYPE 00, zero bits to the byte boundary, LEN = ~NLEN.
__device__ bool stored_at(const uint8_t* d, int64_t n, int64_t b) {
    Reader r;
    r.init(d, n, b);
    if (!r.need(3) || ((r.buf >> 1) & 3) != 0) return false;
    r.drop(3);
    const int pad = r.cnt & 7;
    if (!r.need(pad + 32) || r.peek(pad)) return false;
    r.drop(pad);
    return r.peek(16) == ((uint32_t(r.buf >> 16) & 0xFFFF) ^ 0xFFFF);
}

// The finder's test of bit offset b (see the file comment).  A stored header that starts inside a byte is refused when
// the next byte boundary holds one too: the zero bits before a byte-aligned header (level 0's blocks follow each other
// on byte boundaries) would otherwise pass, with the header byte and LEN read as a LEN / NLEN pair.
__device__ bool plausible(const uint8_t* d, int64_t n, int64_t b, Codes& c) {
    Reader r;
    r.init(d, n, b);
    if (!r.need(3)) return false;
    const int kind = int((r.buf >> 1) & 3);
    if (kind == 0) return stored_at(d, n, b) && !((b & 7) && stored_at(d, n, (b + 7) & ~int64_t(7)));
    if (kind != 2) return false;
    if (r.need(13) && (((r.buf >> 3) & 31) > 29 || ((r.buf >> 8) & 31) > 29)) return false;
    Sink none{nullptr, 0, 0, -1};
    const int64_t st = block<true>(r, c, none, false);
    return st == kOk || st == kFinal;
}

__global__ void __launch_bounds__(kRunThreads) k_inflate_run(const uint8_t* __restrict__ d, int64_t n,
                                                             const int64_t* __restrict__ jobs, int64_t njobs,
                                                             uint16_t* __restrict__ ws, int64_t ws_syms,
                                                             int64_t* __restrict__ res) {
    const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= njobs) return;
    const int64_t* jb = jobs + 6 * j;
    const int64_t lo = jb[0], hi = jb[1], target = jb[2], off = jb[3], cap = jb[4], flags = jb[5];
    int64_t* rs = res + 6 * j;
    const int64_t nbits = 8 * n;
    if (lo < 0 || lo > nbits || off < 0 || cap < 0 || off > ws_syms || cap > ws_syms - off) {
        rs[0] = -1, rs[1] = lo, rs[2] = 0, rs[3] = -1, rs[4] = kBadJob, rs[5] = lo;
        return;
    }
    Codes c;
    int64_t start = lo;
    if (flags & kFind) {
        start = -1;
        // 13 bits of each offset screen it (BTYPE 00, or BTYPE 10 with HLIT <= 29 and HDIST <= 29) before plausible()
        for (int64_t b = lo & ~int64_t(7); b < min(hi, nbits) && start < 0; b += 8) {
            uint64_t w = 0;
            for (int k = 0; k < 8 && (b >> 3) + k < n; ++k) w |= uint64_t(__ldg(d + (b >> 3) + k)) << (8 * k);
            for (int o = 0; o < 8; ++o) {
                const int64_t at = b + o;
                if (at < lo || at >= min(hi, nbits)) continue;
                const uint64_t v = w >> o;
                const int kind = int((v >> 1) & 3);
                if (kind == 1 || kind == 3) continue;
                if (kind == 2 && (((v >> 3) & 31) > 29 || ((v >> 8) & 31) > 29)) continue;
                if (plausible(d, n, at, c)) {
                    start = at;
                    break;
                }
            }
        }
        if (start < 0) {
            rs[0] = -1, rs[1] = lo, rs[2] = 0, rs[3] = -1, rs[4] = kNone, rs[5] = lo;
            return;
        }
    }
    Reader r;
    r.init(d, n, start);
    Sink o{ws + off, cap, 0, -1};
    int64_t st, stop = start;
    for (;;) {
        st = block<false>(r, c, o, flags & kFirst);
        if (st != kOk && st != kFinal) break;
        stop = r.pos();
        if (st == kFinal || stop >= target) break;
    }
    rs[0] = start, rs[1] = stop, rs[2] = o.count, rs[3] = o.last_marker, rs[4] = st, rs[5] = r.pos();
}

// pieces: int64 [npieces, 5] = symbols (device pointer), count, output offset, walk_lo, walk_hi
struct Piece {
    const uint16_t* syms;
    int64_t count, off, walk_lo, walk_hi;
};

__device__ __forceinline__ Piece piece(const int64_t* p, int64_t i) {
    const int64_t* q = p + 5 * i;
    return Piece{reinterpret_cast<const uint16_t*>(q[0]), q[1], q[2], q[3], q[4]};
}

__device__ __forceinline__ void put_marker(const Piece& P, int64_t i, uint16_t s, uint8_t* out,
                                           unsigned long long* status) {
    const int64_t t = P.off - kWindow + (s & 0x7FFF);
    if (t < 0) {
        atomicMin(status, (unsigned long long)(P.off + i));
        return;
    }
    out[P.off + i] = out[t];
}

__global__ void __launch_bounds__(256) k_inflate_bytes(const int64_t* __restrict__ pieces, uint8_t* __restrict__ out) {
    const Piece P = piece(pieces, blockIdx.x);
    for (int64_t i = int64_t(blockIdx.y) * blockDim.x + threadIdx.x; i < P.count; i += int64_t(gridDim.y) * blockDim.x) {
        const uint16_t s = P.syms[i];
        if (!(s & kMark)) out[P.off + i] = uint8_t(s);
    }
}

__global__ void __launch_bounds__(1024) k_inflate_window(const int64_t* __restrict__ pieces, int64_t npieces,
                                                         uint8_t* out, unsigned long long* status) {
    for (int64_t k = 0; k < npieces; ++k) {
        const Piece P = piece(pieces, k);
        for (int64_t i = P.walk_lo + threadIdx.x; i < P.walk_hi; i += blockDim.x) {
            const uint16_t s = P.syms[i];
            if (s & kMark) put_marker(P, i, s, out, status);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_inflate_markers(const int64_t* __restrict__ pieces, uint8_t* out,
                                                         unsigned long long* status) {
    const Piece P = piece(pieces, blockIdx.x);
    for (int64_t i = int64_t(blockIdx.y) * blockDim.x + threadIdx.x; i < P.walk_lo;
         i += int64_t(gridDim.y) * blockDim.x) {
        const uint16_t s = P.syms[i];
        if (s & kMark) put_marker(P, i, s, out, status);
    }
}

}  // namespace
}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_inflate_workspace_bytes(int64_t symbols) {
    if (symbols < 0) return 0;
    return 2 * symbols + 256;
}

int gsx_inflate_run(const uint8_t* data, int64_t n, const int64_t* jobs, int64_t njobs, void* ws, int64_t ws_bytes,
                    int64_t* results, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_inflate_run");
    GSX_REQUIRE(n >= 0 && (data || n == 0) && (jobs || njobs == 0) && (results || njobs == 0) && ws_bytes >= 0 &&
                    (ws || ws_bytes == 0),
                GSX_ERR_ARG, "inflate_run: bad arguments");
    GSX_REQUIRE(njobs >= 0 && njobs < (int64_t(1) << 31) * kRunThreads, GSX_ERR_ARG,
                "inflate_run: njobs must be 0..2^37 (got %lld)", (long long)njobs);
    if (njobs == 0) return GSX_OK;
    const int64_t grid = (njobs + kRunThreads - 1) / kRunThreads;
    k_inflate_run<<<unsigned(grid), kRunThreads, 0, st>>>(data, n, jobs, njobs, (uint16_t*)ws, ws_bytes / 2, results);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_inflate_resolve(const int64_t* pieces, int64_t npieces, uint8_t* out, unsigned long long* status,
                        void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_inflate_resolve");
    GSX_REQUIRE(npieces >= 0 && npieces < (int64_t(1) << 31) && (pieces || npieces == 0) && status, GSX_ERR_ARG,
                "inflate_resolve: bad arguments");
    if (npieces == 0) return GSX_OK;
    const dim3 grid(unsigned(npieces), 16);
    k_inflate_bytes<<<grid, 256, 0, st>>>(pieces, out);
    GSX_KERNEL_CHECK();
    k_inflate_window<<<1, 1024, 0, st>>>(pieces, npieces, out, status);
    GSX_KERNEL_CHECK();
    k_inflate_markers<<<grid, 256, 0, st>>>(pieces, out, status);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

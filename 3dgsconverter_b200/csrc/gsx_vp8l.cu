// gsx_vp8l.cu -- lossless WebP (VP8L, RFC 9649) decoding on the device: the SOG bundle's members (gsx/webp_decode.py).
// tests/vp8l_model.py restates every stage in Python.
//
//   k_vp8l_header   one thread: the VP8L header, the transforms and their sub-images (predictor and cross-colour
//                   tiles, the colour table), the colour cache bits, the entropy image, and every group's five prefix
//                   codes as lookup tables in the workspace.
//   k_vp8l_run      one thread per job: tokens of the main image from a bit offset, at a guessed pixel position (the
//                   position only picks the group).  A token is a literal ARGB, a copy (length, distance code) or a
//                   colour-cache index; each records its first pixel relative to the job's start and its group.
//   k_vp8l_check    per chain piece decoded at another position than the chain gives it: does every token's group
//                   equal the group at its true position.
//   k_vp8l_expand   every token of the chain to its pixels: a literal, a source pixel, or a cache slot.
//   k_vp8l_jump     (no colour cache) pointer jumping over source pixels, in place.
//   k_vp8l_replay   (colour cache) one thread in pixel order, the cache in shared memory.
//   inverse transforms in reverse order of reading: k_vp8l_index, k_vp8l_green, k_vp8l_cross, k_vp8l_predict (a
//   wavefront: one warp per 32 rows, lane r at x = step - 2r, each warp behind the one above it), then k_vp8l_rgba.
#include "../../include/gsx.h"

#include "gsx_common.cuh"
#include "gsx_vp8l_format.cuh"

namespace gsx {
namespace {

enum : int64_t { kOk = 0, kTrunc = 1, kBadCode = 2, kBadHeader = 3, kSpace = 4 };
enum : int64_t { kJobOk = 0, kJobEnd = 1, kJobEof = 2, kJobOverflow = 4 };
enum : uint32_t { kLit = 0, kCopy = 1, kCache = 2 };
constexpr int kFast = 8;
constexpr int kMaxAlpha = 280 + 2048;
// a code in the workspace: [0] the lone symbol of a 0-bit code or 0xFFFFFFFF, [1] longest length, [2..17] counts per
// length, [18..273] the 8-bit table (symbol | length << 16, 0: longer), then the symbols by (length, symbol)
constexpr int kCodeWords = 18 + (1 << kFast) + kMaxAlpha;
constexpr int kGroupWords = 5 * kCodeWords;
constexpr int kCacheScratch = 2048;
constexpr int kInfo = 32;

__constant__ uint8_t kClOrder[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
// RFC 9649 section 4.2.2: distance codes 1..120 as yoffset << 4 | (8 - xoffset)
__constant__ uint8_t kPlane[120] = {
    0x18, 0x07, 0x17, 0x19, 0x28, 0x06, 0x27, 0x29, 0x16, 0x1a, 0x26, 0x2a, 0x38, 0x05, 0x37, 0x39, 0x15, 0x1b, 0x36, 0x3a,
    0x25, 0x2b, 0x48, 0x04, 0x47, 0x49, 0x14, 0x1c, 0x35, 0x3b, 0x46, 0x4a, 0x24, 0x2c, 0x58, 0x45, 0x4b, 0x34, 0x3c, 0x03,
    0x57, 0x59, 0x13, 0x1d, 0x56, 0x5a, 0x23, 0x2d, 0x44, 0x4c, 0x55, 0x5b, 0x33, 0x3d, 0x68, 0x02, 0x67, 0x69, 0x12, 0x1e,
    0x66, 0x6a, 0x22, 0x2e, 0x54, 0x5c, 0x43, 0x4d, 0x65, 0x6b, 0x32, 0x3e, 0x78, 0x01, 0x77, 0x79, 0x53, 0x5d, 0x11, 0x1f,
    0x64, 0x6c, 0x42, 0x4e, 0x76, 0x7a, 0x21, 0x2f, 0x75, 0x7b, 0x31, 0x3f, 0x63, 0x6d, 0x52, 0x5e, 0x00, 0x74, 0x7c, 0x41,
    0x4f, 0x10, 0x20, 0x62, 0x6e, 0x30, 0x73, 0x7d, 0x51, 0x5f, 0x40, 0x72, 0x7e, 0x61, 0x6f, 0x50, 0x71, 0x7f, 0x60, 0x70};

// libwebp's acceptance: not all lengths 0, at most 2^len codes of each length, exactly one used symbol (of any length
// 1..15) is a 0-bit code, anything else must fill the code space.
__device__ int64_t build_code(const uint8_t* len, int n, uint32_t* c) {
    uint32_t count[16];
    for (int i = 0; i < 16; ++i) count[i] = 0;
    for (int s = 0; s < n; ++s) ++count[len[s]];
    if (count[0] == uint32_t(n)) return kBadCode;
    uint32_t used = 0;
    for (int b = 1; b < 16; ++b) {
        if (count[b] > (1u << b)) return kBadCode;
        used += count[b];
    }
    if (used == 1) {
        for (int s = 0; s < n; ++s)
            if (len[s]) c[0] = uint32_t(s);
        return kOk;
    }
    int64_t left = 1;
    int mx = 0;
    for (int b = 1; b < 16; ++b) {
        left = 2 * left - count[b];
        if (left < 0) return kBadCode;
        if (count[b]) mx = b;
    }
    if (left) return kBadCode;
    c[0] = 0xFFFFFFFFu, c[1] = uint32_t(mx);
    uint32_t offs[16], code[16];
    offs[1] = 0, code[1] = 0;
    for (int b = 1; b < 15; ++b) offs[b + 1] = offs[b] + count[b], code[b + 1] = (code[b] + count[b]) << 1;
    for (int b = 0; b < 16; ++b) c[2 + b] = count[b];
    uint32_t* fast = c + 18;
    uint32_t* sym = c + 18 + (1 << kFast);
    for (int i = 0; i < (1 << kFast); ++i) fast[i] = 0;
    for (int s = 0; s < n; ++s) {
        const int b = len[s];
        if (!b) continue;
        sym[offs[b]++] = uint32_t(s);
        const uint32_t cd = code[b]++;
        if (b > kFast) continue;
        const uint32_t rev = __brev(cd) >> (32 - b);
        for (uint32_t r = rev; r < (1u << kFast); r += 1u << b) fast[r] = uint32_t(s) | uint32_t(b) << 16;
    }
    return kOk;
}

__device__ __forceinline__ bool decode(Reader& r, const uint32_t* __restrict__ c, uint32_t& out) {
    const uint32_t single = c[0];
    if (single != 0xFFFFFFFFu) {
        out = single;
        return true;
    }
    r.need(15);
    const uint32_t e = c[18 + r.peek(kFast)];
    if (e) {
        const int b = int(e >> 16);
        if (r.cnt < b) return false;
        r.drop(b);
        out = e & 0xFFFF;
        return true;
    }
    const int mx = int(c[1]);
    int code = 0, first = 0, index = 0;
    for (int b = 1; b <= mx; ++b) {
        if (r.cnt < b) return false;
        code |= int((r.buf >> (b - 1)) & 1);
        const int cn = int(c[2 + b]);
        if (code - cn < first) {
            r.drop(b);
            out = c[18 + (1 << kFast) + index + code - first];
            return true;
        }
        index += cn;
        first = (first + cn) << 1;
        code <<= 1;
    }
    return false;   // unreachable for a complete code
}

// One prefix code of `alphabet` symbols at r into c.  A simple code's symbol past the alphabet (possible only in the
// 40-symbol distance alphabet) gets no length, as in libwebp: the code is built from the others, and none is an error.
__device__ int64_t read_code(Reader& r, int alphabet, uint32_t* c, uint8_t* len) {
    uint32_t v;
    if (!r.bits(1, v)) return kTrunc;
    for (int s = 0; s < alphabet; ++s) len[s] = 0;
    if (v) {
        uint32_t two, wide, s0, s1;
        if (!r.bits(1, two) || !r.bits(1, wide) || !r.bits(wide ? 8 : 1, s0)) return kTrunc;
        if (int(s0) < alphabet) len[s0] = 1;
        if (two) {
            if (!r.bits(8, s1)) return kTrunc;
            if (int(s1) < alphabet) len[s1] = 1;
        }
        return build_code(len, alphabet, c);
    }
    uint8_t cl[19];
    uint32_t clc[18 + (1 << kFast) + 19];
    for (int i = 0; i < 19; ++i) cl[i] = 0;
    uint32_t ncl;
    if (!r.bits(4, ncl)) return kTrunc;
    for (uint32_t i = 0; i < ncl + 4; ++i) {
        if (!r.bits(3, v)) return kTrunc;
        cl[kClOrder[i]] = uint8_t(v);
    }
    int64_t st = build_code(cl, 19, clc);
    if (st != kOk) return st;
    int max_symbol = alphabet;
    if (!r.bits(1, v)) return kTrunc;
    if (v) {
        uint32_t nb, ms;
        if (!r.bits(3, nb) || !r.bits(2 + 2 * int(nb), ms)) return kTrunc;
        max_symbol = 2 + int(ms);
        if (max_symbol > alphabet) return kBadCode;
    }
    int s = 0;
    uint8_t prev = 8;
    while (s < alphabet) {
        if (max_symbol-- == 0) break;
        uint32_t k;
        if (!decode(r, clc, k)) return kTrunc;
        if (k < 16) {
            len[s++] = uint8_t(k);
            if (k) prev = uint8_t(k);
            continue;
        }
        const int extra = k == 16 ? 2 : k == 17 ? 3 : 7, base = k == 18 ? 11 : 3;
        uint32_t rep;
        if (!r.bits(extra, rep)) return kTrunc;
        if (s + int(rep) + base > alphabet) return kBadCode;
        for (int i = 0; i < int(rep) + base; ++i) len[s++] = k == 16 ? prev : 0;
    }
    return build_code(len, alphabet, c);
}

__device__ __forceinline__ int64_t plane_distance(uint32_t code, int64_t xsize) {
    if (code > 120) return int64_t(code) - 120;
    const int p = kPlane[code - 1];
    const int64_t d = int64_t(p >> 4) * xsize + (8 - (p & 15));
    return d >= 1 ? d : 1;
}

__device__ __forceinline__ uint32_t cache_slot(uint32_t v, int bits) { return (0x1E35A7BDu * v) >> (32 - bits); }

// One token with group g's codes: kind, value (ARGB, distance code or cache index), pixels.
__device__ __forceinline__ bool token(Reader& r, const uint32_t* __restrict__ g, uint32_t& kind, uint32_t& val,
                                      uint32_t& npx) {
    uint32_t s;
    if (!decode(r, g, s)) return false;
    if (s < 256) {
        uint32_t red, blue, alpha;
        if (!decode(r, g + kCodeWords, red) || !decode(r, g + 2 * kCodeWords, blue) ||
            !decode(r, g + 3 * kCodeWords, alpha))
            return false;
        kind = kLit, val = alpha << 24 | red << 16 | s << 8 | blue, npx = 1;
        return true;
    }
    if (s < 280) {
        uint32_t d;
        if (!prefix_value(r, s - 256, npx) || !decode(r, g + 4 * kCodeWords, d) || !prefix_value(r, d, val))
            return false;
        kind = kCopy;
        return true;
    }
    kind = kCache, val = s - 280, npx = 1;
    return true;
}

__device__ int64_t read_cache_bits(Reader& r, int& bits) {
    uint32_t v;
    bits = 0;
    if (!r.bits(1, v)) return kTrunc;
    if (!v) return kOk;
    if (!r.bits(4, v)) return kTrunc;
    if (v < 1 || v > 11) return kBadHeader;
    bits = int(v);
    return kOk;
}

__device__ int64_t read_groups(Reader& r, int64_t ngroups, int cache_bits, uint32_t* out, uint8_t* len) {
    const int green = 280 + (cache_bits ? 1 << cache_bits : 0);
    for (int64_t gi = 0; gi < ngroups; ++gi)
        for (int k = 0; k < 5; ++k) {
            const int64_t st = read_code(r, k == 0 ? green : k == 4 ? 40 : 256, out + gi * kGroupWords + k * kCodeWords,
                                         len);
            if (st != kOk) return st;
        }
    return kOk;
}

// An entropy-coded sub-image of w x h pixels into img, decoded and resolved serially.
__device__ int64_t sub_image(Reader& r, int64_t w, int64_t h, uint32_t* img, uint32_t* code, uint32_t* cache,
                             uint8_t* len) {
    int cb;
    int64_t st = read_cache_bits(r, cb);
    if (st != kOk) return st;
    if (cb)   // every image starts with an empty (all zero) cache: a first cache index reads 0x00000000
        for (int i = 0; i < (1 << cb); ++i) cache[i] = 0;
    st = read_groups(r, 1, cb, code, len);
    if (st != kOk) return st;
    const int64_t n = w * h;
    for (int64_t i = 0; i < n;) {
        uint32_t kind, val, npx;
        if (!token(r, code, kind, val, npx)) return kTrunc;
        const int64_t from = i;
        if (kind == kCopy) {
            const int64_t d = plane_distance(val, w);
            if (d > i || i + npx > n) return kBadCode;
            for (uint32_t k = 0; k < npx; ++k, ++i) img[i] = img[i - d];
        } else {
            img[i++] = kind == kLit ? val : cache[val];
        }
        if (cb)
            for (int64_t k = from; k < i; ++k) cache[cache_slot(img[k], cb)] = img[k];
    }
    return kOk;
}

__device__ __forceinline__ int64_t divb(int64_t a, int b) { return (a + (int64_t(1) << b) - 1) >> b; }

// info int64 [32]: 0 status, 1 bit where it stopped, 2 width, 3 height, 4 alpha hint, 5 coded width, 6 cache bits,
// 7 meta bits, 8 groups, 9 entropy image word offset (-1: none), 10 codes word offset, 11 main image's first bit,
// 12 transforms, 13 + 4t: type, width, bits, word offset of transform t (in reading order), 29 words needed.
__global__ void k_vp8l_header(const uint8_t* __restrict__ d, int64_t n, uint32_t* __restrict__ ws, int64_t ws_words,
                              uint8_t* __restrict__ lens, int64_t* __restrict__ info) {
    for (int i = 0; i < kInfo; ++i) info[i] = 0;
    Reader r;
    r.init(d, n, 0);
    int64_t st = kOk;
    uint32_t* cache = ws;
    int64_t bump = kCacheScratch;
    uint32_t v, w1, h1, a, ver;
    auto fail = [&](int64_t s) {
        info[0] = s, info[1] = r.pos();
    };
    if (!r.bits(8, v) || !r.bits(14, w1) || !r.bits(14, h1) || !r.bits(1, a) || !r.bits(3, ver)) return fail(kTrunc);
    if (v != 0x2F || ver != 0) return fail(kBadHeader);
    const int64_t width = int64_t(w1) + 1, height = int64_t(h1) + 1;
    info[2] = width, info[3] = height, info[4] = a;
    // sub-images take at most 2 * tiles (predictor, cross-colour) + 256 (colours) + tiles (entropy) words
    const int64_t tiles = divb(width, 2) * divb(height, 2);
    const int64_t sub_end = kCacheScratch + 3 * tiles + 256;
    uint32_t* subcode = ws + sub_end;   // the sub-images' one group of codes, then the main image's groups
    const int64_t codes_at = sub_end + kGroupWords;
    if (codes_at + kGroupWords > ws_words) {
        info[29] = codes_at + kGroupWords;
        return fail(kSpace);
    }
    int64_t xs = width;
    int seen = 0, nt = 0;
    for (;;) {
        if (!r.bits(1, v)) return fail(kTrunc);
        if (!v) break;
        uint32_t t;
        if (!r.bits(2, t)) return fail(kTrunc);
        if (seen & (1 << t)) return fail(kBadHeader);
        seen |= 1 << t;
        int64_t* ti = info + 13 + 4 * nt++;
        ti[0] = t, ti[1] = xs, ti[2] = 0, ti[3] = bump;
        if (t == 0 || t == 1) {
            uint32_t b;
            if (!r.bits(3, b)) return fail(kTrunc);
            const int bits = int(b) + 2;
            ti[2] = bits;
            const int64_t sw = divb(xs, bits), sh = divb(height, bits);
            st = sub_image(r, sw, sh, ws + bump, subcode, cache, lens);
            if (st != kOk) return fail(st);
            bump += sw * sh;
        } else if (t == 3) {
            uint32_t m;
            if (!r.bits(8, m)) return fail(kTrunc);
            const int ncol = int(m) + 1;
            const int bits = ncol > 16 ? 0 : ncol > 4 ? 1 : ncol > 2 ? 2 : 3;
            ti[2] = bits;
            uint32_t* pal = ws + bump;
            st = sub_image(r, ncol, 1, pal, subcode, cache, lens);
            if (st != kOk) return fail(st);
            for (int i = 1; i < ncol; ++i) {   // delta-coded, per byte
                const uint32_t p = pal[i - 1], q = pal[i];
                pal[i] = (((p & 0x00FF00FFu) + (q & 0x00FF00FFu)) & 0x00FF00FFu) |
                         (((p & 0xFF00FF00u) + (q & 0xFF00FF00u)) & 0xFF00FF00u);
            }
            for (int i = ncol; i < 256; ++i) pal[i] = 0;
            bump += 256;
            xs = divb(xs, bits);
        }
    }
    info[12] = nt, info[5] = xs;
    int cb;
    st = read_cache_bits(r, cb);
    if (st != kOk) return fail(st);
    info[6] = cb;
    if (!r.bits(1, v)) return fail(kTrunc);
    int64_t ngroups = 1;
    info[9] = -1;
    if (v) {
        uint32_t b;
        if (!r.bits(3, b)) return fail(kTrunc);
        const int bits = int(b) + 2;
        const int64_t sw = divb(xs, bits), sh = divb(height, bits);
        uint32_t* img = ws + bump;
        st = sub_image(r, sw, sh, img, subcode, cache, lens);
        if (st != kOk) return fail(st);
        uint32_t mx = 0;
        for (int64_t i = 0; i < sw * sh; ++i) {
            img[i] = (img[i] >> 8) & 0xFFFF;
            mx = max(mx, img[i]);
        }
        ngroups = int64_t(mx) + 1;
        info[7] = bits, info[9] = bump;
        bump += sw * sh;
    }
    info[8] = ngroups, info[10] = codes_at;
    if (codes_at + ngroups * kGroupWords > ws_words) {
        info[29] = codes_at + ngroups * kGroupWords;
        return fail(kSpace);
    }
    st = read_groups(r, ngroups, cb, ws + codes_at, lens);
    if (st != kOk) return fail(st);
    info[11] = r.pos();
    info[0] = kOk, info[1] = r.pos();
}

struct Image {
    const uint32_t* codes;
    const uint32_t* entropy;   // nullptr: one group
    int64_t xsize, npix;
    int meta_bits;
};

__device__ __forceinline__ uint32_t group_at(const Image& im, int64_t p) {
    if (!im.entropy || p >= im.npix) return 0;
    const int64_t y = p / im.xsize, x = p - y * im.xsize;
    return __ldg(im.entropy + (y >> im.meta_bits) * divb(im.xsize, im.meta_bits) + (x >> im.meta_bits));
}

// jobs int64 [njobs, 5] = start bit, target bit, guessed pixel, token offset, capacity;
// results int64 [njobs, 6] = start, stop bit, tokens, pixels, status, bit where it stopped.
__global__ void __launch_bounds__(64) k_vp8l_run(const uint8_t* __restrict__ d, int64_t n, Image im,
                                                 const int64_t* __restrict__ jobs, int64_t njobs,
                                                 uint4* __restrict__ toks, int64_t* __restrict__ res) {
    const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= njobs) return;
    const int64_t* jb = jobs + 5 * j;
    const int64_t start = jb[0], target = jb[1], guess = jb[2], cap = jb[4];
    uint4* out = toks + jb[3];
    Reader r;
    r.init(d, n, start);
    int64_t cnt = 0, px = 0, stop = start, st = kJobOk;
    for (;;) {
        stop = r.pos();
        if (guess + px >= im.npix) {
            st = kJobEnd;
            break;
        }
        if (stop >= target) break;
        if (cnt >= cap) {
            st = kJobOverflow;
            break;
        }
        const uint32_t g = group_at(im, guess + px);
        uint32_t kind, val, npx;
        if (!token(r, im.codes + int64_t(g) * kGroupWords, kind, val, npx)) {
            st = kJobEof;
            break;
        }
        out[cnt++] = make_uint4(val, kind << 28 | npx, uint32_t(px), g);
        px += npx;
    }
    int64_t* rs = res + 6 * j;
    rs[0] = start, rs[1] = stop, rs[2] = cnt, rs[3] = px, rs[4] = st, rs[5] = r.pos();
}

// pieces int64 [npieces, 3] = token address, tokens, true first pixel; flags int32 [npieces] (zeroed): 1 = a group
// differs from the one at the true position.
__global__ void k_vp8l_check(Image im, const int64_t* __restrict__ pieces, int32_t* __restrict__ flags) {
    const int64_t* p = pieces + 3 * blockIdx.x;
    const uint4* t = reinterpret_cast<const uint4*>(p[0]);
    for (int64_t i = int64_t(blockIdx.y) * blockDim.x + threadIdx.x; i < p[1]; i += int64_t(gridDim.y) * blockDim.x) {
        const uint4 k = t[i];
        if (group_at(im, p[2] + k.z) != k.w) flags[blockIdx.x] = 1;
    }
}

// pieces int64 [npieces, 3] = token address, tokens, first pixel.  src[i]: -1 = out[i] is final, >= 0 the pixel it
// copies, -2 - slot the cache slot it reads.  err (zeroed): bit 0 a copy from before the first pixel, bit 1 a copy
// past the last.
__global__ void k_vp8l_expand(const int64_t* __restrict__ pieces, int64_t xsize, int64_t npix,
                              uint32_t* __restrict__ out, int32_t* __restrict__ src, int32_t* __restrict__ err) {
    const int64_t* p = pieces + 3 * blockIdx.x;
    const uint4* t = reinterpret_cast<const uint4*>(p[0]);
    for (int64_t i = int64_t(blockIdx.y) * blockDim.x + threadIdx.x; i < p[1]; i += int64_t(gridDim.y) * blockDim.x) {
        const uint4 k = t[i];
        const int64_t at = p[2] + k.z;
        const uint32_t kind = k.y >> 28, len = k.y & 0x0FFFFFFF;
        if (at >= npix) {
            atomicOr(err, 2);
            continue;
        }
        if (kind == kLit) {
            out[at] = k.x, src[at] = -1;
        } else if (kind == kCache) {
            src[at] = -2 - int32_t(k.x);
        } else {
            const int64_t dist = plane_distance(k.x, xsize);
            const int64_t end = min(at + int64_t(len), npix);
            if (dist > at || at + len > npix) {   // refused: the pixels it covers are left as 0 for the resolve
                atomicOr(err, dist > at ? 1 : 2);
                for (int64_t c = at; c < end; ++c) out[c] = 0, src[c] = -1;
                continue;
            }
            for (uint32_t c = 0; c < len; ++c) src[at + c] = int32_t(at + c - dist);
        }
    }
}

__global__ void k_vp8l_jump(volatile uint32_t* out, volatile int32_t* src, int64_t npix) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < npix; i += int64_t(gridDim.x) * blockDim.x) {
        const int32_t s = src[i];
        if (s < 0) continue;
        const int32_t t = src[s];
        if (t == -1) {
            __threadfence();
            out[i] = out[s];
            __threadfence();
            src[i] = -1;
        } else {
            src[i] = t;
        }
    }
}

__global__ void __launch_bounds__(32) k_vp8l_replay(uint32_t* __restrict__ out, const int32_t* __restrict__ src,
                                                    int64_t npix, int bits) {
    __shared__ uint32_t cache[2048];
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) cache[i] = 0;
    __syncthreads();
    if (threadIdx.x) return;
    for (int64_t i = 0; i < npix; ++i) {
        const int32_t s = src[i];
        const uint32_t v = s == -1 ? out[i] : s >= 0 ? out[s] : cache[-2 - s];
        out[i] = v;
        cache[cache_slot(v, bits)] = v;
    }
}

__global__ void k_vp8l_index(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, const uint32_t* __restrict__ pal,
                             int64_t xs, int64_t height, int bits) {
    const int64_t pw = divb(xs, bits), n = xs * height;
    const int per = 8 >> bits, mask = (1 << per) - 1;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t y = i / xs, x = i - y * xs;
        const uint32_t g = (in[y * pw + (x >> bits)] >> 8) & 0xFF;
        out[i] = __ldg(pal + ((g >> ((x & ((1 << bits) - 1)) * per)) & mask));
    }
}

__global__ void k_vp8l_green(uint32_t* __restrict__ px, int64_t n) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const uint32_t v = px[i], g = (v >> 8) & 0xFF;
        px[i] = (v & 0xFF00FF00u) | ((((v >> 16) + g) & 0xFF) << 16) | ((v + g) & 0xFF);
    }
}

__device__ __forceinline__ int delta(uint32_t t, uint32_t c) { return (int(int8_t(t)) * int(int8_t(c))) >> 5; }

__global__ void k_vp8l_cross(uint32_t* __restrict__ px, const uint32_t* __restrict__ tiles, int64_t xs, int64_t height,
                             int bits) {
    const int64_t n = xs * height, tx = divb(xs, bits);
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t y = i / xs, x = i - y * xs;
        const uint32_t m = __ldg(tiles + (y >> bits) * tx + (x >> bits)), v = px[i];
        const uint32_t g = (v >> 8) & 0xFF;
        const uint32_t red = ((v >> 16) + delta(m, g)) & 0xFF;
        const uint32_t blue = (v + delta(m >> 8, g) + delta(m >> 16, red)) & 0xFF;
        px[i] = (v & 0xFF00FF00u) | red << 16 | blue;
    }
}

__device__ __forceinline__ uint32_t add_pixels(uint32_t a, uint32_t b) {
    return (((a & 0x00FF00FFu) + (b & 0x00FF00FFu)) & 0x00FF00FFu) |
           (((a & 0xFF00FF00u) + (b & 0xFF00FF00u)) & 0xFF00FF00u);
}

// One warp per 32 rows, taken in order from *ticket so that every warp above a running one is running too; lane r
// decodes x = step - 2r of its row, so its T and TR (x + 1 of the row above) are one step old.  The warp's first row
// waits for the last row of the warp above through progress[], which holds each warp's last-row pixels done.
__global__ void __launch_bounds__(32) k_vp8l_predict(uint32_t* px, const uint32_t* __restrict__ tiles, int64_t xs,
                                                     int64_t height, int bits, int32_t* ticket, int32_t* progress) {
    __shared__ int w_s;
    const int lane = threadIdx.x;
    if (lane == 0) w_s = atomicAdd(ticket, 1);
    __syncthreads();
    const int w = w_s;
    const int64_t y = int64_t(w) * 32 + lane, tx = divb(xs, bits);
    volatile uint32_t* v = px;
    volatile int32_t* prog = progress;
    for (int64_t s = 0; s < xs + 62; ++s) {
        if (w > 0 && s < xs) {
            const int64_t need = min(s + 2, xs);
            while (prog[w - 1] < need) {
            }
            __threadfence();
        }
        const int64_t x = s - 2 * lane;
        if (y < height && x >= 0 && x < xs) {
            const int64_t i = y * xs + x;
            uint32_t p;
            if (i == 0) p = 0xFF000000u;
            else if (y == 0) p = v[i - 1];
            else if (x == 0) p = v[i - xs];
            else {
                const int mode = int((__ldg(tiles + (y >> bits) * tx + (x >> bits)) >> 8) & 15);
                p = predict(mode, v[i - 1], v[i - xs], v[i - xs + 1], v[i - xs - 1]);
            }
            v[i] = add_pixels(v[i], p);
        }
        __syncwarp();
        if (lane == 31 && y < height && x >= 0 && x < xs) {
            __threadfence();
            prog[w] = int32_t(x + 1);
        }
    }
}

__global__ void k_vp8l_rgba(const uint32_t* __restrict__ px, uint32_t* __restrict__ out, int64_t n, int alpha) {
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
        const uint32_t v = px[i];
        out[i] = ((v >> 16) & 0xFF) | (v & 0xFF00) | ((v & 0xFF) << 16) | (alpha ? v & 0xFF000000u : 0xFF000000u);
    }
}

inline unsigned grid_for(int64_t n) { return unsigned(std::min<int64_t>(std::max<int64_t>((n + 255) / 256, 1), 16384)); }

}  // namespace
}  // namespace gsx

using namespace gsx;

extern "C" {

int64_t gsx_vp8l_header_words(int64_t width, int64_t height, int64_t groups) {
    if (width < 1 || height < 1 || width > 16384 || height > 16384 || groups < 1 || groups > 65536) return 0;
    const int64_t tiles = ((width + 3) >> 2) * ((height + 3) >> 2);
    return kCacheScratch + 3 * tiles + 256 + (groups + 1) * int64_t(kGroupWords);
}

int gsx_vp8l_header(const uint8_t* data, int64_t n, uint32_t* ws, int64_t ws_words, uint8_t* lens, int64_t* info,
                    void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_vp8l_header");
    GSX_REQUIRE(n >= 0 && (data || n == 0) && ws && ws_words > 0 && lens && info, GSX_ERR_ARG,
                "vp8l_header: bad arguments");
    k_vp8l_header<<<1, 1, 0, st>>>(data, n, ws, ws_words, lens, info);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_vp8l_run(const uint8_t* data, int64_t n, const uint32_t* codes, const uint32_t* entropy, int64_t xsize,
                 int64_t height, int32_t meta_bits, const int64_t* jobs, int64_t njobs, void* tokens, int64_t* results,
                 void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_vp8l_run");
    GSX_REQUIRE(n >= 0 && data && codes && xsize > 0 && height > 0 && njobs >= 0 && njobs < (int64_t(1) << 31) &&
                    (njobs == 0 || (jobs && tokens && results)),
                GSX_ERR_ARG, "vp8l_run: bad arguments");
    if (njobs == 0) return GSX_OK;
    const Image im{codes, entropy, xsize, xsize * height, meta_bits};
    k_vp8l_run<<<unsigned((njobs + 63) / 64), 64, 0, st>>>(data, n, im, jobs, njobs, (uint4*)tokens, results);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_vp8l_check(const uint32_t* codes, const uint32_t* entropy, int64_t xsize, int64_t height, int32_t meta_bits,
                   const int64_t* pieces, int64_t npieces, int32_t* flags, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_vp8l_check");
    GSX_REQUIRE(entropy && pieces && flags && npieces >= 0 && npieces < (int64_t(1) << 31), GSX_ERR_ARG,
                "vp8l_check: bad arguments");
    if (npieces == 0) return GSX_OK;
    const Image im{codes, entropy, xsize, xsize * height, meta_bits};
    k_vp8l_check<<<dim3(unsigned(npieces), 8), 256, 0, st>>>(im, pieces, flags);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_vp8l_resolve(const int64_t* pieces, int64_t npieces, int64_t xsize, int64_t npix,
                     int32_t cache_bits, uint32_t* out, int32_t* src, int32_t* err, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_vp8l_resolve");
    GSX_REQUIRE(pieces && npieces > 0 && npieces < (int64_t(1) << 31) && xsize > 0 && npix > 0 &&
                    npix < (int64_t(1) << 31) && cache_bits >= 0 && cache_bits <= 11 && out && src && err,
                GSX_ERR_ARG, "vp8l_resolve: bad arguments");
    k_vp8l_expand<<<dim3(unsigned(npieces), 16), 256, 0, st>>>(pieces, xsize, npix, out, src, err);
    GSX_KERNEL_CHECK();
    if (cache_bits) {
        k_vp8l_replay<<<1, 32, 0, st>>>(out, src, npix, cache_bits);
        GSX_KERNEL_CHECK();
        return GSX_OK;
    }
    for (int64_t k = 1; k <= 2 * npix; k *= 2) {
        k_vp8l_jump<<<grid_for(npix), 256, 0, st>>>(out, src, npix);
        GSX_KERNEL_CHECK();
    }
    return GSX_OK;
}

int gsx_vp8l_inverse(int32_t type, const uint32_t* in, uint32_t* out, const uint32_t* sub, int64_t xs, int64_t height,
                     int32_t bits, int32_t* scratch, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_vp8l_inverse");
    GSX_REQUIRE(type >= 0 && type <= 3 && in && out && xs > 0 && height > 0 && bits >= 0 && bits <= 9 &&
                    (type == 2 || sub) && (type != 0 || scratch),
                GSX_ERR_ARG, "vp8l_inverse: bad arguments");
    const int64_t n = xs * height;
    if (type == 3) {
        k_vp8l_index<<<grid_for(n), 256, 0, st>>>(in, out, sub, xs, height, bits);
    } else if (type == 2) {
        k_vp8l_green<<<grid_for(n), 256, 0, st>>>(out, n);
    } else if (type == 1) {
        k_vp8l_cross<<<grid_for(n), 256, 0, st>>>(out, sub, xs, height, bits);
    } else {
        const int64_t warps = (height + 31) / 32;
        GSX_CUDA_CHECK(cudaMemsetAsync(scratch, 0, sizeof(int32_t) * (warps + 1), st));
        k_vp8l_predict<<<unsigned(warps), 32, 0, st>>>(out, sub, xs, height, bits, scratch, scratch + 1);
    }
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_vp8l_rgba(const uint32_t* argb, uint8_t* rgba, int64_t n, int32_t alpha, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_NVTX("gsx_vp8l_rgba");
    GSX_REQUIRE(argb && rgba && n > 0, GSX_ERR_ARG, "vp8l_rgba: bad arguments");
    k_vp8l_rgba<<<grid_for(n), 256, 0, st>>>(argb, (uint32_t*)rgba, n, alpha);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

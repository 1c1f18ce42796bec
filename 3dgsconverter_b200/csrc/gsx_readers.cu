// gsx_readers.cu -- the .splat, .ksplat, .spz and compressed PLY readers' per-splat decoding for sm_90a (H100).
//
//   k_splat_decode   splat.py:9-80 (SplatFormat.read): 32-byte records -> rows of define_dtype(has_rgb=True,
//                    sh_degree=0); scales log(max(s, 1e-6)) (numpy_logf), rotations renormalised, nx/ny/nz and
//                    red/green/blue left 0 as the reference leaves them.
//   k_ksplat_decode  ksplat.py:109-264 for one section: interleaved records of level 0 (float32), 1 (float16, uint16
//                    positions against the bucket centre) or >= 2 (uint8 SH); the bucket of splat i is i / bucketSize
//                    in the full buckets, then found in the prefix sums of the partially-filled bucket lengths.
//   k_spz_decode     spz.py:175-296 (_read_body): the planar body of versions 1 (float16 positions, first-three
//                    rotations), 2 (24-bit positions) and 3 (smallest-three rotations in float64), SH de-interleaved.
//   k_cply_decode    compressed_ply.py:14-123, 342-378: the chunk bounds of splat i / 256, 11-10-11 and 8-8-8-8
//                    de-normalisation and the 2-10-10-10 quaternion in float64, rounded once to float32 on store.
//
// Each kernel writes rows in the exact byte layout of the structured array the reference reader returns.  128 threads
// (4 warps) per CTA, one splat per thread: the CTA loads its 128 input records (or the slices of the planar sections)
// into shared memory as the 16-byte words that cover them, each thread builds its row in a shared staging buffer, and
// the CTA stores the rows as 16-byte words whatever the alignment (gsx_staged.cuh).  Rows wider than kStageMax with a
// run of always-zero SH columns (SH degrees above 3) stage only the bytes around that run; the caller zero-fills the
// output first.
//
// Every map of one input byte (opacity logit, DC, RGB, SH, SPZ scale) is a 256-entry float32 table the caller builds
// with the reference's own NumPy expression on the host, so NumPy's float32 and float64 log are reproduced without
// restating them.  All other arithmetic is one __f*_rn / __d*_rn operation per NumPy operation in the reference's
// order and precision (gsx_numpy_scalar.cuh), with x86's NaN results where NaN inputs can reach the output.
#include "../../include/gsx.h"

#include "gsx_bits.cuh"
#include "gsx_common.cuh"
#include "gsx_numpy_scalar.cuh"
#include "gsx_staged.cuh"

namespace gsx {

namespace {

constexpr int kRows = 128;   // rows per CTA
constexpr int kMaxPlySh = 64;
constexpr int kStageMax = 256;   // rows up to this width are staged whole, zero columns included
constexpr size_t kSmemMax = 200 * 1024;

// the Python float constants of the readers, rounded to float32 as NumPy 2 rounds a weak scalar
constexpr float kEps6 = (float)1e-6;
constexpr float kSqrt2 = (float)1.41421356;
constexpr float kSqrt1_2 = (float)0.707106781186547524401;

// staged row width `crow`, of which the first `head` bytes precede the zero run; output rows of row_bytes bytes
struct RowOut {
    int32_t crow, head;
    int64_t row_bytes;
};

__device__ __forceinline__ void store_rows(uint8_t* __restrict__ out, int64_t base, int rows_here, const uint8_t* stage,
                                           const RowOut& o) {
    if (o.row_bytes == o.crow) store_staged(out + base * o.crow, stage, rows_here * o.crow);
    else store_rows_gap(out + base * o.row_bytes, stage, rows_here, o.crow, o.head, o.row_bytes);
}

__device__ __forceinline__ void load_tables(float* tab, const float* __restrict__ tables, int ntab) {
    for (int i = threadIdx.x; i < ntab * 256; i += blockDim.x) tab[i] = __ldg(tables + i);
}

// ---------------------------------------------------------------------------------------------------------- .splat
// tables: DC (splat.py:75-77), opacity logit (:67-69)
__global__ void __launch_bounds__(kRows) k_splat_decode(const uint8_t* __restrict__ in, int64_t n,
                                                        const float* __restrict__ tables, uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float tab[2 * 256];
    load_tables(tab, tables, 2);
    const int t = threadIdx.x;
    const int64_t base = (int64_t)blockIdx.x * kRows;
    const int rows_here = (int)(n - base < kRows ? n - base : kRows);
    const uint8_t* rin = load_staged(smem, in + base * 32, rows_here * 32);
    uint8_t* stage = smem + up16(kRows * 32 + 16);
    __syncthreads();
    if (t < rows_here) {
        const uint8_t* r = rin + t * 32;
        uint8_t* p = stage + t * 71;
        for (int a = 0; a < 3; ++a) put32(p + 4 * a, get32(r + 4 * a));
        for (int a = 12; a < 24; ++a) p[a] = 0;   // nx, ny, nz
        p += 24;
        for (int a = 0; a < 3; ++a) putf(p, tab[r[24 + a]]);
        putf(p, tab[256 + r[27]]);
        for (int a = 0; a < 3; ++a) {   // np.log(np.maximum(s, 1e-6)); np.maximum keeps NaN
            const float s = getf(r + 12 + 4 * a);
            putf(p, numpy_logf(s != s ? s : fmaxf(s, kEps6)));
        }
        float q[4];   // (u8 - 128) / 128.0, renormalised by max(sqrt(r0**2 + r1**2 + r2**2 + r3**2), 1e-6)
        for (int a = 0; a < 4; ++a) q[a] = __fdiv_rn(__fsub_rn((float)r[28 + a], 128.f), 128.f);
        float ss = __fmul_rn(q[0], q[0]);
        for (int a = 1; a < 4; ++a) ss = __fadd_rn(ss, __fmul_rn(q[a], q[a]));
        const float norm = fmaxf(__fsqrt_rn(ss), kEps6);
        for (int a = 0; a < 4; ++a) putf(p, __fdiv_rn(q[a], norm));
        p[0] = p[1] = p[2] = 0;   // red, green, blue
    }
    __syncthreads();
    store_staged(out + base * 71, stage, rows_here * 71);
}

// ---------------------------------------------------------------------------------------------------------- .ksplat
struct KsplatSection {
    const uint8_t* rec;       // the section's first record
    const uint8_t* centres;   // bucket centres, float32 [ncentres, 3] at any 4-byte offset
    const int64_t* pend;      // prefix sums of the partially-filled bucket lengths [npart]
    int64_t n, full, bucket_size, fb;   // splats; splats in full buckets (fb * bucket_size); full buckets
    int32_t npart, level, sh_count, rec_bytes;
    float sr, sf;             // float32(compressionScaleRange), float32((bucketBlockSize / 2.0) / range)
};

// tables: DC, opacity logit (ksplat.py:229-234, 24-27), level >= 2 SH (:257-258)
__global__ void __launch_bounds__(kRows) k_ksplat_decode(const KsplatSection s, const float* __restrict__ tables,
                                                         const RowOut o, uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float tab[3 * 256];
    load_tables(tab, tables, 3);
    const int t = threadIdx.x, rb = s.rec_bytes;
    const int64_t base = (int64_t)blockIdx.x * kRows;
    const int rows_here = (int)(s.n - base < kRows ? s.n - base : kRows);
    const uint8_t* rin = load_staged(smem, s.rec + base * rb, rows_here * rb);
    uint8_t* stage = smem + up16((size_t)kRows * rb + 16);
    __syncthreads();
    if (t < rows_here) {
        const uint8_t* r = rin + t * rb;
        uint8_t* p = stage + t * o.crow;
        const uint8_t *col, *shp;
        float pos[3], scl[3], rot[4];
        if (s.level == 0) {
            for (int a = 0; a < 3; ++a) pos[a] = getf(r + 4 * a), scl[a] = getf(r + 12 + 4 * a);
            for (int a = 0; a < 4; ++a) rot[a] = getf(r + 24 + 4 * a);
            col = r + 40, shp = r + 44;
        } else {
            const int64_t i = base + t;
            int64_t b;
            if (i < s.full) {
                b = i / s.bucket_size;
            } else {   // first partial bucket whose prefix end exceeds i - full
                const int64_t j = i - s.full;
                int lo = 0, hi = s.npart - 1;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (__ldg(s.pend + mid) > j) hi = mid;
                    else lo = mid + 1;
                }
                b = s.fb + lo;
            }
            for (int a = 0; a < 3; ++a) {   // (float32(u16) - sr) * sf + centre
                const float c = __uint_as_float((uint32_t)__ldg(s.centres + 12 * b + 4 * a) |
                                                (uint32_t)__ldg(s.centres + 12 * b + 4 * a + 1) << 8 |
                                                (uint32_t)__ldg(s.centres + 12 * b + 4 * a + 2) << 16 |
                                                (uint32_t)__ldg(s.centres + 12 * b + 4 * a + 3) << 24);
                pos[a] = x86_add(x86_mul(__fsub_rn((float)get16(r + 2 * a), s.sr), s.sf), c);
                scl[a] = numpy_h2f(get16(r + 6 + 2 * a));
            }
            for (int a = 0; a < 4; ++a)   // ((u - 32767.5) / 32767.5) * 1.41421356
                rot[a] = __fmul_rn(__fdiv_rn(__fsub_rn((float)get16(r + 12 + 2 * a), 32767.5f), 32767.5f), kSqrt2);
            col = r + 20, shp = r + 24;
        }
        for (int a = 0; a < 3; ++a) putf(p, pos[a]);
        for (int a = 0; a < 12; ++a) p[a] = 0;   // nx, ny, nz
        p += 12;
        for (int a = 0; a < 3; ++a) putf(p, tab[col[a]]);
        for (int k = 0; k < s.sh_count; ++k)
            putf(p, s.level == 0 ? getf(shp + 4 * k) : s.level == 1 ? numpy_h2f(get16(shp + 2 * k)) : tab[512 + shp[k]]);
        while (p < stage + t * o.crow + o.head) *p++ = 0;   // SH columns this section does not store
        putf(p, tab[256 + col[3]]);
        for (int a = 0; a < 3; ++a) putf(p, scl[a]);
        for (int a = 0; a < 4; ++a) putf(p, rot[a]);
    }
    __syncthreads();
    store_rows(out, base, rows_here, stage, o);
}

// ---------------------------------------------------------------------------------------------------------- .spz
// tables: opacity logit (spz.py:345-348), DC (:207-209), red/green/blue (:213-216), scale (:222), SH (:243)
__global__ void __launch_bounds__(kRows) k_spz_decode(const uint8_t* __restrict__ body, int64_t n, int version,
                                                      int sh_dim, float pos_div, const float* __restrict__ tables,
                                                      const RowOut o, uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float tab[5 * 256];
    load_tables(tab, tables, 5);
    const int t = threadIdx.x;
    const int pb = version == 1 ? 6 : 9, rb = version >= 3 ? 4 : 3, shb = 3 * sh_dim;
    const int64_t base = (int64_t)blockIdx.x * kRows;
    const int rows_here = (int)(n - base < kRows ? n - base : kRows);
    const int64_t off_a = n * pb, off_c = off_a + n, off_s = off_c + 3 * n, off_r = off_s + 3 * n, off_h = off_r + n * rb;
    uint8_t* st = smem;
    const uint8_t* s_pos = load_staged(st, body + base * pb, rows_here * pb);
    st += up16(kRows * pb + 16);
    const uint8_t* s_a = load_staged(st, body + off_a + base, rows_here);
    st += up16(kRows + 16);
    const uint8_t* s_c = load_staged(st, body + off_c + base * 3, rows_here * 3);
    st += up16(kRows * 3 + 16);
    const uint8_t* s_s = load_staged(st, body + off_s + base * 3, rows_here * 3);
    st += up16(kRows * 3 + 16);
    const uint8_t* s_r = load_staged(st, body + off_r + base * rb, rows_here * rb);
    st += up16(kRows * rb + 16);
    const uint8_t* s_h = shb ? load_staged(st, body + off_h + base * shb, rows_here * shb) : nullptr;
    st += up16((size_t)kRows * shb + 16);
    uint8_t* stage = st;
    __syncthreads();
    if (t < rows_here) {
        uint8_t* p = stage + t * o.crow;
        for (int a = 0; a < 3; ++a) {
            if (version == 1) {
                putf(p, numpy_h2f(get16(s_pos + t * 6 + 2 * a)));
            } else {   // sign-extended int24 as float32 / (1 << frac_bits)
                const uint8_t* q = s_pos + t * 9 + 3 * a;
                int32_t v = (int32_t)((uint32_t)q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16);
                if (v & 0x800000) v |= (int32_t)0xff000000u;
                putf(p, __fdiv_rn((float)v, pos_div));
            }
        }
        for (int a = 0; a < 12; ++a) p[a] = 0;   // nx, ny, nz
        p += 12;
        for (int a = 0; a < 3; ++a) putf(p, tab[256 + s_c[t * 3 + a]]);
        for (int c = 0; c < 3; ++c)   // f_rest_{j + c * dim} = channel c of coefficient j
            for (int j = 0; j < sh_dim; ++j) putf(p, tab[1024 + s_h[t * shb + 3 * j + c]]);
        putf(p, tab[s_a[t]]);
        for (int a = 0; a < 3; ++a) putf(p, tab[768 + s_s[t * 3 + a]]);
        float q[4];   // rot_0 .. rot_3 = w, x, y, z
        if (version >= 3) {   // smallest three: the three others in slots 20, 10, 0, the largest from the norm in float64
            const uint32_t w = get32(s_r + t * 4);
            const int big = (int)(w >> 30);
            double v[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {   // (mag / 511.0 as float32) * SQRT1_2 * (1.0 - 2.0 * neg)
                const uint32_t c = w >> (20 - 10 * k) & 0x3ffu;
                const double f = (double)__fmul_rn(__fdiv_rn((float)(c & 0x1ffu), 511.f), kSqrt1_2);
                v[k] = c >> 9 ? -f : f;
            }
            const double s2 = __dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2]));
            const double m = __dsqrt_rn(fmax(0.0, __dadd_rn(1.0, -s2)));
            float xyzw[4];   // component i != big holds v[i - (i > big)]
#pragma unroll
            for (int i = 0; i < 4; ++i)
                xyzw[i] = i == big ? __double2float_rn(m) : (float)(i - (i > big) == 0 ? v[0] : i - (i > big) == 1 ? v[1] : v[2]);
            q[0] = xyzw[3], q[1] = xyzw[0], q[2] = xyzw[1], q[3] = xyzw[2];
        } else {   // first three: u8 / 127.5 - 1.0, w = sqrt(max(0, 1 - sum(xyz**2)))
            for (int a = 0; a < 3; ++a) q[1 + a] = __fsub_rn(__fdiv_rn((float)s_r[t * 3 + a], 127.5f), 1.f);
            const float s2 = __fadd_rn(__fadd_rn(__fmul_rn(q[1], q[1]), __fmul_rn(q[2], q[2])), __fmul_rn(q[3], q[3]));
            q[0] = __fsqrt_rn(fmaxf(0.f, __fsub_rn(1.f, s2)));
        }
        for (int a = 0; a < 4; ++a) putf(p, q[a]);
        for (int a = 0; a < 3; ++a) p[a] = (uint8_t)tab[512 + s_c[t * 3 + a]];
    }
    __syncthreads();
    store_rows(out, base, rows_here, stage, o);
}

// ---------------------------------------------------------------------------------------------------------- compressed PLY
struct CplyLayout {
    int32_t vrow, voff[4];            // vertex row bytes; packed_position, _rotation, _scale, _color
    int32_t crow, coff[18];           // chunk row bytes; min_x .. max_b in CHUNK_DTYPE order
    int32_t srow, soff[kMaxPlySh];    // sh row bytes; the uchar properties in file order
    int32_t nsh;
};

// (nv / t) * (v_max - v_min) + v_min: the bound difference in float32 (NumPy scalars), the rest in float64
__device__ __forceinline__ double cply_denorm(uint32_t nv, double t, float lo, float hi) {
    return x86_add(x86_mul(__ddiv_rn((double)nv, t), x86_f2d(x86_sub(hi, lo))), x86_f2d(lo));
}

// tables: opacity logit (compressed_ply.py:113-115, float64), SH (:121-122)
__global__ void __launch_bounds__(kRows) k_cply_decode(const uint8_t* __restrict__ chunk, int64_t nchunk,
                                                       const uint8_t* __restrict__ vertex, const uint8_t* __restrict__ sh,
                                                       int64_t n, const CplyLayout L, const float* __restrict__ tables,
                                                       uint8_t* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float tab[2 * 256];
    __shared__ float bnd[18];
    __shared__ int32_t soff[kMaxPlySh];
    load_tables(tab, tables, 2);
    const int t = threadIdx.x, crow = 4 * (17 + L.nsh);
    for (int k = t; k < L.nsh; k += kRows) soff[k] = L.soff[k];
    const int64_t base = (int64_t)blockIdx.x * kRows, ci = base / 256;   // 256 % kRows == 0: one chunk per CTA
    const int rows_here = (int)(n - base < kRows ? n - base : kRows);
    const bool have_chunk = ci < nchunk;
    if (have_chunk && t < 18) bnd[t] = getf(chunk + ci * L.crow + L.coff[t]);
    uint8_t* st = smem;
    const uint8_t* s_v = have_chunk ? load_staged(st, vertex + base * L.vrow, rows_here * L.vrow) : nullptr;
    st += up16((size_t)kRows * L.vrow + 16);
    const uint8_t* s_h = have_chunk && L.nsh ? load_staged(st, sh + base * L.srow, rows_here * L.srow) : nullptr;
    st += L.nsh ? up16((size_t)kRows * L.srow + 16) : 0;
    uint8_t* stage = st;
    __syncthreads();
    if (t < rows_here) {
        uint8_t* p = stage + t * crow;
        if (!have_chunk) {   // rows past len(chunks) * 256 stay zero
            for (int k = 0; k < crow; ++k) p[k] = 0;
        } else {
            const uint8_t* v = s_v + t * L.vrow;
            const uint32_t pp = get32(v + L.voff[0]), pr = get32(v + L.voff[1]), ps = get32(v + L.voff[2]),
                           pc = get32(v + L.voff[3]);
            const uint32_t npos[3] = {pp >> 21 & 0x7ffu, pp >> 11 & 0x3ffu, pp & 0x7ffu};
            const uint32_t nscl[3] = {ps >> 21 & 0x7ffu, ps >> 11 & 0x3ffu, ps & 0x7ffu};
#pragma unroll
            for (int a = 0; a < 3; ++a) putf(p, x86_d2f(cply_denorm(npos[a], a == 1 ? 1023.0 : 2047.0, bnd[a], bnd[3 + a])));
            for (int a = 0; a < 12; ++a) p[a] = 0;   // nx, ny, nz
            p += 12;
            for (int a = 0; a < 3; ++a) {   // (c - 0.5) / SH_C0 on the float64 colour
                const double c = cply_denorm(pc >> (24 - 8 * a) & 0xffu, 255.0, bnd[12 + a], bnd[15 + a]);
                putf(p, x86_d2f(x86_div(x86_sub(c, 0.5), 0.28209479177387814)));
            }
            putf(p, tab[pc & 0xffu]);
#pragma unroll
            for (int a = 0; a < 3; ++a) putf(p, x86_d2f(cply_denorm(nscl[a], a == 1 ? 1023.0 : 2047.0, bnd[6 + a], bnd[9 + a])));
            double d[3];   // (nv / 1023.0 - 0.5) / SQRT2_2; missing = sqrt(clip(1 - (d0**2 + d1**2 + d2**2), 0, 1))
#pragma unroll
            for (int k = 0; k < 3; ++k)
                d[k] = __ddiv_rn(__dadd_rn(__ddiv_rn((double)(pr >> (20 - 10 * k) & 0x3ffu), 1023.0), -0.5),
                                 0.7071067811865476);
            const double s2 = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
            const double m = __dsqrt_rn(fmin(fmax(__dadd_rn(1.0, -s2), 0.0), 1.0));
            const int big = (int)(pr >> 30);
#pragma unroll
            for (int i = 0; i < 4; ++i)   // component i != big holds d[i - (i > big)]
                putf(p, __double2float_rn(i == big ? m : i - (i > big) == 0 ? d[0] : i - (i > big) == 1 ? d[1] : d[2]));
            for (int k = 0; k < L.nsh; ++k) putf(p, tab[256 + s_h[t * L.srow + soff[k]]]);
        }
    }
    __syncthreads();
    store_staged(out + base * crow, stage, rows_here * crow);
}

// --------------------------------------------------------------------------------------------------------- host side
int check_rows(int64_t n, const char* who) {
    GSX_REQUIRE(n >= 0, GSX_ERR_ARG, "%s: n=%lld < 0", who, (long long)n);
    GSX_REQUIRE(n < 2147483648ll, GSX_ERR_UNSUPPORTED, "%s: n=%lld needs n < 2^31", who, (long long)n);
    return GSX_OK;
}

template <typename K>
int set_smem(K kernel, size_t smem, const char* who) {
    GSX_REQUIRE(smem <= kSmemMax, GSX_ERR_UNSUPPORTED, "%s: %zu bytes of shared memory per CTA", who, smem);
    if (smem > 48 * 1024) GSX_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                              (int)smem));
    return GSX_OK;
}

// rows with a zero run stage only the bytes around it, into zero-filled output
int prepare_out(uint8_t* out, int64_t n, const RowOut& o, cudaStream_t st) {
    if (o.row_bytes != o.crow) GSX_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)n * o.row_bytes, st));
    return GSX_OK;
}

int grid(int64_t n) { return (int)((n + kRows - 1) / kRows); }

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_splat_decode(const uint8_t* data, int64_t n, const float* tables, uint8_t* rows, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_rows(n, "splat_decode");
    if (rc) return rc;
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(data && tables && rows, GSX_ERR_ARG, "splat_decode: null device pointer");
    const size_t smem = up16(kRows * 32 + 16) + (size_t)kRows * 71 + 16;
    k_splat_decode<<<grid(n), kRows, smem, st>>>(data, n, tables, rows);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_ksplat_decode_section(const uint8_t* rec, int64_t n, int32_t level, int32_t sh_count, float sr, float sf,
                              const uint8_t* centres, int64_t ncentres, int64_t full_buckets, int64_t bucket_size,
                              const int64_t* partial_end, int32_t npartial, const float* tables, int32_t row_bytes,
                              uint8_t* rows, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_rows(n, "ksplat_decode_section");
    if (rc) return rc;
    GSX_REQUIRE(level >= 0 && level <= 2, GSX_ERR_ARG, "ksplat_decode_section: level %d (0, 1, or 2 for any >= 2)",
                level);
    GSX_REQUIRE(sh_count == 0 || sh_count == 9 || sh_count == 24, GSX_ERR_ARG, "ksplat_decode_section: sh_count %d",
                sh_count);
    GSX_REQUIRE(row_bytes >= 4 * (17 + sh_count) && row_bytes % 4 == 0, GSX_ERR_ARG,
                "ksplat_decode_section: %d-byte rows cannot hold %d SH values", row_bytes, sh_count);
    GSX_REQUIRE(full_buckets >= 0 && bucket_size >= 0 && npartial >= 0 && ncentres >= 0, GSX_ERR_ARG,
                "ksplat_decode_section: negative bucket count");
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(rec && tables && rows, GSX_ERR_ARG, "ksplat_decode_section: null device pointer");
    if (level >= 1) {
        // every splat needs a bucket (the host checks the partial lengths cover n) and that bucket a centre
        const int64_t full = full_buckets * bucket_size;
        GSX_REQUIRE(centres && (n <= full || (partial_end && npartial >= 1)), GSX_ERR_ARG,
                    "ksplat_decode_section: splats past the full buckets need partial bucket ends");
        const int64_t last = n <= full ? (n - 1) / bucket_size : full_buckets + npartial - 1;
        GSX_REQUIRE(last < ncentres, GSX_ERR_ARG, "ksplat_decode_section: bucket %lld has no centre (%lld)",
                    (long long)last, (long long)ncentres);
    }
    KsplatSection s{};
    s.rec = rec, s.centres = centres, s.pend = partial_end, s.n = n;
    s.full = full_buckets * bucket_size, s.bucket_size = bucket_size, s.fb = full_buckets, s.npart = npartial;
    s.level = level, s.sh_count = sh_count, s.sr = sr, s.sf = sf;
    s.rec_bytes = level == 0 ? 44 + 4 * sh_count : 24 + (level == 1 ? 2 : 1) * sh_count;
    const int head = 4 * (9 + sh_count);
    RowOut o{head + 32, head, row_bytes};
    const bool whole = row_bytes <= kStageMax;
    if (whole) o.crow = row_bytes, o.head = row_bytes - 32;   // stage the zero columns as well
    if ((rc = prepare_out(rows, n, o, st))) return rc;
    const size_t smem = up16((size_t)kRows * s.rec_bytes + 16) + (size_t)kRows * o.crow + 16;
    if ((rc = set_smem(k_ksplat_decode, smem, "ksplat_decode_section"))) return rc;
    k_ksplat_decode<<<grid(n), kRows, smem, st>>>(s, tables, o, rows);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_spz_decode(const uint8_t* body, int64_t n, int32_t version, int32_t sh_dim, int32_t frac_bits,
                   const float* tables, int32_t row_bytes, uint8_t* rows, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_rows(n, "spz_decode");
    if (rc) return rc;
    GSX_REQUIRE(version >= 1 && version <= 3, GSX_ERR_ARG, "spz_decode: version %d", version);
    GSX_REQUIRE(sh_dim == 0 || sh_dim == 3 || sh_dim == 8 || sh_dim == 15, GSX_ERR_ARG, "spz_decode: sh_dim %d", sh_dim);
    GSX_REQUIRE(frac_bits >= 0 && frac_bits <= 127, GSX_ERR_ARG,
                "spz_decode: 1 << %d is not a finite float32", frac_bits);
    GSX_REQUIRE(row_bytes >= 4 * (17 + 3 * sh_dim) + 3 && (row_bytes - 3) % 4 == 0, GSX_ERR_ARG,
                "spz_decode: %d-byte rows cannot hold %d SH values", row_bytes, 3 * sh_dim);
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(body && tables && rows, GSX_ERR_ARG, "spz_decode: null device pointer");
    const int head = 4 * (9 + 3 * sh_dim);
    RowOut o{head + 35, head, row_bytes};
    if ((rc = prepare_out(rows, n, o, st))) return rc;
    const int pb = version == 1 ? 6 : 9, rb = version >= 3 ? 4 : 3;
    const size_t smem = up16(kRows * pb + 16) + up16(kRows + 16) + 2 * up16(kRows * 3 + 16) + up16(kRows * rb + 16) +
                        up16((size_t)kRows * 3 * sh_dim + 16) + (size_t)kRows * o.crow + 16;
    if ((rc = set_smem(k_spz_decode, smem, "spz_decode"))) return rc;
    k_spz_decode<<<grid(n), kRows, smem, st>>>(body, n, version, sh_dim, ldexpf(1.f, frac_bits), tables, o, rows);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

int gsx_cply_decode(const uint8_t* chunk, int64_t nchunk, int32_t chunk_row, const int32_t* chunk_offs,
                    const uint8_t* vertex, int64_t n, int32_t vertex_row, const int32_t* vertex_offs, const uint8_t* sh,
                    int32_t sh_row, const int32_t* sh_offs, int32_t nsh, const float* tables, uint8_t* rows,
                    void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_rows(n, "cply_decode");
    if (rc) return rc;
    GSX_REQUIRE(nchunk >= 0, GSX_ERR_ARG, "cply_decode: nchunk < 0");
    GSX_REQUIRE(nsh >= 0 && nsh <= kMaxPlySh, GSX_ERR_ARG, "cply_decode: %d SH properties (at most %d)", nsh, kMaxPlySh);
    GSX_REQUIRE(chunk_offs && vertex_offs && (nsh == 0 || sh_offs), GSX_ERR_ARG, "cply_decode: no offset table");
    GSX_REQUIRE(chunk_row >= 72 && chunk_row <= 1024 && vertex_row >= 16 && vertex_row <= 1024 &&
                    (nsh == 0 || (sh_row >= nsh && sh_row <= 1024)),
                GSX_ERR_ARG, "cply_decode: row sizes %d / %d / %d outside the supported range", chunk_row, vertex_row,
                sh_row);
    CplyLayout L{};
    L.crow = chunk_row, L.vrow = vertex_row, L.srow = nsh ? sh_row : 0, L.nsh = nsh;
    for (int k = 0; k < 18; ++k) {
        GSX_REQUIRE(chunk_offs[k] >= 0 && chunk_offs[k] + 4 <= chunk_row, GSX_ERR_ARG,
                    "cply_decode: chunk property %d at byte %d outside the row", k, chunk_offs[k]);
        L.coff[k] = chunk_offs[k];
    }
    for (int k = 0; k < 4; ++k) {
        GSX_REQUIRE(vertex_offs[k] >= 0 && vertex_offs[k] + 4 <= vertex_row, GSX_ERR_ARG,
                    "cply_decode: vertex property %d at byte %d outside the row", k, vertex_offs[k]);
        L.voff[k] = vertex_offs[k];
    }
    for (int k = 0; k < nsh; ++k) {
        GSX_REQUIRE(sh_offs[k] >= 0 && sh_offs[k] < sh_row, GSX_ERR_ARG,
                    "cply_decode: sh property %d at byte %d outside the row", k, sh_offs[k]);
        L.soff[k] = sh_offs[k];
    }
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(vertex && tables && rows && (nchunk == 0 || chunk) && (nsh == 0 || sh), GSX_ERR_ARG,
                "cply_decode: null device pointer");
    const size_t smem = up16((size_t)kRows * vertex_row + 16) + (nsh ? up16((size_t)kRows * sh_row + 16) : 0) +
                        (size_t)kRows * 4 * (17 + nsh) + 16;
    if ((rc = set_smem(k_cply_decode, smem, "cply_decode"))) return rc;
    k_cply_decode<<<grid(n), kRows, smem, st>>>(chunk, nchunk, vertex, sh, n, L, tables, rows);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

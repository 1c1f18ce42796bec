// gsx_ply.cu -- the plain PLY readers' and writers' row transcode for sm_90a (H100): formats/ply_3dgs.py and
// formats/ply_cc.py map each field of a structured array to a field of another (`converted[t] = vertices[s]` in read,
// `output_data[o] = data[f]` in write) and leave every other field 0.  One kernel does that for both readers and both
// writers: contiguous rows of one byte layout in, contiguous rows of another out.
//
//   k_ply_transcode  a CTA owns kRows rows, a contiguous byte range in the source and in the destination.  It loads the
//                    source tile into shared memory as the 16-byte words that cover it (load_staged), zeroes the
//                    destination tile, writes every (row, field) pair of the tile with one thread each (the warp's
//                    lanes walk rows of the same field), and stores the tile as 16-byte words (store_staged).
//
// Casts, each what NumPy's structured-field assignment gives on x86:
//   identity (any PLY type)    the bytes, copied
//   integer -> f4               round to nearest (exact below 2^24)
//   f8 -> f4                    round to nearest, x86's NaN rule (cvtsd2ss: quieted, high payload bits kept)
//   integer -> u1               the low byte
//   f4 / f8 -> u1               cvttss2si / cvttsd2si to int32, then the low byte: NaN and values whose truncation is
//                               outside int32 give 0.  NumPy's strided and contiguous loops agree on every float32
//                               pattern and on the float64 edges (DESIGN 4.8).
// Every other pairing is refused.  Field offsets may be any byte; rows up to kRowMax bytes.
#include "../../include/gsx.h"

#include "gsx_bits.cuh"
#include "gsx_common.cuh"
#include "gsx_numpy_scalar.cuh"
#include "gsx_staged.cuh"

namespace gsx {

namespace {

constexpr int kRows = 64;          // rows per CTA
constexpr int kThreads = 256;
constexpr int kRowMax = 1024;      // source and destination rows, bytes
constexpr int kMaxFields = 1024;   // at most one field per destination byte

// PLY property types, as gsx.ply numbers them
enum PlyType : uint8_t { kI1, kU1, kI2, kU2, kI4, kU4, kF4, kF8, kNumTypes };
constexpr int kWidth[kNumTypes] = {1, 1, 2, 2, 4, 4, 4, 8};

struct PlyField {
    int16_t src_off, dst_off;
    uint8_t src_t, dst_t, src_w, dst_w;
};
struct PlyFields {   // a kernel parameter (8 KB), copied to shared memory by every CTA
    PlyField f[kMaxFields];
};

__host__ __device__ constexpr bool is_int(int t) { return t <= kU4; }

__host__ __device__ constexpr bool supported(int s, int d) {
    return s == d || (d == kF4 && (is_int(s) || s == kF8)) || d == kU1;
}

__device__ __forceinline__ uint64_t get_le(const uint8_t* p, int w) {
    uint64_t v = 0;
    for (int i = 0; i < w; ++i) v |= (uint64_t)p[i] << (8 * i);
    return v;
}
__device__ __forceinline__ void put_le(uint8_t* p, uint64_t v, int w) {
    for (int i = 0; i < w; ++i) p[i] = (uint8_t)(v >> (8 * i));
}

__device__ __forceinline__ float int_to_f4(uint64_t v, int t) {
    switch (t) {
        case kI1: return (float)(int8_t)v;
        case kU1: return (float)(uint8_t)v;
        case kI2: return (float)(int16_t)v;
        case kU2: return (float)(uint16_t)v;
        case kI4: return __int2float_rn((int32_t)v);
        default: return __uint2float_rn((uint32_t)v);
    }
}

// cvttsd2si to int32, low byte: 0 for NaN and for values whose truncation is outside int32
__device__ __forceinline__ uint8_t f8_to_u1(double v) {
    return (v > -2147483649.0 && v < 2147483648.0) ? (uint8_t)(uint32_t)(int32_t)v : 0;
}

__device__ __forceinline__ void transcode_one(const uint8_t* s, uint8_t* d, const PlyField& f) {
    const uint64_t v = get_le(s, f.src_w);
    if (f.src_t == f.dst_t) {
        put_le(d, v, f.dst_w);
    } else if (f.dst_t == kF4) {
        const float r = f.src_t == kF8 ? x86_d2f(__longlong_as_double((long long)v)) : int_to_f4(v, f.src_t);
        put_le(d, __float_as_uint(r), 4);
    } else {   // u1
        d[0] = f.src_t == kF4   ? np_u8(__uint_as_float((uint32_t)v))
               : f.src_t == kF8 ? f8_to_u1(__longlong_as_double((long long)v))
                                : (uint8_t)v;
    }
}

__global__ void __launch_bounds__(kThreads) k_ply_transcode(const uint8_t* __restrict__ src, int64_t n, int32_t src_row,
                                                            uint8_t* __restrict__ dst, int32_t dst_row, const PlyFields T,
                                                            int32_t nf) {
    extern __shared__ __align__(16) uint8_t smem[];
    PlyField* tab = reinterpret_cast<PlyField*>(smem);
    uint8_t* s_in = smem + up16((size_t)nf * sizeof(PlyField));
    uint8_t* s_out = s_in + up16((size_t)kRows * src_row + 16);
    const int64_t base = (int64_t)blockIdx.x * kRows;
    const int rows_here = (int)(n - base < kRows ? n - base : kRows);
    const int out_bytes = rows_here * dst_row;
    for (int k = threadIdx.x; k < nf; k += kThreads) tab[k] = T.f[k];
    const uint8_t* in = load_staged(s_in, src + base * src_row, rows_here * src_row);
    uint4* z = reinterpret_cast<uint4*>(s_out);
    for (int v = threadIdx.x; v < (out_bytes + 15) >> 4; v += kThreads) z[v] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    for (int e = threadIdx.x; e < nf * rows_here; e += kThreads) {
        const int k = e / rows_here, r = e - k * rows_here;
        const PlyField f = tab[k];
        transcode_one(in + r * src_row + f.src_off, s_out + r * dst_row + f.dst_off, f);
    }
    __syncthreads();
    store_staged(dst + base * dst_row, s_out, out_bytes);
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_ply_transcode(const uint8_t* src, int64_t n, int32_t src_row, uint8_t* dst, int32_t dst_row,
                      const int32_t* fields, int32_t nf, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GSX_REQUIRE(n >= 0, GSX_ERR_ARG, "ply_transcode: n=%lld < 0", (long long)n);
    GSX_REQUIRE(n < 2147483648ll, GSX_ERR_UNSUPPORTED, "ply_transcode: n=%lld needs n < 2^31", (long long)n);
    GSX_REQUIRE(src_row >= 1 && src_row <= kRowMax && dst_row >= 1 && dst_row <= kRowMax, GSX_ERR_ARG,
                "ply_transcode: rows of %d / %d bytes (source / destination; 1 .. %d)", src_row, dst_row, kRowMax);
    GSX_REQUIRE(nf >= 0 && nf <= kMaxFields && (nf == 0 || fields), GSX_ERR_ARG,
                "ply_transcode: %d fields (0 .. %d) or no field table", nf, kMaxFields);
    PlyFields T{};
    bool written[kRowMax] = {};
    for (int k = 0; k < nf; ++k) {
        const int32_t so = fields[4 * k], s = fields[4 * k + 1], d_o = fields[4 * k + 2], d = fields[4 * k + 3];
        GSX_REQUIRE(s >= 0 && s < kNumTypes && d >= 0 && d < kNumTypes && supported(s, d), GSX_ERR_ARG,
                    "ply_transcode: field %d: no cast from type %d to type %d", k, s, d);
        GSX_REQUIRE(so >= 0 && so + kWidth[s] <= src_row && d_o >= 0 && d_o + kWidth[d] <= dst_row, GSX_ERR_ARG,
                    "ply_transcode: field %d at bytes %d / %d outside the rows", k, so, d_o);
        for (int b = d_o; b < d_o + kWidth[d]; ++b) {
            GSX_REQUIRE(!written[b], GSX_ERR_ARG, "ply_transcode: field %d overlaps another at destination byte %d", k,
                        b);
            written[b] = true;
        }
        T.f[k] = PlyField{(int16_t)so, (int16_t)d_o, (uint8_t)s, (uint8_t)d, (uint8_t)kWidth[s], (uint8_t)kWidth[d]};
    }
    if (n == 0) return GSX_OK;
    GSX_REQUIRE(src && dst, GSX_ERR_ARG, "ply_transcode: null device pointer");
    const size_t smem = up16((size_t)nf * sizeof(PlyField)) + up16((size_t)kRows * src_row + 16) +
                        (size_t)kRows * dst_row + 16;
    if (smem > 48 * 1024)
        GSX_CUDA_CHECK(cudaFuncSetAttribute(k_ply_transcode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_ply_transcode<<<(unsigned)((n + kRows - 1) / kRows), kThreads, smem, st>>>(src, n, src_row, dst, dst_row, T, nf);
    GSX_KERNEL_CHECK();
    return GSX_OK;
}

}  // extern "C"

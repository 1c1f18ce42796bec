#pragma once
#include "gsx_common.cuh"
namespace gsx {
// Raw DEFLATE (RFC 1951) and CRC-32 over a device byte buffer; the gzip framing is gsx/deflate.py.  Dynamic blocks
// hold literals and, where that is fewer bits, distance-1 copies; each block is planned (histograms, code lengths,
// header) by one CTA, the blocks' bit offsets are scanned, and each block's bits are emitted by one CTA.
constexpr int64_t kDeflateMaxBlock = int64_t(1) << 20;   // a dynamic block covers at most 1 MiB of input
constexpr int64_t kDeflateStoredBlock = 65535;
int64_t deflate_workspace_bytes(int64_t nblocks);
int crc32_trailer(const uint8_t* data, int64_t n, void* ws, int64_t ws_bytes, uint8_t* trailer, cudaStream_t st);
int deflate_stored(const uint8_t* data, int64_t n, uint8_t* out, cudaStream_t st);
int deflate_plan(const uint8_t* data, int64_t n, const int64_t* starts, int64_t nblocks, void* ws, int64_t ws_bytes,
                 uint64_t bit_offset, unsigned long long* total_bits, cudaStream_t st);
int deflate_emit(const uint8_t* data, int64_t n, const int64_t* starts, int64_t nblocks, void* ws, int64_t ws_bytes,
                 uint32_t* words, int64_t nwords, unsigned long long* mismatches, cudaStream_t st);
}

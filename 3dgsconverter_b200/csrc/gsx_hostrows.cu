// gsx_hostrows.cu -- HOST-side row movement around the device filter chain, on several CPU threads (no GPU work).
//
// a1 of the scope table names where the reference's time goes once the masks are cheap: the `np.column_stack` of the
// filter columns (data_processor.py:38,139) and the final `vertices[mask]` fancy-index gather of the 248-byte records
// (:114,149,209,224) -- both single-threaded NumPy passes over 2.5 GB per 10 M splats.  The device-resident record
// mode (gsx_records.cu) avoids them; when the records stay on the host (the default wiring) these two entry points do
// the same passes with every core's memory bandwidth instead of one's.
#include "../../include/gsx.h"

#include "gsx_common.cuh"

#include <algorithm>
#include <atomic>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <vector>

namespace gsx {

namespace {

int host_threads(int64_t work_bytes) {
    const char* e = getenv("GSX_HOST_THREADS");
    int T = e && *e ? atoi(e) : 0;
    if (T <= 0) {
        const unsigned hw = std::thread::hardware_concurrency();
        T = hw >= 32 ? 16 : (hw >= 2 ? (int)hw / 2 : 1);
    }
    const int64_t by_size = work_bytes / (4 << 20) + 1;      // do not spawn threads for a few MiB
    return (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)T, by_size, 64}));
}

template <typename F>
void parallel_rows(int64_t m, int T, F&& body) {   // body(begin, end) on T threads, contiguous slices
    if (T <= 1 || m < 2) {
        body((int64_t)0, m);
        return;
    }
    std::vector<std::thread> th;
    th.reserve((size_t)T - 1);
    for (int t = 1; t < T; ++t) th.emplace_back([&, t] { body(m * t / T, m * (t + 1) / T); });
    body((int64_t)0, m / T);
    for (auto& x : th) x.join();
}

}  // namespace

}  // namespace gsx

using namespace gsx;

extern "C" {

int gsx_host_gather_rows(const void* src, int64_t n_rows, int64_t row_bytes, const int64_t* idx, int64_t m, void* dst) {
    GSX_REQUIRE(n_rows >= 0 && m >= 0 && row_bytes > 0, GSX_ERR_ARG, "host_gather_rows: bad sizes");
    if (m == 0) return GSX_OK;
    GSX_REQUIRE(src && idx && dst, GSX_ERR_ARG, "host_gather_rows: null pointer");
    std::atomic<int64_t> bad{-1};
    const char* s = (const char*)src;
    char* d = (char*)dst;
    parallel_rows(m, host_threads(m * row_bytes), [&](int64_t b, int64_t e) {
        for (int64_t j = b; j < e; ++j) {
            const int64_t i = idx[j];
            if (i < 0 || i >= n_rows) {
                bad.store(j);
                return;
            }
            memcpy(d + j * row_bytes, s + i * row_bytes, (size_t)row_bytes);
        }
    });
    const int64_t bj = bad.load();
    GSX_REQUIRE(bj < 0, GSX_ERR_ARG, "host_gather_rows: idx[%lld] = %lld is outside [0, %lld)", (long long)bj,
                (long long)idx[bj], (long long)n_rows);
    return GSX_OK;
}

int gsx_host_extract_xyz_opacity(const void* src, int64_t n_rows, int64_t row_bytes, int64_t off_x, int64_t off_y,
                                 int64_t off_z, int64_t off_op, float* xyz_out, float* op_out) {
    GSX_REQUIRE(n_rows >= 0 && row_bytes >= 4, GSX_ERR_ARG, "host_extract: bad sizes");
    if (n_rows == 0) return GSX_OK;
    GSX_REQUIRE(src && xyz_out, GSX_ERR_ARG, "host_extract: null pointer");
    const int64_t offs[4] = {off_x, off_y, off_z, off_op};
    for (int a = 0; a < 4; ++a) {
        if (a == 3 && off_op < 0) continue;
        GSX_REQUIRE(offs[a] >= 0 && offs[a] + 4 <= row_bytes, GSX_ERR_ARG, "host_extract: field offset %lld outside the row",
                    (long long)offs[a]);
    }
    GSX_REQUIRE((off_op >= 0) == (op_out != nullptr), GSX_ERR_ARG, "host_extract: opacity offset / output mismatch");
    const char* s = (const char*)src;
    parallel_rows(n_rows, host_threads(n_rows * row_bytes), [&](int64_t b, int64_t e) {
        for (int64_t i = b; i < e; ++i) {
            const char* r = s + i * row_bytes;
            float v[3];
            memcpy(&v[0], r + off_x, 4);      // (fields may sit at any byte offset: no aligned-load assumption)
            memcpy(&v[1], r + off_y, 4);
            memcpy(&v[2], r + off_z, 4);
            xyz_out[3 * i] = v[0];
            xyz_out[3 * i + 1] = v[1];
            xyz_out[3 * i + 2] = v[2];
            if (op_out) memcpy(op_out + i, r + off_op, 4);
        }
    });
    return GSX_OK;
}

}  // extern "C"

/*
 * gsx.h -- C ABI of libgsx.so, the H100-native (sm_90a) backend for the per-point
 * filtering + codebook clustering hot path of francescofugazzi/3dgsconverter.
 *
 * The reference has no FFI of its own (it is pure Python + Taichi); the boundary it
 * exposes is the Python module surface gsconverter.processing.{gpu_ops,data_processor}.
 * Each entry point below names the reference interface it replaces (path:line relative
 * to /root/reference/gsconverter/).  INTEGRATION.md shows the ctypes binding.
 * The Python binding (gsx/_abi.py) is derived from this file: it parses every gsx_* prototype.
 *
 * Conventions
 *   - plain C types only; device pointers are ordinary pointers into CUDA device
 *     memory of the *current* device; `stream` is a cudaStream_t passed as void*
 *     (NULL = default stream).
 *   - every function returns 0 on success, <0 on error (GSX_ERR_*); the message is
 *     available from gsx_last_error() (thread-local).  The Python wrapper turns a
 *     non-zero status into an exception, which preserves the reference's
 *     "GPU exception => caller falls back" convention (data_processor.py:146-153,
 *     gpu_ops.py:40-46).
 *   - the library never owns device memory in the *_device entry points: the caller
 *     provides outputs and one scratch blob whose size comes from *_workspace_bytes.
 *     The *_host convenience entry points take host buffers and manage device memory
 *     internally (cudaMallocAsync), copies included.
 *   - all masks are uint8 (0/1), one byte per point, like numpy bool.
 *   - N < 2^31 - 64 (int32 indices, as in gpu_ops.py:224,233-234).
 */
#ifndef GSX_H
#define GSX_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSX_HASH_I32WRAP 0 /* probe hash with wrapping int32 products: Taichi default_ip (faithful, SURVEY F8) */
#define GSX_HASH_I64 1     /* probe hash with int64 products: what the host table build uses (intended) */

/* ---- library ---------------------------------------------------------------------- */
const char* gsx_last_error(void);
int gsx_version(void);          /* 100*major + minor */
const char* gsx_build_info(void); /* tuning constants of the SOR query kernel ("knn=r02c;epi_smem=1;..."): names the
                                   * build an ncu capture / a bench line was taken with */
int gsx_device_sm_count(void);  /* SMs of the current device (grid sizing), <0 on error */
long long gsx_kernel_launches(void); /* cumulative number of gsx kernels launched by this process */

/* ---- SOR, Taichi semantics: gpu_ops.py:193-263 (filter_sor_gpu) + :98-176 (kernel) - */

/* Scratch needed by gsx_sor_filter_device / the gsx_sor_* stages for n points.  The grid the query kernel reads
 * (sorted positions, bucket table, boxes) is a PREFIX of that blob: gsx_sor_build_from_sorted and
 * gsx_sor_mean_dists[_range] also accept a blob of only gsx_sor_grid_workspace_bytes(n) (no sort buffers) -- what
 * every rank of the distributed build holds for the union cloud. */
int64_t gsx_sor_workspace_bytes(int64_t n);
int64_t gsx_sor_grid_workspace_bytes(int64_t n);

/* gpu_ops.py:203-204: per-axis min/max of xyz[n,3] -> minmax_dev[6] = {minx,miny,minz,maxx,maxy,maxz}.
 * Scratch: the first 24 KiB of ws (any workspace of gsx_sor_workspace_bytes, or a small blob of its own). */
int gsx_sor_minmax(const float* xyz_dev, int64_t n, float* minmax_dev, void* ws, int64_t ws_bytes, void* stream);

/* gpu_ops.py:205-213 on the host (NumPy-2 float32 semantics, powf).  minmax is a HOST array of 6. */
float gsx_sor_cell_size(const float* minmax_host, int64_t n);

/* gpu_ops.py:216-237: grid index, int64 hash mod n, sort by bucket, bucket table.  Fills the
 * workspace with the hash-sorted float4 positions (w = original index), the bucket table and the
 * 32-/1024-point bounding boxes used for exact pruning.  bmin = the 3 minima, cell = cell size. */
int gsx_sor_build(const float* xyz_dev, int64_t n, const float* bmin_host, float cell, void* ws, int64_t ws_bytes,
                  void* stream);

/* Distributed form of gsx_sor_build for a cloud sharded over G processes (one per GPU); the collectives
 * between the stages are the caller's (gsx/dist.py uses NCCL).  Bucket-range ownership: rank o owns the
 * buckets [ceil(o*n_global/G), ceil((o+1)*n_global/G)).
 *  A. local_run:  stable partition of the slab by bucket owner (one radix pass); outputs float4
 *     {x,y,z, bits(idx_base + local index)} grouped by owner and cuts_dev[G+1] = first position of every owner
 *     -> the caller exchanges the groups (all-to-all).
 *  B. merge:      sorts the m received points of this rank's bucket range [bucket_lo, bucket_hi) by (bucket, in-cell Hilbert code)
 *     -> the caller all-gathers the segments in owner order = the globally hash-sorted array.  With flags_sorted_dev
 *     the owner also emits one byte per sorted point (bit 0: starts a bucket, bit 1: other grid cell than the point
 *     before) -- exchanged along with the segment (1 B/pt next to 16 B/pt), it spares every receiving rank the
 *     re-hash of every point in its replicated stage C.
 *  C. build_from_sorted: bucket table ({start,end} per bucket, 8 B, the only part that is pre-zeroed), bucket boxes
 *     and chunk/super boxes from that array in one fused pass + one pass over the bucket starts (what
 *     gsx_sor_build leaves in the workspace), after which gsx_sor_mean_dists[_range] can run.  If spos4_dev already points at
 *     ws + gsx_sor_spos_offset(n) (all-gather straight into the workspace) no copy is made.
 * ws of A and B: gsx_sor_workspace_bytes(n_local) resp. (m); of C: gsx_sor_workspace_bytes(n_global). */
int gsx_sor_dist_local_run(const float* xyz_local_dev, int64_t n_local, int64_t idx_base, int64_t n_global,
                           int32_t world, const float* bmin_host, float cell, float* pos4_out_dev,
                           int64_t* cuts_dev, void* ws, int64_t ws_bytes, void* stream);
int gsx_sor_dist_merge(const float* pos4_dev, int64_t m, int64_t n_global, int64_t bucket_lo, int64_t bucket_hi,
                       const float* bmin_host, float cell, float* pos4_sorted_dev,
                       uint8_t* flags_sorted_dev /* uint8[m] or NULL */, void* ws, int64_t ws_bytes, void* stream);
int64_t gsx_sor_spos_offset(int64_t n);
int gsx_sor_build_from_sorted(const float* spos4_dev, const uint8_t* flags_dev /* uint8[n] or NULL */, int64_t n,
                              const float* bmin_host, float cell, void* ws, int64_t ws_bytes, void* stream);

/* gpu_ops.py:98-176 + :255-256: K = min(k,50) nearest candidates over the 27 probed buckets, mean of
 * their distances, written in the caller's point order (the "unsort" is fused).  Must follow
 * gsx_sor_build on the same workspace.  hash_mode = GSX_HASH_*.  stats_dev (may be NULL) receives
 * 4 uint64 counters {reference-model visits V, candidates actually scanned, box tests, queries}. */
int gsx_sor_mean_dists(int64_t n, int32_t k, int32_t hash_mode, const float* bmin_host, float cell, void* ws,
                       int64_t ws_bytes, float* final_means_dev, unsigned long long* stats_dev, void* stream);

/* Multi-GPU variant: only the hash-sorted positions [q_begin, q_end) are queried; the rows of
 * final_means_dev belonging to other queries are left untouched (caller zero-fills and all-reduces). */
int gsx_sor_mean_dists_range(int64_t n, int64_t q_begin, int64_t q_end, int32_t k, int32_t hash_mode,
                             const float* bmin_host, float cell, void* ws, int64_t ws_bytes, float* final_means_dev,
                             unsigned long long* stats_dev, void* stream);

/* Multi-GPU variant with COST-balanced sharding: the hash-sorted positions are cut into batches of 16; this call
 * queries the batches b with b % stride == phase (stride = number of ranks, phase = rank), so every rank samples the
 * whole hash range -- the expensive (clustered) buckets are spread over all ranks instead of falling to the owner of
 * their hash range.  Rows of final_means_dev belonging to other batches are left untouched. */
int gsx_sor_mean_dists_strided(int64_t n, int32_t stride, int32_t phase, int32_t k, int32_t hash_mode,
                               const float* bmin_host, float cell, void* ws, int64_t ws_bytes, float* final_means_dev,
                               unsigned long long* stats_dev, void* stream);

/* The query kernel's own counters of the last gsx_sor_mean_dists* call on this workspace that passed a non-NULL
 * stats_dev (that call zeroes them, also for an empty query range), copied to the HOST array out8_host after a
 * synchronise of `stream`: {serial inserts, first merges (sort only), full merges, probe-loop bucket visits, super-box
 * visits, chunk-group box-test rounds, chunk visits, scan steps of 32 candidates (chunk visits + small-bucket steps +
 * own-chunk seeds)}.  They count what a query spends on warp shuffles, votes and reductions (DESIGN 4.2). */
int gsx_sor_query_counters(int64_t n, void* ws, int64_t ws_bytes, unsigned long long* out8_host, void* stream);

/* gpu_ops.py:227 (np.argsort of the bucket hashes): stable LSD radix sort, in place, of (uint64 key, int32
 * value) pairs on the key bits [begin_bit, end_bit): 8-bit digits, one "onesweep" kernel per digit (decoupled
 * look-back over per-tile digit counts) after a single histogram pass.  vals_dev == NULL sorts bare 64-bit words
 * (n < 2^30): the form the hash-grid build uses, with word = bucket | in-cell Hilbert code | original index and only the
 * bits above the index sorted -- 8 instead of 12 bytes moved per point and pass. */
int64_t gsx_sort_pairs_workspace_bytes(int64_t n);
int gsx_sort_pairs(uint64_t* keys_dev, int32_t* vals_dev, int64_t n, int32_t begin_bit, int32_t end_bit, void* ws,
                   int64_t ws_bytes, void* stream);

/* gpu_ops.py:259-260 / data_processor.py:176-177: np.mean and np.std of a float32 vector with
 * float32 accumulators and NumPy's pairwise summation order, bit-for-bit.  out_dev[0]=mean, [1]=std. */
int64_t gsx_mean_std_workspace_bytes(int64_t n);
int gsx_mean_std_f32(const float* a_dev, int64_t n, float* out_dev, void* ws, int64_t ws_bytes, void* stream);

/* The same statistics for a vector sharded over G processes (rank r holds a[bases[r] .. bases[r+1]) ): NumPy's
 * pairwise tree depends only on n, so every leaf (<= 128 consecutive elements) is summed by the rank that holds
 * its first element -- spill-over elements come from halo_dev = float32[G*128], the first 128 elements of every
 * slab (all-gathered by the caller) -- into slot_dev[gsx_pairwise_slots(n)] (0 elsewhere); the caller all-reduces
 * (sum, exact: one writer per slot) and gsx_pairwise_finish combines the inner nodes: sq=0 writes meanstd_dev[0] =
 * mean, sq=1 (after the mean is known) writes meanstd_dev[1] = std.  Bit-identical to gsx_mean_std_f32 on the
 * concatenated vector.  bases_dev: int64[G+1] on the device. */
int64_t gsx_pairwise_slots(int64_t n);
int gsx_pairwise_leaves_dist(const float* a_local_dev, int64_t base, int64_t n_local, int64_t n_global, int32_t sq,
                             const float* meanstd_dev, const float* halo_dev, const int64_t* bases_dev, int32_t world,
                             float* slot_dev, void* stream);
int gsx_pairwise_finish(float* slot_dev, int64_t n_global, int32_t sq, float* meanstd_dev, void* stream);

/* gpu_ops.py:261-263 / data_processor.py:178-180: mask[i] = a[i] < mean + f32(threshold_factor)*std. */
int gsx_threshold_mask(const float* a_dev, int64_t n, const float* meanstd_dev, float threshold_factor,
                       uint8_t* mask_dev, void* stream);

/* Whole filter on device buffers (one 24-byte D2H sync inside for the cell size).
 * means_dev may be NULL.  Equivalent of filter_sor_gpu(data, k, threshold_factor). */
int gsx_sor_filter_device(const float* xyz_dev, int64_t n, int32_t k, float threshold_factor, int32_t hash_mode,
                          uint8_t* mask_dev, float* means_dev, void* ws, int64_t ws_bytes, void* stream);

/* Whole filter on HOST buffers: the binding target for gpu_ops.filter_sor_gpu (gpu_ops.py:193).
 * xyz_host float32[n,3]; mask_host uint8[n]; means_host float32[n] or NULL. */
int gsx_sor_filter_host(const float* xyz_host, int64_t n, int32_t k, float threshold_factor, int32_t hash_mode,
                        uint8_t* mask_host, float* means_host);

/* ---- SOR, cKDTree semantics: data_processor.py:155-180 (the reference's CPU path) ------------ */
/* data_processor.py:160-173: exact (k+1)-NN in float64 over the float32 coordinates (the nearest is the
 * point itself or a coincident twin and is dropped), mean of neighbours 1..k in float64 (NumPy pairwise
 * row reduction), stored as float32 in the caller's point order.  1 <= k <= 63. */
int64_t gsx_knn_exact_workspace_bytes(int64_t n);
int gsx_knn_exact_mean_dists(const float* xyz_dev, int64_t n, int32_t k, float* means_dev, void* ws, int64_t ws_bytes,
                             void* stream);
/* the same plus data_processor.py:176-180 (threshold and mask -- the mask the reference computes and then
 * discards, SURVEY F5) on HOST buffers. */
int gsx_sor_ckdtree_filter_host(const float* xyz_host, int64_t n, int32_t k, float threshold_factor, uint8_t* mask_host,
                                float* means_host);

/* ---- bbox / alpha masks: data_processor.py:215-231, :184-213 ------------------------ */
/* keep <=> lo <= v <= hi on all axes, float32 compares (bounds already rounded to float32 by caller). */
int gsx_bbox_mask(const float* xyz_dev, int64_t n, const float* lohi_host /*[6]*/, uint8_t* mask_dev, void* stream);
/* keep <=> (double)opacity >= logit_thresh (float64 compare, data_processor.py:208). */
int gsx_alpha_mask(const float* opacity_dev, int64_t n, double logit_thresh, uint8_t* mask_dev, void* stream);
/* host helper: data_processor.py:203-205 -> logit threshold for min_opacity_u8 in (0,255), libm log
 * (NumPy's SIMD log may differ by one float64 ulp; the Python plugin passes NumPy's own value). */
double gsx_alpha_logit_threshold(double min_opacity_u8);

/* ---- compaction of the filters' working set: the `vertices[mask]` steps of data_processor.py:114,149,209,
 * 217-224 for the columns the filters read (xyz, opacity) plus the surviving ORIGINAL row indices; stable like
 * NumPy boolean indexing.  opacity_dev/opacity_out_dev may both be NULL; idx_dev NULL = identity.
 * *count_host = number of survivors (one 4-byte D2H sync).  Any non-zero mask byte keeps its row.
 * n >= 2^31 is refused with GSX_ERR_UNSUPPORTED (the surviving row indices are int32). */
int64_t gsx_compact_workspace_bytes(int64_t n);
int gsx_compact_points(const uint8_t* mask_dev, int64_t n, const float* xyz_dev, const float* opacity_dev,
                       const int32_t* idx_dev, float* xyz_out_dev, float* opacity_out_dev, int32_t* idx_out_dev,
                       int64_t* count_host, void* ws, int64_t ws_bytes, void* stream);

/* ---- density filter: data_processor.py:38-52 (voxel histogram) and :111-112 (member mask) ---- */
int64_t gsx_density_workspace_bytes(int64_t n, int64_t cap);
/* q = floor(xyz / f32(voxel)) -> int64 triple (data_processor.py:39); counts per voxel (:43); every voxel
 * with count >= max(min_points,1) (:48-51) is returned to the HOST arrays dense_vox_host (int64[cap,3]) and
 * dense_cnt_host (int32[cap]), in no particular order; *n_dense_host = how many (> cap => GSX_ERR_WORKSPACE);
 * *n_voxels_host (may be NULL) = number of distinct voxels (len(unique_voxels), :45) inside the finite bounding
 * box.  Rows with a NaN coordinate fall outside that box and are not counted; when max(min_points,1) or more such
 * rows exist one of their voxels could be dense, and the call returns GSX_ERR_UNSUPPORTED. */
int gsx_density_voxel_count(const float* xyz_dev, int64_t n, float voxel, int64_t min_points, int64_t* dense_vox_host,
                            int32_t* dense_cnt_host, int64_t cap, int64_t* n_dense_host, int64_t* n_voxels_host,
                            void* ws, int64_t ws_bytes, void* stream);
/* data_processor.py:111-112: mask[i] = voxel(point i) is one of the n_keep voxels of keep_vox_host
 * (HOST int64[n_keep,3], the output of the host-side cluster selection :59-106). */
int gsx_density_member_mask(const float* xyz_dev, int64_t n, float voxel, const int64_t* keep_vox_host, int64_t n_keep,
                            uint8_t* mask_dev, void* ws, int64_t ws_bytes, void* stream);

/* Staged form for sharded clouds (one process per GPU): every rank counts its slab into an int32 grid over
 * the GLOBAL voxel box (q0[3], dim[3] voxels; from the all-reduced min/max via gsx_density_voxel_range), the
 * caller all-reduces the grid (sum) and extracts the dense voxels from it.  Same results as
 * gsx_density_voxel_count on the union cloud.  *oob_dev accumulates the points outside the box; over the global
 * box these are the rows with a NaN coordinate, and a caller refuses when there are >= max(min_points,1) of them
 * in the union cloud (gsx/dist.py: N minus the sum of the all-reduced grid). */
void gsx_density_voxel_range(const float* minmax_host /*[6]*/, float voxel, int64_t* q0_out, int64_t* dim_out);
int gsx_density_grid_count(const float* xyz_dev, int64_t n, float voxel, const int64_t* q0, const int64_t* dim,
                           int32_t* grid_dev, unsigned long long* oob_dev, void* stream);
int gsx_density_grid_dense(const int32_t* grid_dev, const int64_t* q0, const int64_t* dim, int64_t min_points,
                           int64_t* dense_vox_host, int32_t* dense_cnt_host, int64_t cap, int64_t* n_dense_host,
                           int64_t* n_voxels_host, void* ws, int64_t ws_bytes, void* stream);

/* ---- SOG writer helpers, the steps either side of K-Means (SURVEY 8(f) item 1) ------------------- */
/* formats/sog.py:264  np.lexsort((z, y, x)): order_dev[j] = index of the j-th splat in (x, then y, then z) order,
 * stable; -0.0 == +0.0 as in NumPy; every NaN (either sign, any payload) sorts after +inf and NaNs compare equal,
 * as in NumPy. */
int64_t gsx_lexsort_workspace_bytes(int64_t n);
int gsx_lexsort_zyx(const float* xyz_dev, int64_t n, int32_t* order_dev, void* ws, int64_t ws_bytes, void* stream);
/* formats/sog.py:408-419 quantize_to_codebook: index of the nearest entry of an ascending float32 codebook
 * (searchsorted-left, clip, prefer the left neighbour if strictly closer), as uint8.  1 <= m <= 4096; ws >= 4*m B. */
int gsx_quantize_to_codebook(const float* vals_dev, int64_t n, const float* codebook_host, int32_t m,
                             uint8_t* labels_dev, void* ws, int64_t ws_bytes, void* stream);

/* ---- SOG writer on the device: SogFormat.write, formats/sog.py:258-602 (gsx/sog.py) ---------------- */
/* Record rows are float32 [n, F]; every kernel reads row order_dev[j] for the j-th splat of the file (the lexsort
 * order).  Textures are uchar4 [pixels] (pixels >= n, 4-byte aligned); the padding pixels are written too.  Float
 * steps follow NumPy-2 float32 order; float -> u8/u16 conversions map NaN to 0.  n < 2^31.
 * The position logarithm and the opacity exponential are NumPy's SIMD float32 log and exp, restated exactly: every
 * byte is bit-exact.  The sign of a zero min or max of gsx_sog_means_minmax is not NumPy's (which depends on where
 * the zeros sit); the value is. */
/* sog.py:279-287: minmax_dev[6] = min x, y, z, max x, y, z of sign(v) * log(|v| + 1), NaN-propagating as
 * np.min / np.max.  cols3_host = columns of x, y, z; ws_dev >= 24576 B; n >= 1. */
int gsx_sog_means_minmax(const float* rows_dev, int64_t n, int32_t F, const int32_t* cols3_host, float* ws_dev,
                         int64_t ws_bytes, float* minmax_dev, void* stream);
/* sog.py:289-309: means_l / means_u, the low and high bytes of clip((l - min) / (max - min) * 65535) as u16 (0/0 of a
 * degenerate axis -> 0), alpha 255; padding 255. */
int gsx_sog_means(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev, const int32_t* cols3_host,
                  const float* minmax_dev, int64_t pixels, uint8_t* means_l_dev, uint8_t* means_u_dev, void* stream);
/* sog.py:315-386: quats (cols4_host = rot_0..3): the three non-largest components of the normalised, sign-fixed,
 * sqrt(2)-scaled quaternion through quantize_vec, alpha = 252 + argmax |q|; padding 255. */
int gsx_sog_quats(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev, const int32_t* cols4_host,
                  int64_t pixels, uint8_t* quats_dev, void* stream);
/* sog.py:392-400, 435-441: out_dev[t] = v[s] of v = np.concatenate([col_0, .., col_ncols-1]) in file order, with
 * s = sel_dev[t] (int64) or t when sel_dev is NULL -- the fit data of a 1-D codebook and its K-Means init rows. */
int gsx_sog_gather_values(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev,
                          const int32_t* cols_host, int32_t ncols, const int64_t* sel_dev, int64_t m, float* out_dev,
                          void* stream);
/* sog.py:421-459: scales (scale_0..2 against scale_cb, alpha 255) and sh0 (f_dc_0..2 against color_cb, alpha
 * clip(sigmoid(opacity) * 255)) in one pass; cols7_host = scale_0..2, f_dc_0..2, opacity; codebooks ascending,
 * 1..256 entries, on the device; padding 0. */
int gsx_sog_scales_sh0(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev,
                       const int32_t* cols7_host, const float* scale_cb_dev, int32_t m_scale,
                       const float* color_cb_dev, int32_t m_color, int64_t pixels, uint8_t* scales_dev,
                       uint8_t* sh0_dev, void* stream);
/* sog.py:483-503: out_dev[j, k] = column cols_host[k] of the j-th splat (float32 [n, ncols], 1 <= ncols <= 45) and
 * *nonzero_dev bit k = some value of that column != 0 (the band detection; -0.0 counts as zero). */
int gsx_sog_sh_gather(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev, const int32_t* cols_host,
                      int32_t ncols, float* out_dev, unsigned long long* nonzero_dev, void* stream);
/* sog.py:546-600: shN_labels.  Row j is in chunk c = j / chunk_size (nchunks <= 64); its label is labels_dev[j]
 * (chunk-local, as gsx_kmeans_lloyd_device returns it) or j - c * chunk_size where passthrough_host[c] != 0;
 * pixel = (label + offsets_host[c]) as u16 -> (lo, hi, 0, 255); padding 0. */
int gsx_sog_labels(const int32_t* labels_dev, int64_t n, int64_t chunk_size, int32_t nchunks,
                   const int32_t* offsets_host, const int32_t* passthrough_host, int64_t pixels, uint8_t* out_dev,
                   void* stream);
/* sog.py:566-588: shN_centroids.  The palette float32 [P, coeffs] (coeffs in {9, 24, 45}) against the ascending
 * codebook cb_dev (1..256 entries), laid out as (P, coeffs / 3, 3) RGB pixels, alpha 255; padding 255. */
int gsx_sog_centroids(const float* palette_dev, int64_t P, int32_t coeffs, const float* cb_dev, int32_t m,
                      int64_t pixels, uint8_t* out_dev, void* stream);

/* ---- lossless WebP (VP8L, RFC 9649) on the device: the SOG bundle's members (gsx/webp.py) ------------------------
 * The input is an RGBA uint8 image in HBM, [height * width, 4], 1 <= width, height <= 16384 (else GSX_ERR_ARG).
 * gsx_webp_analyze builds five entropy-coded images in the workspace: 0 = the pixels with RGB cleared where alpha is
 * 0, 1 = predictor residuals (16x16 tiles, per tile the mode 0..13 with the least sum of |residual as int8|, lowest
 * on a tie), 2 = subtract-green then the same, 3 / 4 = the predictor sub-images of 1 / 2 (alpha 255, mode in green);
 * their run copies of the left pixel (greedy, 3..4096 pixels) and their histograms: hist_dev uint32
 * [5 * 1088 + 1] = per image green + 24 length codes (280), red, blue, alpha (256 each), distance (40), then 1 when
 * some alpha is not 255.  modes_dev (nullable): uint8 [2 * tiles], the tile modes of images 1 and 2.
 * gsx_webp_emit writes the tokens of one image as LSB-first bits at bit_offset into words_dev (zeroed by the
 * caller; a token past nwords is dropped) with table_dev uint32 [1088] = bit-reversed code | length << 16 per
 * symbol, and stores the image's bit count in *total_bits_dev.  The workspace must hold what analyze left there.
 * gsx_webp_patch ORs npatches (word index, bits) pairs of uint32 into words_dev (the host-written headers). */
int64_t gsx_webp_workspace_bytes(int64_t width, int64_t height);
int gsx_webp_analyze(const uint8_t* rgba_dev, int64_t width, int64_t height, void* ws_dev, int64_t ws_bytes,
                     uint32_t* hist_dev, uint8_t* modes_dev, void* stream);
int gsx_webp_emit(int64_t width, int64_t height, int32_t image, const uint32_t* table_dev, uint64_t bit_offset,
                  void* ws_dev, int64_t ws_bytes, uint32_t* words_dev, int64_t nwords,
                  unsigned long long* total_bits_dev, void* stream);
int gsx_webp_patch(uint32_t* words_dev, int64_t nwords, const uint32_t* patches_dev, int64_t npatches, void* stream);

/* ---- lossless WebP (VP8L, RFC 9649) decoding on the device: the SOG reader's members (gsx/webp_decode.py) ---------
 * data_dev is the n-byte VP8L payload (from its 0x2f signature); bit offsets count LSB first from its byte 0.
 * gsx_vp8l_header_words(width, height, groups): uint32 words of the header workspace for an image of that size whose
 * main image has `groups` prefix-code groups (0 for sides outside 1..16384 or groups outside 1..65536).
 * gsx_vp8l_header (one thread) parses the header, transforms, sub-images, cache bits, entropy image and every group's
 * prefix codes into ws_dev; lens_dev is 2328 bytes of scratch.  info_dev int64 [32]: 0 status (0 ok, 1 truncated,
 * 2 a bad prefix code or sub-image copy, 3 a bad header field, 4 the workspace is too small: [29] words needed), 1 bit
 * where it stopped, 2 width, 3 height, 4 alpha hint, 5 coded width, 6 cache bits, 7 meta prefix bits, 8 groups,
 * 9 entropy image word offset (-1: none), 10 codes word offset, 11 first bit of the main image, 12 transforms, then
 * per transform in reading order 4 values: type (0 predictor, 1 cross-colour, 2 subtract-green, 3 colour indexing),
 * the width it applies at, its bits, its sub-image's word offset.
 * gsx_vp8l_run runs njobs jobs, one thread each: jobs_dev int64 [njobs, 5] = start bit, target bit, guessed first
 * pixel, token offset, capacity in tokens.  A job decodes tokens (16 bytes each in tokens_dev: value, kind << 28 |
 * pixels, first pixel relative to the job, group) until it stands at or past target, or its pixels reach the image's
 * end.  results_dev int64 [njobs, 6] = start, stop bit, tokens, pixels, status (0 target, 1 image end, 2 the input
 * ended, 4 capacity), bit where it stopped.
 * gsx_vp8l_check sets flags_dev[k] (zeroed by the caller) when a token of piece k (pieces_dev int64 [npieces, 3] =
 * device address of its tokens, tokens, true first pixel) used a group other than the one at its true position.
 * gsx_vp8l_resolve writes the chain's pieces (same layout, in pixel order) as ARGB into out_dev [npix], with src_dev
 * int32 [npix] as scratch; *err_dev (zeroed) gains 1 for a copy from before the first pixel, 2 for one past the last.
 * gsx_vp8l_inverse applies one inverse transform to the xs x height image: colour indexing reads in_dev (the packed
 * image) and writes out_dev; the others work in place on out_dev.  scratch_dev: int32 [height / 32 + 2] (predictor).
 * gsx_vp8l_rgba writes n ARGB pixels as RGBA bytes, alpha 255 when alpha is 0. */
int64_t gsx_vp8l_header_words(int64_t width, int64_t height, int64_t groups);
int gsx_vp8l_header(const uint8_t* data_dev, int64_t n, uint32_t* ws_dev, int64_t ws_words, uint8_t* lens_dev,
                    int64_t* info_dev, void* stream);
int gsx_vp8l_run(const uint8_t* data_dev, int64_t n, const uint32_t* codes_dev, const uint32_t* entropy_dev,
                 int64_t xsize, int64_t height, int32_t meta_bits, const int64_t* jobs_dev, int64_t njobs,
                 void* tokens_dev, int64_t* results_dev, void* stream);
int gsx_vp8l_check(const uint32_t* codes_dev, const uint32_t* entropy_dev, int64_t xsize, int64_t height,
                   int32_t meta_bits, const int64_t* pieces_dev, int64_t npieces, int32_t* flags_dev, void* stream);
int gsx_vp8l_resolve(const int64_t* pieces_dev, int64_t npieces, int64_t xsize, int64_t npix, int32_t cache_bits,
                     uint32_t* out_dev, int32_t* src_dev, int32_t* err_dev, void* stream);
int gsx_vp8l_inverse(int32_t type, const uint32_t* in_dev, uint32_t* out_dev, const uint32_t* sub_dev, int64_t xs,
                     int64_t height, int32_t bits, int32_t* scratch_dev, void* stream);
int gsx_vp8l_rgba(const uint32_t* argb_dev, uint8_t* rgba_dev, int64_t n, int32_t alpha, void* stream);

/* ---- raw DEFLATE (RFC 1951) decoding on the device: the bodies of gzip members (gsx/deflate.py gunzip) -----------
 * data_dev is n bytes of HBM starting at a DEFLATE stream (64-bit n); bit offsets count LSB first from its byte 0.
 * The workspace holds 16-bit symbols: gsx_inflate_workspace_bytes(symbols) bytes hold `symbols` of them.
 * gsx_inflate_run runs njobs jobs, one thread each.  jobs_dev int64 [njobs, 6] = lo, hi, target, symbol offset into
 * the workspace, capacity in symbols, flags (1 = FIND: start at the first plausible block start in bits [lo, hi), a
 * dynamic block that decodes to its end-of-block or a stored block with zero padding and LEN = ~NLEN; else start at
 * lo.  2 = FIRST: the start is the stream's first bit, so a distance past the first byte is an error).  A job decodes
 * blocks until one ends at or past `target` or the final block ends.  Symbols: a byte (0..255), or 0x8000 | w, byte w
 * of the 32 KiB before the start.  results_dev int64 [njobs, 6] = start (-1: none found), stop (bit after the last
 * whole block), symbols written, position of the last 0x8000 symbol (-1: none), status, bit where it stopped.
 * Status: 0 target reached, 1 final block ended, 2 the input ended (zlib: EOFError), 3 invalid stream (zlib.error),
 * 4 capacity exceeded, 5 no plausible start, 6 a job outside the input or the workspace.
 * gsx_inflate_resolve writes the pieces pieces_dev int64 [npieces, 5] = symbols (device pointer), count, output
 * offset, first and one-past-last position of the markers resolved in chain order (a piece's last 32 KiB: the next
 * piece's window) into out_dev, pieces in chain order and each window byte before its piece.  A marker before out_dev's
 * first byte is zlib's "invalid distance too far back": *status_dev (set to 2^64-1 by the caller) becomes the least
 * such output offset. */
int64_t gsx_inflate_workspace_bytes(int64_t symbols);
int gsx_inflate_run(const uint8_t* data_dev, int64_t n, const int64_t* jobs_dev, int64_t njobs, void* ws_dev,
                    int64_t ws_bytes, int64_t* results_dev, void* stream);
int gsx_inflate_resolve(const int64_t* pieces_dev, int64_t npieces, uint8_t* out_dev,
                        unsigned long long* status_dev, void* stream);

/* ---- raw DEFLATE (RFC 1951) and CRC-32 on the device: the body and trailer of .gz files (gsx/deflate.py) ---------
 * data_dev is n bytes of HBM (64-bit n).  Every pointer is a device pointer; every entry runs on `stream`.
 * gsx_deflate_workspace_bytes(nblocks): the workspace of gsx_crc32 (nblocks 0), gsx_deflate_plan and
 * gsx_deflate_emit: 4 KiB + about 1.6 KiB per block, independent of n.
 * gsx_crc32 writes the 8-byte gzip trailer at trailer_dev: zlib's crc32 of the n bytes, then n mod 2^32, both
 * little-endian (the CRC of each 4 KiB chunk is shifted by x^(8 * bytes after it) mod P and XORed).
 * gsx_deflate_stored writes 5 * max(1, ceil(n / 65535)) + n bytes at out_dev: stored blocks of 65535 bytes, the
 * last one shorter and final (an empty input: one empty final block).
 * gsx_deflate_plan plans the dynamic blocks starts_dev int64 [nblocks] (block b is [starts[b], starts[b + 1]) or up
 * to n; starts[0] = 0, ascending, each block at most 1 MiB; one empty block when n = 0).  Per block: the
 * histograms of literals only and of literals plus distance-1 copies (a run of r >= 4 equal bytes -> one literal,
 * then copies of 258, then one copy of the remainder when it is >= 3, else that many literals), Huffman code lengths
 * (15 bits, 7 for the code-length code; the rule of gsx/webp.py code_lengths), the run-length-coded header, and the
 * candidate with fewer bits (literals on a tie).  Writes the body's bit count to *total_bits_dev; block b starts at
 * bit bit_offset + the bits of the blocks before it.
 * gsx_deflate_emit ORs the planned blocks' bits into words_dev (uint32 LSB-first, zeroed by the caller and sized
 * from the total; bits past nwords are dropped) and adds 1 to *mismatches_dev for every block whose emitted bits
 * differ from its plan.  The workspace must hold what gsx_deflate_plan left there. */
int64_t gsx_deflate_workspace_bytes(int64_t nblocks);
int gsx_crc32(const uint8_t* data_dev, int64_t n, void* ws_dev, int64_t ws_bytes, uint8_t* trailer_dev, void* stream);
int gsx_deflate_stored(const uint8_t* data_dev, int64_t n, uint8_t* out_dev, void* stream);
int gsx_deflate_plan(const uint8_t* data_dev, int64_t n, const int64_t* starts_dev, int64_t nblocks, void* ws_dev,
                     int64_t ws_bytes, uint64_t bit_offset, unsigned long long* total_bits_dev, void* stream);
int gsx_deflate_emit(const uint8_t* data_dev, int64_t n, const int64_t* starts_dev, int64_t nblocks, void* ws_dev,
                     int64_t ws_bytes, uint32_t* words_dev, int64_t nwords, unsigned long long* mismatches_dev,
                     void* stream);

/* ---- Parquet writer on the device: ParquetFormat.write, formats/parquet.py:59-112 (gsx/parquet.py) ---------------
 * n rows (n <= 2^31) of row_bytes bytes each (1 .. 1024); ncols columns (1 .. 1024).  Row group g is rows
 * [g * 2^20, (g + 1) * 2^20), data page p rows [p * 2^18, (p + 1) * 2^18), tile t rows [t * 2048, (t + 1) * 2048).
 * A value is null when its pattern is a float32 NaN; uint8 columns are widened and never null.  Every pointer but
 * cols_host is a device pointer; every entry runs on `stream`.
 * gsx_parquet_split (parquet.py:94-108, the frame's columns): cols_host int32 [ncols][2] = (byte offset in the row,
 * kind: 0 float32, 1 uint8).  Writes out_dev uint32 [ncols][n] (column-major patterns), tile_nulls_dev uint32
 * [ncols][tiles] and keys_dev uint32 [2][ncols][groups]: each chunk's least and greatest order-preserving key of its
 * non-null values (float32: sign bit flipped for positives, all bits for negatives; uint8: the value), 0xFFFFFFFF and
 * 0 for a chunk without one.
 * gsx_parquet_dict_insert (pyarrow's dictionary encoding): the non-null patterns of row groups [g0, g0 + ng) into
 * table_dev (uint64 [ng][ncols][2^slots_log2], zeroed by the caller, slots_log2 20 .. 24); distinct_dev uint32
 * [ncols][groups] (zeroed) counts the distinct patterns of each chunk, exactly up to 262 144, and ends above it
 * otherwise.  2^20 slots is the least safe table: a chunk stops inserting only once a thread sees its count above
 * 262 144, so every thread already past that check (up to one resident grid, 132 x 2048 on an H100) may still insert;
 * 262 144 + 270 336 > 2^19, and a full table could wrap the count back below the limit.  gsx_parquet_dictionary and
 * gsx_parquet_dict_index take the same slots_log2 (20 .. 24).
 * gsx_parquet_dictionary: for jobs_dev int64 [njobs][3] = (table index c + ncols * (g - g0), first key, first
 * dictionary value), njobs <= 65535, whose first keys leave room for each chunk's distinct count (nkeys in all):
 * the chunk's patterns ascending to dict_vals_dev, and each one's rank into the table.  Workspace from
 * gsx_parquet_dictionary_workspace_bytes(nkeys).
 * gsx_parquet_dict_index: every non-null value of the chunks of row groups [g0, g0 + ng) with dict_chunk_dev[c][g - g0]
 * != 0 replaced in cols_dev by its rank; page_idx_dev uint32 [2][ncols][pages] (0xFF.. and 0 filled by the caller)
 * gets each page's least and greatest rank.
 * gsx_parquet_pages: the page bodies into body_dev (uint32 words, zeroed by the caller).  info_dev int64
 * [ncols][pages][4] = (body byte offset, 16-byte aligned; nulls; bit width, 0 for PLAIN; all ranks equal) of each data
 * page; dict_jobs_dev int64 [ndict][3] = (first dictionary value, body offset, entries <= max_dict) of each
 * dictionary page.  A data page is the 4-byte length and RLE / bit-packed hybrid of its definition levels (one RLE
 * run, or one bit-packed run over its rows when it has nulls), then PLAIN values, or the bit width byte and the ranks
 * as one bit-packed run (one RLE run when they are all equal; nothing when the page has no value).
 * gsx_parquet_snappy: pieces_dev int64 [npieces][3] = (page, body offset (16-byte aligned), bytes 1 .. 65536).  Piece
 * i's Snappy elements go to scratch_dev + i * gsx_parquet_piece_bytes(), their length to sizes_dev[i], and it is added
 * to page_csize_dev[page] (zeroed by the caller).  Copies of distance 1 or 4 and length >= 8 inside the piece, taken
 * greedily from the left (the longer one; the two never tie at a chosen start); literals elsewhere.
 * gsx_parquet_assemble: the file: the pieces of each page back to back from page_dst_dev[page] (page_first_dev: its
 * first piece), and hjobs_dev int64 [nh][3] = (offset in heads_dev, file offset, bytes) of the headers and footer. */
int gsx_parquet_split(const uint8_t* rows_dev, int64_t n, int32_t row_bytes, const int32_t* cols_host, int32_t ncols,
                      uint32_t* out_dev, uint32_t* tile_nulls_dev, uint32_t* keys_dev, void* stream);
int gsx_parquet_dict_insert(const uint32_t* cols_dev, int64_t n, int32_t ncols, int32_t g0, int32_t ng,
                            unsigned long long* table_dev, int32_t slots_log2, uint32_t* distinct_dev, void* stream);
int64_t gsx_parquet_dictionary_workspace_bytes(int64_t nkeys);
int gsx_parquet_dictionary(unsigned long long* table_dev, int32_t slots_log2, const int64_t* jobs_dev, int32_t njobs,
                           int64_t nkeys, void* ws_dev, int64_t ws_bytes, uint32_t* dict_vals_dev, void* stream);
int gsx_parquet_dict_index(uint32_t* cols_dev, int64_t n, int32_t ncols, int32_t g0, int32_t ng,
                           const unsigned long long* table_dev, int32_t slots_log2, const int32_t* dict_chunk_dev,
                           uint32_t* page_idx_dev, void* stream);
int gsx_parquet_pages(const uint32_t* cols_dev, int64_t n, int32_t ncols, const uint32_t* tile_nulls_dev,
                      const int64_t* info_dev, const uint32_t* dict_vals_dev, const int64_t* dict_jobs_dev,
                      int32_t ndict, int64_t max_dict, uint32_t* body_dev, void* stream);
int64_t gsx_parquet_piece_bytes(void);
int gsx_parquet_snappy(const uint8_t* body_dev, const int64_t* pieces_dev, int64_t npieces, uint8_t* scratch_dev,
                       uint32_t* sizes_dev, uint32_t* page_csize_dev, void* stream);
int gsx_parquet_assemble(const uint8_t* scratch_dev, const int64_t* pieces_dev, int64_t npieces,
                         const uint32_t* sizes_dev, const int64_t* page_first_dev, const int64_t* page_dst_dev,
                         const uint8_t* heads_dev, const int64_t* hjobs_dev, int64_t nh, uint8_t* file_dev,
                         void* stream);

/* ---- K-Means: gpu_ops.py:57-96 (kernels) + :186-188 (Lloyd loop) ---------------------- */
/* Batched over `nprob` independent problems stored back to back (SOG shN chunks, sog.py:527-549):
 * problem p has rows [row_off[p], row_off[p+1]) of X[*,D] and K centroids at C[p*K*D].
 * One call = max_iter x (assign ; update) with the serial index-order float32 sums of SURVEY A.5.
 * labels are those of the last assign (one update behind C, SURVEY F9); counts int32[nprob*K]. */
int64_t gsx_kmeans_workspace_bytes(int64_t n_total, int32_t nprob, int32_t K, int32_t D);
/* assign_mode (per call; the labels are bit-identical in every mode; any other value is GSX_ERR_ARG):
 *   AUTO    tensor cores when the shape allows it (gsx_kmeans_tensor_core_supported), else STRICT
 *   STRICT  the contract's distance for every (point, centroid) on the FP32 pipes
 *   TENSOR  the score matrix X.C^T - ||c||^2/2 computed by wgmma.mma_async (TF32, float32 accumulators in registers,
 *           two-pass epilogue: row maximum, candidate mask), then the contract's distance only for the centroids
 *           within a proven rounding-error margin of the best score; error if the shape is unsupported
 *           (D in {9,24,45}, K <= 256)
 * tc_stats_dev (may be NULL): 3 uint64 counters accumulated by the TENSOR path {strict distance evaluations,
 * points with more than one candidate, points that needed the full strict scan}. */
#define GSX_KM_ASSIGN_AUTO 0
#define GSX_KM_ASSIGN_STRICT 1
#define GSX_KM_ASSIGN_TENSOR 3
int gsx_kmeans_lloyd_device(const float* X_dev, const int64_t* row_off_host, int32_t nprob, int32_t K, int32_t D,
                            int32_t max_iter, float* C_dev, int32_t* labels_dev, int32_t* counts_dev, void* ws,
                            int64_t ws_bytes, int32_t assign_mode, unsigned long long* tc_stats_dev, void* stream);
/* 1 if the TENSOR assign takes this shape, else 0 */
int32_t gsx_kmeans_tensor_core_supported(int32_t K, int32_t D);
/* Test hook of the tensor-core assign: raw scores s[r][c] = x_r.c - ||c||^2/2 of the first min(rows,128) rows
 * against the K centroids, scores_dev float32[128 * roundup32(K)].  ws >= 1024 bytes. */
int gsx_kmeans_tc_debug_scores(const float* X_dev, int64_t rows, const float* C_dev, int32_t K, int32_t D,
                               float* scores_dev, void* ws, int64_t ws_bytes, void* stream);
/* Single problem on HOST buffers: binding target for gpu_ops.kmeans on the GPU path (gpu_ops.py:178-191)
 * with the init centroids chosen by the caller (the reference's np.random.choice draw). */
int gsx_kmeans_host(const float* X_host, int64_t n, int32_t K, int32_t D, int32_t max_iter, float* C_host_inout,
                    int32_t* labels_host, int32_t assign_mode);

/* ---- device-resident splat records (SURVEY 8(f) items 2 and 4) ------------------------------------------------
 * rows_dev: the reference's interchange records (structures.py:23-59) as a row-major float32 matrix [n, F]
 * (F = 62 for SH degree 3), uploaded once.  Column arguments are field positions inside a row.
 *  extract : np.column_stack((x,y,z)) / v['opacity'] of data_processor.py:38,139,184 -> xyz [n,3], opacity [n] (or NULL)
 *  gather  : vertices[mask] of data_processor.py:114,149,209,224 for the surviving (ascending) row indices
 *  color   : RGBA8 of formats/splat.py:131-144, ksplat.py:464-468: clip((0.5 + scale*f_dc)*255).astype(u8) x3 (bit-exact
 *            float32 ops; scale = SH_C0 for .splat/.ksplat, 0.15 for spz.py:131) and clip(sigmoid(opacity)*255).astype(u8)
 *            (NumPy's SIMD float32 exp, restated exactly: bit-exact)
 *  scale   : np.exp(scale_0..2) of formats/splat.py:108, ksplat.py:447 -> float32 [n,3] */
int gsx_records_extract_xyz_opacity(const float* rows_dev, int64_t n, int32_t F, int32_t cx, int32_t cy, int32_t cz,
                                    int32_t cop, float* xyz_dev, float* opacity_dev, void* stream);
int gsx_records_gather_rows(const float* rows_dev, const int32_t* idx_dev, int64_t m, int32_t F, float* out_dev,
                            void* stream);
int gsx_records_color_rgba8(const float* rows_dev, int64_t n, int32_t F, int32_t c0, int32_t c1, int32_t c2, int32_t cop,
                            float scale, uint8_t* rgba_dev, void* stream);
int gsx_records_scale_exp(const float* rows_dev, int64_t n, int32_t F, int32_t s0, int32_t s1, int32_t s2, float* out_dev,
                          void* stream);

/* ---- Morton ordering as a shared primitive (SURVEY 8(f) item 3) ----------------------------------------------
 * formats/compressed_ply.py:252-297 (_sort_morton_order): order_dev[j] = index of the j-th splat in the recursive
 * 3 x 10-bit Morton order (codes relative to the bounding box of the group; every run of equal codes longer than
 * run_limit (the reference: 256) is re-normalised to its own box and sorted again, until it is short or has no
 * extent).  Equal codes inside a finished run come out in ascending original index (the reference's unstable
 * np.argsort leaves that order unspecified).  The levels run until no run is left; *levels_out = number of levels that
 * ran (the reference's recursion depth + 1).  A NaN position makes its run's box NaN on that axis, as cx.min() does.
 * Returns GSX_ERR_UNSUPPORTED when a run longer than run_limit does not split (zero, infinite or NaN extent on every
 * axis, not all zero): the reference recurses into it for ever. */
int64_t gsx_morton_workspace_bytes(int64_t n);
int gsx_morton_order(const float* xyz_dev, int64_t n, int32_t* order_dev, int32_t run_limit, int32_t* levels_out, void* ws,
                     int64_t ws_bytes, void* stream);
/* compressed_ply.py:206-246 (per-256-splat chunk bounds) / ksplat.py:426-441 (np.minimum/maximum.reduceat per
 * bucket): min and max of ncol (<= 8) columns cols_host[] of the row-major float32 matrix rows_dev [n,F] over
 * consecutive chunks of `chunk` rows taken in the order order_dev (NULL = identity); values are clipped to
 * [clip_lo, clip_hi] first (np.clip(scale, -20, 20) of compressed_ply.py:213-215; pass -inf/+inf for none).  A NaN
 * (kept by the clip, as np.clip does) makes its chunk's min and max NaN; of -0.0 and +0.0 the min is -0.0, the max +0.0.
 * lo_dev / hi_dev: float32 [ceil(n/chunk), ncol].  ws >= 64 bytes. */
int gsx_chunk_minmax(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev, int32_t chunk,
                     const int32_t* cols_host, int32_t ncol, float clip_lo, float clip_hi, float* lo_dev, float* hi_dev,
                     void* ws, int64_t ws_bytes, void* stream);
/* compressed_ply.py:174-246 (CompressedPlyFormat.write after the Morton sort): the packed chunk, vertex and SH blocks of
 * the PlayCanvas compressed PLY, one 256-splat chunk per CTA, rows taken in order_dev (gsx_morton_order).
 *   cols14_host: columns of x y z f_dc_0 f_dc_1 f_dc_2 opacity scale_0 scale_1 scale_2 rot_0 rot_1 rot_2 rot_3;
 *   rest_cols_host[n_rest] (n_rest <= 45): the columns of the present f_rest_i, i < 45, in ascending i.
 *   lo/hi_pos_dc_dev [C,6]: gsx_chunk_minmax of x y z f_dc_0..2 over the ordered rows (no clip);
 *   lo/hi_scale_dev [C,3]: the same of scale_0..2 with clip [-20, 20]  (C = ceil(n/256)).
 * Outputs: chunk_dev float32[C,18] (min_x..max_z, min/max_scale_x..z, min_r..max_b; colour = f32(f32(f_dc*SH_C0)+0.5)),
 * vertex_dev uint32[n,4] {packed_position, packed_rotation, packed_scale, packed_color}, sh_dev uint8[n,n_rest]
 * (may be NULL when n_rest == 0), *rest_nonzero_dev (device uint64, zeroed here) = bit k set iff packed SH column k holds
 * a value != 0 -- the input of the SH-degree rule of :141-169, which the caller applies (gsx_cply_narrow_sh).
 * NumPy-2 float32 arithmetic and NumPy's SIMD float32 exp, bit-exact.  vertex_dev and
 * sh_dev 16-byte aligned; n < 2^31; n = 0 launches nothing.  A NaN field packs as NumPy's x86 cast gives it,
 * 0x80000000 shifted into the word (DESIGN §4.5); a quaternion's first NaN component is its largest. */
int gsx_cply_pack(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev, const int32_t* cols14_host,
                  const int32_t* rest_cols_host, int32_t n_rest, const float* lo_pos_dc_dev, const float* hi_pos_dc_dev,
                  const float* lo_scale_dev, const float* hi_scale_dev, float* chunk_dev, uint32_t* vertex_dev,
                  uint8_t* sh_dev, uint64_t* rest_nonzero_dev, void* stream);
/* compressed_ply.py:163-169: out_dev[j, :keep] = sh_dev[j, :keep] for the uint8 [n, width] block of gsx_cply_pack, when
 * the detected SH degree keeps fewer columns than were packed.  0 <= keep <= width <= 45. */
int gsx_cply_narrow_sh(const uint8_t* sh_dev, int64_t n, int32_t width, int32_t keep, uint8_t* out_dev, void* stream);

/* The .ksplat / .spz / .splat writers (formats/ksplat.py:319-544, spz.py:49-173, splat.py:82-166) over device-resident
 * float32 records [n, F].  cols14_host: the columns of x y z f_dc_0 f_dc_1 f_dc_2 opacity scale_0 scale_1 scale_2
 * rot_0 rot_1 rot_2 rot_3.  NumPy-2 float32 arithmetic in the reference's order, NumPy's SIMD float32 exp restated
 * exactly, NumPy's x86-64 casts (NaN -> 0 in uint8 / uint16, INT32_MIN in int32, 0x80000000 in a SIMD uint32 cast;
 * float16 NaN = sign | 0x7c00 | mantissa >> 13).  n >= 2^31 is refused with GSX_ERR_UNSUPPORTED (int32 row indices,
 * uint32 counts in the ksplat header); n = 0 launches nothing.
 *
 * ksplat.py:340-368 / spz.py:53-77 (np.all(x == 0) / np.any(x != 0) per f_rest column): *mask_dev (zeroed here) gets
 * bit k iff column sh_cols_host[k] holds a value != 0 (NaN included, -0.0 excluded).  nsh <= 45.  The degree rules
 * run on the host from this mask. */
int gsx_codec_sh_mask(const float* rows_dev, int64_t n, int32_t F, const int32_t* sh_cols_host, int32_t nsh,
                      uint64_t* mask_dev, void* stream);
/* ksplat.py:396-403: bytes of one interleaved record at `level` (0: float32; 1: float16; >= 2: float16 with uint8 SH)
 * for sh_count = 0, 9 or 24 SH values. */
int32_t gsx_ksplat_record_bytes(int32_t level, int32_t sh_count);
/* ksplat.py:439-445: centres_dev[b, a] = (lo_dev[b, a] + hi_dev[b, a]) / 2.0 in float32, for the bucket bounds
 * [nbucket, 3] of gsx_chunk_minmax(x, y, z; chunk = bucket_size). */
int gsx_ksplat_centres(const float* lo_dev, const float* hi_dev, int64_t nbucket, float* centres_dev, void* stream);
/* ksplat.py:419-536: the interleaved records, n * gsx_ksplat_record_bytes(level, sh_count) bytes into out_dev, rows in
 * stored order.  sh_cols_host: the columns of f_rest_0 .. f_rest_{sh_count-1}.  Level 0 writes the float32 position,
 * exp(scale) and rotation bits; levels >= 1 write clip(rint((x - centre) * sf_inv) + 32767, 0, 65535) as uint16
 * (centre = centres_dev row j / bucket_size) and float16 exp(scale), rotation and SH; level 2 stores the SH as
 * uint8 clip((v + 2) / 4 * 255, 0, 255), and levels >= 3, as the reference does, the raw uint8 cast of v. */
int gsx_ksplat_pack(const float* rows_dev, int64_t n, int32_t F, const int32_t* cols14_host, const int32_t* sh_cols_host,
                    int32_t sh_count, int32_t level, int64_t bucket_size, float sf_inv, const float* centres_dev,
                    uint8_t* out_dev, void* stream);
/* spz.py:106-173 (_pack_v3): the planar SPZ body of n * (20 + 3 * sh_dim) bytes into body_dev: 24-bit positions
 * (rint(x * 4096) as int32, low three bytes), alpha, colour, scales, smallest-three rotations (spz.py:298-343), then the
 * SH bytes.  sh_dim = 0, 3, 8 or 15; sh_cols_host[3 * sh_dim] holds the columns of f_rest_i, f_rest_{i+15},
 * f_rest_{i+30} for i < sh_dim, interleaved in that order. */
int gsx_spz_pack(const float* rows_dev, int64_t n, int32_t F, const int32_t* cols14_host, const int32_t* sh_cols_host,
                 int32_t sh_dim, uint8_t* body_dev, void* stream);
/* splat.py:92-98: keys_dev[i] = an order-preserving uint32 key (bits 0..31 of the uint64 word) of
 * -(exp(scale_0 + scale_1 + scale_2) * (1 / (1 + exp(-opacity)))), -0.0 sorted as +0.0 and every NaN above +inf, and
 * vals_dev[i] = i.  cols4_host: scale_0 scale_1 scale_2 opacity.  gsx_sort_pairs on bits [0, 32) then gives NumPy's
 * stable argsort of -metric. */
int gsx_splat_sort_keys(const float* rows_dev, int64_t n, int32_t F, const int32_t* cols4_host, uint64_t* keys_dev,
                        int32_t* vals_dev, void* stream);
/* splat.py:100-164: the 32-byte .splat records of rows order_dev[0 .. n) into out_dev: float32 position,
 * float32 exp(scale), RGBA8, and uint8 clip(r / |r| * 128 + 128, 0, 255) of the rotation. */
int gsx_splat_pack(const float* rows_dev, int64_t n, int32_t F, const int32_t* order_dev, const int32_t* cols14_host,
                   uint8_t* out_dev, void* stream);
/* out_dev[j, k] = the float32 at byte offsets_host[k] of row j of src_dev (n rows of row_bytes bytes, any alignment):
 * the float32 fields of a structured array that also holds other fields (the converter's red/green/blue u1), as the
 * packed float32 rows the writers read.  1 <= nf <= 256. */
int gsx_records_from_bytes(const uint8_t* src_dev, int64_t n, int64_t row_bytes, const int32_t* offsets_host, int32_t nf,
                           float* out_dev, void* stream);

/* Readers: the file's bytes on the device -> rows in the exact byte layout of the structured array the reference
 * reader returns (row_bytes = that dtype's itemsize; red/green/blue u1 fields included).  tables_dev holds 256-entry
 * float32 tables, one per map of a single input byte, which the caller builds with the reference's own NumPy expression
 * (gsx.splat / gsx.ksplat / gsx.spz / gsx.compressed_ply build them): NumPy's float32 and float64 log come out as the
 * host computes them.  Input buffers may start at any byte.  n < 2^31.
 * gsx_splat_decode (splat.py:9-80): n 32-byte records -> n rows of 71 bytes (define_dtype(has_rgb=True, sh_degree=0));
 *   scales log(max(s, 1e-6)) with NumPy's float32 log, rotations (b - 128) / 128 renormalised by max(norm, 1e-6);
 *   nx/ny/nz and red/green/blue stay 0.  tables: DC, opacity logit. */
int gsx_splat_decode(const uint8_t* data_dev, int64_t n, const float* tables_dev, uint8_t* rows_dev, void* stream);
/* gsx_ksplat_decode_section (ksplat.py:109-264): one section's n records of level 0, 1 or 2 (any stored level >= 2)
 * into rows of row_bytes bytes (define_dtype(sh_degree = the file's largest section degree)); the section's sh_count
 * (0, 9 or 24) values fill f_rest_0 .., the other f_rest columns stay 0.  Levels >= 1: splat i lies in bucket
 * i / bucket_size below full_buckets * bucket_size, past it in partial bucket full_buckets + k for the first k with
 * partial_end_dev[k] (the prefix sums of the partially-filled bucket lengths) > i - full_buckets * bucket_size;
 * positions are (float32(u16) - scale_range) * scale_factor + centre in float32.  Every splat's bucket must have a
 * centre among the ncentres of centres_dev (checked from the last splat's).  tables: DC, opacity logit, level-2 SH. */
int gsx_ksplat_decode_section(const uint8_t* records_dev, int64_t n, int32_t level, int32_t sh_count, float scale_range,
                              float scale_factor, const uint8_t* centres_dev, int64_t ncentres, int64_t full_buckets,
                              int64_t bucket_size, const int64_t* partial_end_dev, int32_t npartial,
                              const float* tables_dev, int32_t row_bytes, uint8_t* rows_dev, void* stream);
/* gsx_spz_decode (spz.py:175-296): the gunzipped body after the 16-byte header of version 1, 2 or 3 -> rows of
 * row_bytes bytes (define_dtype(has_rgb=True, sh_degree = the header's degree)).  sh_dim = 0, 3, 8 or 15 (0 for
 * degrees above 3, whose f_rest columns stay 0); positions float16 (v1) or int24 / 2^frac_bits (frac_bits <= 127);
 * rotations first-three (v1, v2) or smallest-three in float64 (v3).  tables: opacity logit, DC, RGB, scale, SH. */
int gsx_spz_decode(const uint8_t* body_dev, int64_t n, int32_t version, int32_t sh_dim, int32_t frac_bits,
                   const float* tables_dev, int32_t row_bytes, uint8_t* rows_dev, void* stream);
/* gsx_cply_decode (compressed_ply.py:14-123, 342-378): a binary little-endian compressed PLY's elements chunk (nchunk
 * rows of chunk_row bytes; chunk_offs_host[18]: byte offsets of min_x .. max_b in gsx.compressed_ply.CHUNK_DTYPE
 * order, float32), vertex (n rows of vertex_row bytes; vertex_offs_host[4]: packed_position, packed_rotation,
 * packed_scale, packed_color, uint32) and sh (sh_row bytes; sh_offs_host[nsh]: its uchar properties in file order,
 * nsh <= 64) -> n rows of 4 * (17 + nsh) bytes.  Bounds and de-normalisation in float64 as NumPy promotes them, rounded
 * once on store; rows past nchunk * 256 stay 0.  tables: opacity logit, SH. */
int gsx_cply_decode(const uint8_t* chunk_dev, int64_t nchunk, int32_t chunk_row, const int32_t* chunk_offs_host,
                    const uint8_t* vertex_dev, int64_t n, int32_t vertex_row, const int32_t* vertex_offs_host,
                    const uint8_t* sh_dev, int32_t sh_row, const int32_t* sh_offs_host, int32_t nsh,
                    const float* tables_dev, uint8_t* rows_dev, void* stream);
/* The SOG reader (formats/sog.py:23-247, SogFormat.read) after the WebP step, in two launches on the same stream.
 * Textures are the decoded members' RGBA pixels (4 bytes each, 4-byte aligned).  An index the reference rejects with
 * IndexError ORs a bit into *error_dev (1: scales codebook, 2: sh0 codebook, 4: shN codebook, 8: label >= P); the
 * caller zeroes the word first and refuses the file if it is non-zero afterwards.
 * gsx_sog_decode_palette (sog.py:181-211, the palette double loop): palette_dev float32 [palette_size, coeffs]
 *   (coeffs 0, 9, 24 or 45), entry [i, c * C + j] = codebook_dev[byte c of centroids pixel (i / 64) * 64 * coeffs +
 *   (i % 64) * C + j], C = coeffs / 3: the reader's index formula, which differs from the writer's layout for entries
 *   >= 64 (reproduced, not fixed).  codebook_len entries past 256 are never indexed.
 * gsx_sog_decode (sog.py:60-179, 213-245): textures_host[6] = device pointers to the means_l, means_u, quats, scales,
 *   sh0 and shN_labels pixels (the last null without shN) -> n rows of 4 * (17 + coeffs) bytes, define_dtype(sh_degree =
 *   bands).  position_tables_dev float32 [3, 65536]: x, y, z of each u16 code; tables_dev float32 [4, 256]: quaternion
 *   component (u8 / 255 - 0.5) * 2, opacity logit, scales codebook, sh0 codebook (each padded to 256).  Quaternion:
 *   max_comp = uint8(alpha - 252), missing = sqrt(max(1 - ((a*a + b*b) + c*c), 0)) in float32, rot_* 0 for max_comp
 *   > 3; f_rest = palette_dev[R | G << 8 of the labels].  n < 2^31. */
int gsx_sog_decode_palette(const uint8_t* centroids_dev, int64_t palette_size, int32_t coeffs, const float* codebook_dev,
                           int32_t codebook_len, float* palette_dev, int32_t* error_dev, void* stream);
/* gsx_ply_transcode: the field mapping of the plain PLY readers and writers (formats/ply_3dgs.py:44-58 and :103-109,
 * formats/ply_cc.py:44-60 and :111-116: `converted[t] = vertices[s]`, `output_data[o] = data[f]` into np.zeros rows).
 * n rows of src_row_bytes bytes at src_dev -> n rows of dst_row_bytes bytes at dst_dev, both contiguous, any alignment,
 * rows of 1 .. 1024 bytes, n < 2^31.  fields_host int32 [nfields][4] = {src_off, src_type, dst_off, dst_type}, types
 * numbered 0 char (i1), 1 uchar (u1), 2 short, 3 ushort, 4 int, 5 uint, 6 float (f4), 7 double (f8); destination
 * bytes no field writes are 0 (the zero fill), fields may not overlap in the destination.  Casts as NumPy's structured
 * assignment on x86: identity (bytes copied); integer -> float round to nearest; double -> float round to nearest with
 * x86's NaN rule; integer -> uchar the low byte; float or double -> uchar the low byte of the truncation to int32, 0
 * for NaN and out-of-range values.  Other pairings are refused (GSX_ERR_ARG). */
int gsx_ply_transcode(const uint8_t* src_dev, int64_t n, int32_t src_row_bytes, uint8_t* dst_dev, int32_t dst_row_bytes,
                      const int32_t* fields_host, int32_t nfields, void* stream);
int gsx_sog_decode(const uint8_t* const* textures_host, int64_t n, const float* position_tables_dev,
                   const float* tables_dev, int32_t scale_codebook_len, int32_t sh0_codebook_len,
                   const float* palette_dev, int64_t palette_size, int32_t coeffs, uint8_t* rows_dev, int32_t* error_dev,
                   void* stream);

/* The SOG shN schedule (formats/sog.py:536-549: up to 64 chunks of one SH block, each clustered by its own
 * gpu_ops.kmeans call) in ONE call on HOST buffers: one upload of the block, one batched launch per phase.
 * nprob problems back to back in X_host (rows row_off[p] .. row_off[p+1]), K centroids each;
 * C_host_inout float32[nprob*K*D]: the init rows on entry, the centroids on return; labels_host int32[n]. */
int gsx_kmeans_host_batched(const float* X_host, const int64_t* row_off_host, int32_t nprob, int32_t K, int32_t D,
                            int32_t max_iter, float* C_host_inout, int32_t* labels_host, int32_t assign_mode);
/* Copies between a caller's HOST buffer and HBM, used by every *_host entry point above.  The reference's call sites
 * pass ordinary (pageable) NumPy arrays -- np.column_stack at data_processor.py:139, the shN block of
 * sog.py:536-549 -- which cudaMemcpy stages on one CPU thread; these stage through a pool of pinned
 * chunks filled / drained by several host threads (GSX_COPY_THREADS, default 8), each enqueueing its own DMAs, so
 * the PCIe link stays busy.  Pinned / registered / managed buffers and copies below 8 MiB take plain
 * cudaMemcpyAsync (GSX_STAGED_COPY=0 forces that path).
 * gsx_copy_h2d: on return src_host has been read completely and `stream` is ordered after the last chunk.
 * gsx_copy_d2h: waits for what `stream` has produced and BLOCKS until dst_host is complete. */
int gsx_copy_h2d(void* dst_dev, const void* src_host, int64_t bytes, void* stream);
int gsx_copy_d2h(void* dst_host, const void* src_dev, int64_t bytes, void* stream);
/* HOST-side row movement around the device filter chain when the 248-byte records stay on the host (no GPU work, several
 * CPU threads -- GSX_HOST_THREADS, default 16 on a big host): what the reference does with single-threaded NumPy.
 * gsx_host_gather_rows: dst[j] = src[idx[j]] for rows of row_bytes bytes -- the `vertices[mask]` compaction of
 *   data_processor.py:114,149,209,224 with the surviving row indices; every idx must lie in [0, n_rows).
 * gsx_host_extract_xyz_opacity: np.column_stack((v['x'], v['y'], v['z'])) and v['opacity'] of data_processor.py:38,139
 *   from packed records; the fields are float32 at the given byte offsets of a row (off_opacity < 0 and a null
 *   opacity_out_host: no opacity field). */
int gsx_host_gather_rows(const void* src_host, int64_t n_rows, int64_t row_bytes, const int64_t* idx_host, int64_t m,
                         void* dst_host);
int gsx_host_extract_xyz_opacity(const void* src_host, int64_t n_rows, int64_t row_bytes, int64_t off_x, int64_t off_y,
                                 int64_t off_z, int64_t off_opacity, float* xyz_out_host, float* opacity_out_host);
/* Free / total memory of the current device, for the sizing decisions of the host-buffer callers. */
int gsx_device_memory(int64_t* free_bytes, int64_t* total_bytes);

#ifdef __cplusplus
}
#endif
#endif /* GSX_H */

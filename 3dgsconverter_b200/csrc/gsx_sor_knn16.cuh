// gsx_sor_knn16.cuh -- the K <= 16 form of the neighbour search (included by gsx_sor.cu after k_sor_knn).
//
// k_sor_knn gives a whole warp to one query: its sorted K-list lives one rank per lane, so with K = 16 (the benchmark
// configuration, and every --sor_intensity up to 2.3) half of every list instruction is wasted, and ~60 % of the ~700
// warp instructions per query are list maintenance (serial inserts at ~11, 32-lane bitonic merges at ~95).  Here a warp
// carries TWO queries, one per 16-lane half: rank r of a half's list lives in lane r of that half, a scan step looks at
// 16 candidates per half, a serial insert serves both halves with one instruction stream, and the merge network is the
// 16-lane one (10 + 4 compare-exchange stages instead of 15 + 5).  Each half owns its own batch of 16 consecutive
// hash-sorted positions and the two halves walk their batches in lock step (query t of both batches together).
//
// The warp NEVER diverges: every loop runs while EITHER half still needs it (`__any_sync`) and a half that is done is
// predicated off with no-op inputs (an empty range, a sentinel candidate, an all-ones key).  A first version let the
// halves branch independently with half-warp masks on every shuffle / vote: once apart they never re-joined and every
// instruction issued twice with 16 lanes -- 3x SLOWER than k_sor_knn.  All
// shuffles here are full-mask with width 16 (or xor < 16), votes are full-mask ballots shifted to the half.
//
// Semantics are those of k_sor_knn (gpu_ops.py:98-176): same candidate set per query (the buckets of the 27 probes),
// same float32 op sequence for d^2, exact box pruning, and only the multiset of the K smallest d^2 matters -- the
// visiting order is free, and scanning a sentinel or re-inserting a value >= rank K-1 changes nothing.  With 16 lanes a
// lane carries two of the 27 probes (p and p + 16) and, inside a long bucket, two of the 32 chunk boxes of a super.

#ifndef GSX_MERGE16_THRESHOLD
#define GSX_MERGE16_THRESHOLD 4
#endif
#ifndef GSX_KNN16_MINBLOCKS
#define GSX_KNN16_MINBLOCKS 6
#endif

struct Lanes16 {
    int base;   // first lane of this half (0 or 16)
    int hl;     // lane inside the half
    __device__ __forceinline__ unsigned ballot(bool p) const { return (__ballot_sync(GSX_FULL, p) >> base) & 0xffffu; }
    template <class T>
    __device__ __forceinline__ T bcast(T x, int src_hl) const { return __shfl_sync(GSX_FULL, x, src_hl, 16); }
    // minima over both halves, known to every lane (one redux per half, the other half feeds the neutral element):
    // returns this half's minimum, `either` = some half has a key that is not all-ones -- no vote needed
    __device__ __forceinline__ unsigned hmin(unsigned x, bool& either) const {
        const unsigned lo = __reduce_min_sync(GSX_FULL, base ? 0xffffffffu : x);
        const unsigned hi = __reduce_min_sync(GSX_FULL, base ? x : 0xffffffffu);
        either = (lo & hi) != 0xffffffffu;
        return base ? hi : lo;
    }
};

struct TopK16 {
    float v;     // lane hl holds rank hl of the ascending d^2 list
    float tau;   // rank K-1, uniform inside the half
    int K;
    __device__ __forceinline__ void init(int k) {
        K = k;
        v = tau = __uint_as_float(GSX_D2LIM_BITS);
    }
    __device__ __forceinline__ void refresh_tau(const Lanes16& L) { tau = L.bcast(v, K - 1); }
    // insert x (uniform inside the half; x >= rank K-1, e.g. the sentinel, only moves ranks >= K or nothing)
    __device__ __forceinline__ void insert(float x, const Lanes16& L) {
        float up = __shfl_up_sync(GSX_FULL, v, 1, 16);
        if (L.hl == 0) up = 0.f;
        if (v > x) v = fmaxf(up, x);
    }
    // merge one candidate per lane (sentinel where there is none): bitonic sort of the 16 new values, reversed,
    // lane-wise min with the ascending list = the 16 smallest of the union as a bitonic sequence, 4 stages sort it.
    // All sentinels in => the list comes out unchanged.
    __device__ __forceinline__ void merge16(float nv, const Lanes16& L) {
        const int hl = L.hl;
#pragma unroll
        for (int k = 2; k <= 16; k <<= 1) {
#pragma unroll
            for (int j = k >> 1; j > 0; j >>= 1) {
                const float o = __shfl_xor_sync(GSX_FULL, nv, j);
                nv = (((hl & k) == 0) == ((hl & j) == 0)) ? fminf(nv, o) : fmaxf(nv, o);
            }
        }
        const float r = L.bcast(nv, 15 - hl);
        float m = fminf(v, r);
#pragma unroll
        for (int j = 8; j > 0; j >>= 1) {
            const float o = __shfl_xor_sync(GSX_FULL, m, j);
            m = ((hl & j) == 0) ? fminf(m, o) : fmaxf(m, o);
        }
        v = m;
    }
};

// 16 candidates per half: position j of this lane (valid where inside the bucket this half is scanning; a half with
// nothing to scan passes valid == false everywhere)
template <bool STATS>
__device__ __forceinline__ void scan16(const float4* __restrict__ spos, pos_t j, bool valid, float qx, float qy, float qz,
                                       TopK16& tk, const Lanes16& L, unsigned long long& n_scanned) {
    const float sentinel = __uint_as_float(GSX_D2LIM_BITS);
    float d2 = sentinel;
    if (valid) {
        const float4 c = __ldg(spos + j);
        const float ax = __fsub_rn(qx, c.x), ay = __fsub_rn(qy, c.y), az = __fsub_rn(qz, c.z);
        d2 = __fadd_rn(__fadd_rn(__fmul_rn(ax, ax), __fmul_rn(ay, ay)), __fmul_rn(az, az));
    }
    if (STATS) n_scanned += __popc(L.ballot(valid));
    const bool pass = valid && d2 > 1.0e-12f && d2 < tk.tau;
    // one full-warp vote: every lane knows BOTH halves' masks, so the loop conditions below need no further votes
    const unsigned mall = __ballot_sync(GSX_FULL, pass);
    if (!mall) return;
    unsigned mlo = mall & 0xffffu, mhi = mall >> 16;
    const bool mg_lo = __popc(mlo) >= GSX_MERGE16_THRESHOLD, mg_hi = __popc(mhi) >= GSX_MERGE16_THRESHOLD;
    if (mg_lo || mg_hi) {
        const bool domerge = L.base ? mg_hi : mg_lo;
        tk.merge16((domerge && pass) ? d2 : sentinel, L);   // a half that is not merging feeds sentinels: no change
        if (mg_lo) mlo = 0u;
        if (mg_hi) mhi = 0u;
    }
    while (mlo | mhi) {
        const unsigned m = L.base ? mhi : mlo;
        float x = L.bcast(d2, m ? __ffs(m) - 1 : 0);
        if (!m) x = sentinel;                               // this half has nothing left: a no-op insert
        mlo &= mlo - 1;
        mhi &= mhi - 1;
        tk.insert(x, L);
    }
    tk.refresh_tau(L);
}

template <bool STATS>
__global__ void __launch_bounds__(256, GSX_KNN16_MINBLOCKS)
    k_sor_knn16(const float4* __restrict__ spos, const int2* __restrict__ tab_se, const float4* __restrict__ tab_box,
                const uint32_t* __restrict__ cellbits, const float4* __restrict__ caabb, const float4* __restrict__ saabb,
                float* __restrict__ final_means, unsigned int* __restrict__ work, int64_t q_begin, int64_t q_end,
                int q_stride, int q_phase, int K, int hash_mode, float bx, float by, float bz, float cell, uint32_t n,
                uint64_t M, unsigned long long* __restrict__ stats) {
    static_assert(!GSX_KNN16 || kQueryBatch == 16, "a half-warp batch is one 16-position run");
    const int lane = lane_id();
    Lanes16 L;
    L.base = lane & 16;
    L.hl = lane & 15;
    const int hl = L.hl;
    unsigned long long st_visits = 0, st_scanned = 0, st_boxes = 0, st_queries = 0;
    // probes of lane hl: p0 = hl (always < 27) and p1 = hl + 16 (< 27 for hl < 11), reference loop order (dx outer)
    const int p1 = hl + 16;
    const bool has1 = p1 < 27;
    const int dx0 = hl / 9 - 1, dy0 = (hl / 3) % 3 - 1, dz0 = hl % 3 - 1;
    const int dx1 = p1 / 9 - 1, dy1 = (p1 / 3) % 3 - 1, dz1 = p1 % 3 - 1;

    for (;;) {
        unsigned int b0 = 0;
        if (lane == 0) b0 = atomicAdd(work, 2u * (unsigned)kQueryBatch);
        b0 = __shfl_sync(GSX_FULL, b0, 0);
        // the warp took two consecutive batches of this launch; half h works on batch b0/16 + h (global batch number
        // (.)*q_stride + q_phase, see k_sor_knn)
        const int64_t qb_lo = q_begin + ((int64_t)(b0 / kQueryBatch) * q_stride + q_phase) * kQueryBatch;
        if (qb_lo >= q_end) break;   // the lower batch is the earlier one: nothing left for either half
        const int64_t qb64 = q_begin + ((int64_t)(b0 / kQueryBatch + (L.base >> 4)) * q_stride + q_phase) * kQueryBatch;
        const bool have = qb64 < q_end;                      // (only the upper half can be without a batch)
        const pos_t qb = have ? (pos_t)qb64 : 0;             // positions fit 31 bits (pos_t)
        const int nq = !have ? 0 : (qb64 + kQueryBatch <= q_end ? kQueryBatch : (int)(q_end - qb64));
        int ps0 = 0, pc0 = 0, ps1 = 0, pc1 = 0;
        float l0x = 0.f, l0y = 0.f, l0z = 0.f, h0x = 0.f, h0y = 0.f, h0z = 0.f;
        float l1x = 0.f, l1y = 0.f, l1z = 0.f, h1x = 0.f, h1y = 0.f, h1z = 0.f;
#pragma unroll 1
        for (int t = 0; t < kQueryBatch; ++t) {
            const bool aq = t < nq;                          // this half has a query in this round
            if (!__any_sync(GSX_FULL, aq)) break;
            const pos_t i = qb + t;
            float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
            bool newcell = false;
            if (aq) {
                q = __ldg(spos + i);
                newcell = t == 0 || ((__ldg(cellbits + (i >> 5)) >> (i & 31)) & 1u);
            }
            if (__any_sync(GSX_FULL, newcell)) {
                const int gx = (int)floorf(__fdiv_rn(__fsub_rn(q.x, bx), cell));
                const int gy = (int)floorf(__fdiv_rn(__fsub_rn(q.y, by), cell));
                const int gz = (int)floorf(__fdiv_rn(__fsub_rn(q.z, bz), cell));
                if (newcell) {
                    const uint32_t h = probe_hash(gx + dx0, gy + dy0, gz + dz0, n, M, hash_mode);
                    const int2 se = __ldg(tab_se + h);
                    ps0 = se.x, pc0 = se.y - se.x;
                    if (pc0 > 0) {
                        const float4 a = __ldg(tab_box + 2 * (size_t)h), b = __ldg(tab_box + 2 * (size_t)h + 1);
                        l0x = a.x, l0y = a.y, l0z = a.z, h0x = b.x, h0y = b.y, h0z = b.z;
                    }
                    ps1 = 0, pc1 = 0;
                    if (has1) {
                        const uint32_t g = probe_hash(gx + dx1, gy + dy1, gz + dz1, n, M, hash_mode);
                        const int2 se1 = __ldg(tab_se + g);
                        ps1 = se1.x, pc1 = se1.y - se1.x;
                        if (pc1 > 0) {
                            const float4 a = __ldg(tab_box + 2 * (size_t)g), b = __ldg(tab_box + 2 * (size_t)g + 1);
                            l1x = a.x, l1y = a.y, l1z = a.z, h1x = b.x, h1y = b.y, h1z = b.z;
                        }
                    }
                }
            }
            if (STATS) {
                int tot = aq ? pc0 + pc1 : 0;
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) tot += __shfl_xor_sync(GSX_FULL, tot, o);
                if (hl == 0 && aq) {
                    st_visits += (unsigned long long)tot;
                    st_queries += 1;
                }
            }
            TopK16 tk;
            tk.init(K);
            // lower bounds of d^2 to the probes' boxes (same monotone op sequence as d^2, see box_lb); a half without a
            // query keeps all-ones keys and therefore visits nothing
            unsigned pk0 = 0xffffffffu, pk1 = 0xffffffffu;
            if (aq && pc0 > 0) {
                const float dx = fmaxf(fmaxf(__fsub_rn(l0x, q.x), __fsub_rn(q.x, h0x)), 0.f);
                const float dy = fmaxf(fmaxf(__fsub_rn(l0y, q.y), __fsub_rn(q.y, h0y)), 0.f);
                const float dz = fmaxf(fmaxf(__fsub_rn(l0z, q.z), __fsub_rn(q.z, h0z)), 0.f);
                pk0 = __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            }
            if (aq && pc1 > 0) {
                const float dx = fmaxf(fmaxf(__fsub_rn(l1x, q.x), __fsub_rn(q.x, h1x)), 0.f);
                const float dy = fmaxf(fmaxf(__fsub_rn(l1y, q.y), __fsub_rn(q.y, h1y)), 0.f);
                const float dz = fmaxf(fmaxf(__fsub_rn(l1z, q.z), __fsub_rn(q.z, h1z)), 0.f);
                pk1 = __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            }

            // seed from the 32-position chunk that holds the query when its own bucket is a long one (legal only if
            // the centre probe -- lane 13, slot 0 -- really reaches the query's bucket range, SURVEY F8)
            int skip_chunk = -1;
            {
                const int s13 = L.bcast(ps0, 13), c13 = L.bcast(pc0, 13);
                const bool seed = aq && c13 > kSmallBucket && i >= s13 && i < (pos_t)s13 + c13;
                if (__any_sync(GSX_FULL, seed)) {
                    if (seed) skip_chunk = (int)(i >> 5);
                    const pos_t j0 = ((pos_t)(i >> 5) << 5) + hl;
                    scan16<STATS>(spos, j0, seed && j0 >= s13 && j0 < (pos_t)s13 + c13, q.x, q.y, q.z, tk, L, st_scanned);
                    scan16<STATS>(spos, j0 + 16, seed && j0 + 16 >= s13 && j0 + 16 < (pos_t)s13 + c13, q.x, q.y, q.z, tk, L,
                                  st_scanned);
                }
            }

#pragma unroll 1
            for (;;) {
                // keys >= tau can never be visited again (tau only falls): mask them here, so "some key left" is the
                // whole loop condition and both halves' minima tell every lane whether either half goes on
                const unsigned taub = __float_as_uint(tk.tau);
                unsigned mine = pk0 < pk1 ? pk0 : pk1;
                if (!(mine < taub)) mine = 0xffffffffu;
                bool either;
                const unsigned mp = L.hmin(mine, either);
                if (!either) break;
                const bool go = mp != 0xffffffffu;                                   // uniform inside the half
                const unsigned holders = L.ballot(go && mine == mp);
                const int pl = holders ? __ffs(holders) - 1 : 0;                   // lane (in the half) of the nearest probe
                const bool slot0 = pk0 == mp;                                      // (meaningful in lane pl)
                const int s = L.bcast(slot0 ? ps0 : ps1, pl);
                int c = L.bcast(slot0 ? pc0 : pc1, pl);
                const bool centre = L.bcast((int)(slot0 && hl == 13), pl) != 0;
                if (go && hl == pl) {
                    if (slot0) pk0 = 0xffffffffu;
                    else pk1 = 0xffffffffu;
                }
                if (!go) c = 0;                                                    // this half is done: empty range
                const pos_t e = (pos_t)s + c;
                const bool big = c > kSmallBucket;
                {   // short buckets (the common case), both halves together
                    pos_t b = s;
                    const pos_t eb = big ? s : e;
#pragma unroll 1
                    while (__any_sync(GSX_FULL, b < eb)) {
                        scan16<STATS>(spos, b + hl, b + hl < eb, q.x, q.y, q.z, tk, L, st_scanned);
                        b += 16;
                    }
                }
                if (!__any_sync(GSX_FULL, big)) continue;
                // long bucket: supers (1024 positions) nearest box first, then their chunks (32 positions)
                const int skip = centre ? skip_chunk : -1;
                const int fc = s >> 5, lc = (int)((e - 1) >> 5);
                const int fs = big ? fc >> 5 : 1, ls = big ? lc >> 5 : 0;          // not big: an empty super range
                int sb = fs;
#pragma unroll 1
                while (__any_sync(GSX_FULL, sb <= ls)) {
                    const int sid = sb + hl;
                    const bool sv = sb <= ls && sid <= ls;
                    unsigned skey = 0xffffffffu;
                    if (sv) {
                        const float lb = box_lb(saabb, sid, q.x, q.y, q.z);
                        if (lb < tk.tau) skey = __float_as_uint(lb);
                    }
                    if (STATS) st_boxes += __popc(L.ballot(sv));
#pragma unroll 1
                    for (;;) {
                        if (!(skey < __float_as_uint(tk.tau))) skey = 0xffffffffu;
                        bool either_s;
                        const unsigned ms = L.hmin(skey, either_s);
                        if (!either_s) break;
                        const bool gos = ms != 0xffffffffu;
                        const unsigned sh = L.ballot(gos && skey == ms);
                        const int sl = sh ? __ffs(sh) - 1 : 0;
                        if (gos && hl == sl) skey = 0xffffffffu;
                        const int sup = sb + sl;
                        // the 32 chunks of the super: lane hl holds chunks hl and hl + 16
                        const int cid0 = sup * 32 + hl, cid1 = cid0 + 16;
                        const bool cv0 = gos && cid0 >= fc && cid0 <= lc && cid0 != skip;
                        const bool cv1 = gos && cid1 >= fc && cid1 <= lc && cid1 != skip;
                        unsigned ck0 = 0xffffffffu, ck1 = 0xffffffffu;
                        if (cv0) {
                            const float lb = box_lb(caabb, cid0, q.x, q.y, q.z);
                            if (lb < tk.tau) ck0 = __float_as_uint(lb);
                        }
                        if (cv1) {
                            const float lb = box_lb(caabb, cid1, q.x, q.y, q.z);
                            if (lb < tk.tau) ck1 = __float_as_uint(lb);
                        }
                        if (STATS) st_boxes += __popc(L.ballot(cv0)) + __popc(L.ballot(cv1));
#pragma unroll 1
                        for (;;) {
                            unsigned cmine = ck0 < ck1 ? ck0 : ck1;
                            if (!(cmine < __float_as_uint(tk.tau))) cmine = 0xffffffffu;
                            bool either_c;
                            const unsigned mc = L.hmin(cmine, either_c);
                            if (!either_c) break;
                            const bool goc = mc != 0xffffffffu;
                            const unsigned chh = L.ballot(goc && cmine == mc);
                            const int cl = chh ? __ffs(chh) - 1 : 0;
                            const bool cs0 = ck0 == mc;
                            const int chunk = L.bcast(cs0 ? cid0 : cid1, cl);
                            if (goc && hl == cl) {
                                if (cs0) ck0 = 0xffffffffu;
                                else ck1 = 0xffffffffu;
                            }
                            const pos_t j0 = ((pos_t)chunk << 5) + hl;
                            scan16<STATS>(spos, j0, goc && j0 >= s && j0 < e, q.x, q.y, q.z, tk, L, st_scanned);
                            scan16<STATS>(spos, j0 + 16, goc && j0 + 16 >= s && j0 + 16 < e, q.x, q.y, q.z, tk, L, st_scanned);
                        }
                    }
                    sb += 16;
                }
            }

            // gpu_ops.py:163-174: ascending serial float32 sum of the valid (< 0.9e10) distances (a prefix of the list)
            const float d = __fsqrt_rn(tk.v);
            const int valid = __popc(L.ballot(hl < K && d < 0.9e10f));
            float sum = 0.f;
#pragma unroll 1
            for (int r = 0; __any_sync(GSX_FULL, r < valid); ++r) {
                const float x = L.bcast(d, r & 15);
                if (r < valid) sum = __fadd_rn(sum, x);
            }
            if (aq && hl == 0) final_means[__float_as_int(q.w)] = valid > 0 ? __fdiv_rn(sum, (float)valid) : 0.f;
        }
    }
    if (STATS && hl == 0) {
        atomicAdd(stats + 0, st_visits);
        atomicAdd(stats + 1, st_scanned);
        atomicAdd(stats + 2, st_boxes);
        atomicAdd(stats + 3, st_queries);
    }
}

// Device-side matcher (S2 + S3) shared by k_match_triangulate (match_kernels.cu) and the fused
// pipeline kernel (fused_kernel.cu).  Semantics: see match_kernels.cu.
#pragma once
#include "common.cuh"
#include "geom.cuh"

#define FULL_MASK 0xffffffffu

struct WarpState {
    uint8_t* rcam;     // [RMAX] camera of the root
    uint8_t* rpt;      // [RMAX] blob index of the root in its camera
    uint8_t* ncand;    // [RMAX][C]
    uint8_t* cand;     // [RMAX][C][KC] blob indices sorted by distance to the root's epipolar line
    uint32_t* gcount;  // [RMAX] number of candidate groups (0: root has < 2 views)
    uint32_t* gprefix; // [RMAX+1]
    unsigned long long* best_key;  // [RMAX]
    uint32_t* best_g;  // [RMAX]
    double* best_xe;   // [RMAX][4]  X and error of the best group so far
    int32_t* xy_s;     // [C][MB][2] the frame-set's blob centres, staged once (every later read is a shared-memory load)
};

static __host__ __device__ size_t warp_state_bytes(int RMAX, int C, int KC, int MB) {
    size_t b = 0;
    b += (size_t)RMAX * 32;                      // best_xe
    b += (size_t)RMAX * 8;                       // best_key
    b += (size_t)RMAX * 4 * 2 + (RMAX + 1) * 4;  // gcount, best_g, gprefix
    b += (size_t)C * MB * 8;                     // xy_s
    b += (size_t)RMAX * 2;                       // rcam, rpt
    b += (size_t)RMAX * C;                       // ncand
    b += (size_t)RMAX * C * KC;                  // cand
    return (b + 15) & ~(size_t)15;
}
inline size_t match_smem_bytes(const mocap_config& cfg, int warps) {
    return warp_state_bytes(cfg.max_roots, cfg.n_cam, cfg.max_cands, cfg.max_blobs) * warps;
}
__device__ __forceinline__ WarpState carve_warp_state(unsigned char* raw, int RMAX, int C, int KC, int MB) {
    WarpState s;
    s.best_xe = reinterpret_cast<double*>(raw);              raw += (size_t)RMAX * 32;
    s.best_key = reinterpret_cast<unsigned long long*>(raw); raw += (size_t)RMAX * 8;
    s.gcount = reinterpret_cast<uint32_t*>(raw);             raw += (size_t)RMAX * 4;
    s.best_g = reinterpret_cast<uint32_t*>(raw);             raw += (size_t)RMAX * 4;
    s.gprefix = reinterpret_cast<uint32_t*>(raw);            raw += (size_t)(RMAX + 1) * 4;
    s.xy_s = reinterpret_cast<int32_t*>(raw);                raw += (size_t)C * MB * 8;
    s.rcam = raw;                                            raw += RMAX;
    s.rpt = raw;                                             raw += RMAX;
    s.ncand = raw;                                           raw += (size_t)RMAX * C;
    s.cand = raw;
    return s;
}

// error -> ordered integer key.  np.argmin treats NaN as the minimum (first NaN wins).
__device__ __forceinline__ unsigned long long err_key(double e) {
    if (e != e) return 0ull;
    return (unsigned long long)__double_as_longlong(e) + 1ull;    // e >= 0
}

// views of group g of root r: the root's own blob plus, per later camera with candidates, the
// candidate selected by g's mixed-radix digit (earliest camera = least significant digit)
__device__ __forceinline__ int decode_group(const WarpState& ws, int C, int KC, int r, uint32_t g,
                                            int cams[MOCAP_MAX_CAM], int pts[MOCAP_MAX_CAM]) {
    const int rc = ws.rcam[r];
    cams[0] = rc; pts[0] = ws.rpt[r];
    int nv = 1;
    uint32_t rem = g;
    for (int i = rc + 1; i < C; ++i) {
        const int k = ws.ncand[r * C + i];
        if (k > 0) {
            int d = 0;
            if (k > 1) {                                           // most cameras offer a single candidate: no division
                const uint32_t qd = rem / (uint32_t)k;
                d = (int)(rem - qd * (uint32_t)k);
                rem = qd;
            }
            cams[nv] = i;
            pts[nv] = ws.cand[((size_t)r * C + i) * KC + d];
            ++nv;
        }
    }
    return nv;
}

// DLT + reprojection error of group g of root r.
static __device__ __noinline__ void eval_group(const CameraTables* __restrict__ tb, const WarpState& ws,
                                           const int32_t* xy, int MB, int C, int KC,
                                           int r, uint32_t g, double X[3], double& err) {
    Sym4 B;
    sym4_zero(B);
    int cams[MOCAP_MAX_CAM];
    int pts[MOCAP_MAX_CAM];
    const int nv = decode_group(ws, C, KC, r, g, cams, pts);
#pragma unroll 1
    for (int k = 0; k < nv; ++k) {
        const int c = cams[k];
        const double px = (double)xy[((size_t)c * MB + pts[k]) * 2 + 0];
        const double py = (double)xy[((size_t)c * MB + pts[k]) * 2 + 1];
        dlt_add_view(B, tb->Pkc[k][c], px, py);      // K of the k-th PRESENT view (helpers.py:305-307)
    }
    dlt_solve(B, X);
    double sq[2 * MOCAP_MAX_CAM];
#pragma unroll 1
    for (int k = 0; k < nv; ++k) {
        const int c = cams[k];
        float u, v;
        project_like_cv(tb->R[c], tb->t[c], tb->fx[k], tb->fy[k], tb->cx[k], tb->cy[k], X, u, v);
        const double dx = DSUB((double)xy[((size_t)c * MB + pts[k]) * 2 + 0], (double)u);
        const double dy = DSUB((double)xy[((size_t)c * MB + pts[k]) * 2 + 1], (double)v);
        sq[2 * k] = DMUL(dx, dx);
        sq[2 * k + 1] = DMUL(dy, dy);
    }
    // a group without None entries is an int64 array in the reference (pairwise float64 sum);
    // any None turns it into an object array (left fold)
    err = mean_like_numpy(sq, 2 * nv, nv == C);
}

// cv.computeCorrespondEpilines of the float32 point (rx, ry) with F (helpers.py:362-364): double math, the float32 line
// (a, b, c) returned as doubles.  The detection overlay draws the same lines (overlay.cu).
__device__ __forceinline__ void epiline_f32(const double* F, double rx, double ry, double& a, double& b, double& c) {
    a = DADD(DADD(DMUL(F[0], rx), DMUL(F[1], ry)), F[2]);
    b = DADD(DADD(DMUL(F[3], rx), DMUL(F[4], ry)), F[5]);
    c = DADD(DADD(DMUL(F[6], rx), DMUL(F[7], ry)), F[8]);
    double nu = DADD(DMUL(a, a), DMUL(b, b));
    nu = (nu != 0.0) ? 1.0 / sqrt(nu) : 1.0;
    a = (double)(float)DMUL(a, nu);
    b = (double)(float)DMUL(b, nu);
    c = (double)(float)DMUL(c, nu);
}

// The matcher of one frame-set is three steps of one warp: prepare (roots, candidate lists, group counts), evaluate a
// range of the frame-set's candidate groups (per-root best so far in shared memory), emit (winners in root order).
// match_triangulate_warp runs them back to back; k_match_chunks (match_kernels.cu) gives the middle step of a frame-set
// with thousands of groups to several warps, one range each.
struct MatchPrep { int nr; uint32_t total; int flags; };

// xy / nb are read with ld.global.cg so that the function may consume blob lists written earlier IN THE SAME KERNEL by
// other warps (fused pipeline).  Leaves the staged blob centres in ws.xy_s (every later step reads those).
static __device__ __forceinline__ MatchPrep match_prepare_warp(
    const CameraTables* __restrict__ tb, const WarpState& ws, const int32_t* xy, const int32_t* nb, int lane,
    int C, int MB, int RMAX, int KC, uint32_t GMAX, const int32_t* img_flags) {
    int flags = 0;
    // inside a pipeline: what S1 reported for the frame-set's images (truncated blob lists, blobs with holes) travels
    // with the frame-set
    if (img_flags) {
        int f = lane < C ? __ldcg(img_flags + lane) : 0;
#pragma unroll 1
        for (int o = 16; o > 0; o >>= 1) f |= __shfl_xor_sync(FULL_MASK, f, o);
        flags = f;
    }

    // stage the blob centres of the frame-set's cameras (read with ld.global.cg: they may have been written earlier
    // in the same kernel by other warps) -- the matcher re-reads them hundreds of times
    {
        const int32_t* gxy = xy;
        for (int c = 0; c < C; ++c) {
            const int k2 = 2 * min(__ldcg(nb + c), MB);
            for (int q = lane; q < k2; q += 32) ws.xy_s[c * MB * 2 + q] = __ldcg(gxy + (size_t)c * MB * 2 + q);
        }
        __syncwarp();
        xy = ws.xy_s;
    }

    // roots from camera 0 (helpers.py:349,357)
    int nr = min(__ldcg(nb), MB);
    if (nr > RMAX) { nr = RMAX; flags |= MOCAP_F_ROOTS; }
    for (int r = lane; r < RMAX; r += 32) {
        if (r < nr) { ws.rcam[r] = 0; ws.rpt[r] = (uint8_t)r; }
        for (int i = 0; i < C; ++i) ws.ncand[r * C + i] = 0;
    }
    __syncwarp();

    for (int i = 1; i < C; ++i) {                              // helpers.py:359
        const int ni = min(__ldcg(nb + i), MB);
        unsigned long long matched = 0ull;                     // "closest match" blobs of camera i
        for (int j = lane; j < nr; j += 32) {                  // roots that exist before camera i
            const int rc = ws.rcam[j];
            const double rx = (double)xy[((size_t)rc * MB + ws.rpt[j]) * 2 + 0];
            const double ry = (double)xy[((size_t)rc * MB + ws.rpt[j]) * 2 + 1];
            double a, b, c;
            epiline_f32(tb->F[rc][i], rx, ry, a, b, c);
            const double den = sqrt(DADD(DMUL(a, a), DMUL(b, b)));      // helpers.py:373
            double dist[MOCAP_MAX_CANDS];
            uint8_t* cl = ws.cand + ((size_t)j * C + i) * KC;
            int cnt = 0;
#pragma unroll 1
            for (int q = 0; q < ni; ++q) {
                const double px = (double)xy[((size_t)i * MB + q) * 2 + 0];
                const double py = (double)xy[((size_t)i * MB + q) * 2 + 1];
                const double d = fabs(DADD(DADD(DMUL(a, px), DMUL(b, py)), c)) / den;
                if (d < 5.0) {                                  // helpers.py:375
                    if (cnt == KC) {
                        flags |= MOCAP_F_CANDS;
                        if (!(d < dist[KC - 1])) continue;
                        --cnt;
                    }
                    int pos = cnt;                              // stable insertion: after every dist <= d
                    while (pos > 0 && dist[pos - 1] > d) { dist[pos] = dist[pos - 1]; cl[pos] = cl[pos - 1]; --pos; }
                    dist[pos] = d; cl[pos] = (uint8_t)q;
                    ++cnt;
                }
            }
            ws.ncand[j * C + i] = (uint8_t)cnt;
            if (cnt > 0) {                                      // helpers.py:391: drop every row equal to the closest match
                const int q0 = cl[0];
                const int cx0 = xy[((size_t)i * MB + q0) * 2 + 0], cy0 = xy[((size_t)i * MB + q0) * 2 + 1];
                for (int q = 0; q < ni; ++q)
                    if (xy[((size_t)i * MB + q) * 2 + 0] == cx0 && xy[((size_t)i * MB + q) * 2 + 1] == cy0)
                        matched |= 1ull << q;
            }
        }
#pragma unroll 1
        for (int o = 16; o > 0; o >>= 1) matched |= __shfl_xor_sync(FULL_MASK, matched, o);
        // blobs of camera i that were nobody's closest match become roots (helpers.py:402-406)
        for (int q0 = 0; q0 < ni; q0 += 32) {
            const int q = q0 + lane;
            const bool un = q < ni && !((matched >> q) & 1ull);
            const unsigned bal = __ballot_sync(FULL_MASK, un);
            const int pos = nr + __popc(bal & ((1u << lane) - 1u));
            if (un) {
                if (pos < RMAX) { ws.rcam[pos] = (uint8_t)i; ws.rpt[pos] = (uint8_t)q; }
                else flags |= MOCAP_F_ROOTS;
            }
            nr = min(nr + __popc(bal), RMAX);
        }
        __syncwarp();
    }

    // number of candidate groups of every root
    for (int r0 = 0; r0 < nr; r0 += 32) {
        const int r = r0 + lane;
        uint32_t G = 0;
        if (r < nr) {
            unsigned long long prod = 1ull;
            int views = 1;
            for (int i = ws.rcam[r] + 1; i < C; ++i) {
                const int k = ws.ncand[r * C + i];
                if (k > 0) { prod *= (unsigned long long)k; ++views; if (prod > GMAX) { prod = GMAX; flags |= MOCAP_F_GROUPS; } }
            }
            G = views >= 2 ? (uint32_t)prod : 0u;
            ws.gcount[r] = G;
            ws.best_key[r] = ~0ull;
            ws.best_g[r] = 0u;
        }
    }
    __syncwarp();
    if (lane == 0) {
        uint32_t acc = 0;
        for (int r = 0; r < nr; ++r) { ws.gprefix[r] = acc; acc += ws.gcount[r]; }
        ws.gprefix[nr] = acc;
    }
    __syncwarp();
    MatchPrep prep;
    prep.nr = nr; prep.total = ws.gprefix[nr]; prep.flags = flags;
    return prep;
}

// groups [w_lo, w_hi) of the frame-set (numbered through the roots in order; w_lo a multiple of 32): every group's point
// and error; segmented warp argmin; the head lane of every root's segment pulls the winner's point over by shuffle and
// folds it into shared memory.  Ranges evaluated in ascending order give what one pass over [0, total) gives.
static __device__ __forceinline__ void match_eval_range_warp(
    const CameraTables* __restrict__ tb, const WarpState& ws, int lane, int C, int MB, int KC, int nr, uint32_t w_lo, uint32_t w_hi) {
    const int32_t* xy = ws.xy_s;
    for (uint32_t w0 = w_lo; w0 < w_hi; w0 += 32) {
        const uint32_t w = w0 + lane;
        int r = -1;
        uint32_t g = 0;
        unsigned long long key = ~0ull;
        double X[3] = {0.0, 0.0, 0.0}, e = 0.0;
        if (w < w_hi) {
            int lo = 0, hi = nr;                               // last r with gprefix[r] <= w
            while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (ws.gprefix[mid] <= w) lo = mid; else hi = mid; }
            r = lo;
            g = w - ws.gprefix[r];
            eval_group(tb, ws, xy, MB, C, KC, r, g, X, e);
            key = err_key(e);
        }
        int src = lane;
#pragma unroll 1
        for (int o = 1; o < 32; o <<= 1) {
            const int r2 = __shfl_down_sync(FULL_MASK, r, o);
            const uint32_t g2 = __shfl_down_sync(FULL_MASK, g, o);
            const unsigned long long k2 = __shfl_down_sync(FULL_MASK, key, o);
            const int s2 = __shfl_down_sync(FULL_MASK, src, o);
            if (lane + o < 32 && r2 == r && (k2 < key || (k2 == key && g2 < g))) { key = k2; g = g2; src = s2; }
        }
        const double bx = __shfl_sync(FULL_MASK, X[0], src), by = __shfl_sync(FULL_MASK, X[1], src);
        const double bz = __shfl_sync(FULL_MASK, X[2], src), be = __shfl_sync(FULL_MASK, e, src);
        const int rprev = __shfl_up_sync(FULL_MASK, r, 1);
        const bool head = (r >= 0) && (lane == 0 || rprev != r);
        if (head && key < ws.best_key[r]) {                    // ties keep the earlier group (np.argmin)
            ws.best_key[r] = key; ws.best_g[r] = g;
            ws.best_xe[4 * r + 0] = bx; ws.best_xe[4 * r + 1] = by; ws.best_xe[4 * r + 2] = bz; ws.best_xe[4 * r + 3] = be;
        }
        __syncwarp();
    }
}

// winners, compacted in root order (helpers.py:413-419 skips roots without a 3D point)
static __device__ __forceinline__ void match_emit_warp(
    const CameraTables* __restrict__ tb, const WarpState& ws, int set, int lane, int C, int MB, int RMAX, int KC, int nr, int flags,
    double* __restrict__ obj, double* __restrict__ err_out, int32_t* __restrict__ n_obj, int32_t* __restrict__ set_flags,
    int32_t* __restrict__ chosen, int32_t* __restrict__ track_xy) {
    const int32_t* xy = ws.xy_s;
    int n_out = 0;
    double* obj_s = obj + (size_t)set * RMAX * 3;
    double* err_s = err_out + (size_t)set * RMAX;
    int32_t* ch_s = chosen ? chosen + (size_t)set * RMAX * C : nullptr;
    int32_t* tx_s = track_xy ? track_xy + (size_t)set * RMAX * C * 2 : nullptr;   // the winner's pixel per camera, (-1, -1) = no view
    for (int r0 = 0; r0 < nr; r0 += 32) {
        const int r = r0 + lane;
        const bool has = r < nr && ws.gcount[r] > 0;
        const unsigned bal = __ballot_sync(FULL_MASK, has);
        if (has) {
            const int o = n_out + __popc(bal & ((1u << lane) - 1u));
            double X[3] = {ws.best_xe[4 * r], ws.best_xe[4 * r + 1], ws.best_xe[4 * r + 2]};
            const double e = ws.best_xe[4 * r + 3];
            if (ch_s || tx_s) {
                int cams[MOCAP_MAX_CAM], pts[MOCAP_MAX_CAM];
                const int nv = decode_group(ws, C, KC, r, ws.best_g[r], cams, pts);
                if (ch_s) {
                    for (int i = 0; i < C; ++i) ch_s[(size_t)o * C + i] = -1;
                    for (int k = 0; k < nv; ++k) ch_s[(size_t)o * C + cams[k]] = pts[k];
                }
                if (tx_s) {
                    for (int i = 0; i < 2 * C; ++i) tx_s[(size_t)o * C * 2 + i] = -1;
                    for (int k = 0; k < nv; ++k) {
                        tx_s[((size_t)o * C + cams[k]) * 2 + 0] = xy[((size_t)cams[k] * MB + pts[k]) * 2 + 0];
                        tx_s[((size_t)o * C + cams[k]) * 2 + 1] = xy[((size_t)cams[k] * MB + pts[k]) * 2 + 1];
                    }
                }
            }
            if (tb->use_world) {                               // helpers.py:96-103
                const double* M = tb->world;
                const double x = -X[0], y = -X[1], z = X[2];
                const double wx = DFMA(M[0], x, DFMA(M[1], y, DFMA(M[2], z, M[3])));
                const double wy = DFMA(M[4], x, DFMA(M[5], y, DFMA(M[6], z, M[7])));
                const double wz = DFMA(M[8], x, DFMA(M[9], y, DFMA(M[10], z, M[11])));
                const double ww = DFMA(M[12], x, DFMA(M[13], y, DFMA(M[14], z, M[15])));
                X[0] = wx / ww; X[1] = wz / ww; X[2] = wy / ww;
            }
            obj_s[3 * o + 0] = X[0]; obj_s[3 * o + 1] = X[1]; obj_s[3 * o + 2] = X[2];
            err_s[o] = e;
        }
        n_out += __popc(bal);
    }
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) flags |= __shfl_xor_sync(FULL_MASK, flags, o);
    if (lane == 0) {
        n_obj[set] = n_out;
        if (set_flags) set_flags[set] = flags;
    }
}

// One warp: the whole matcher for frame-set `set`.
static __device__ __noinline__ void match_triangulate_warp(
    const CameraTables* __restrict__ tb, WarpState ws, const int32_t* xy, const int32_t* nb, int set, int lane,
    int C, int MB, int RMAX, int KC, uint32_t GMAX, double* __restrict__ obj, double* __restrict__ err_out,
    int32_t* __restrict__ n_obj, int32_t* __restrict__ set_flags, int32_t* __restrict__ chosen,
    int32_t* __restrict__ track_xy = nullptr, const int32_t* img_flags = nullptr) {
    const MatchPrep p = match_prepare_warp(tb, ws, xy, nb, lane, C, MB, RMAX, KC, GMAX, img_flags);
    match_eval_range_warp(tb, ws, lane, C, MB, KC, p.nr, 0u, p.total);
    match_emit_warp(tb, ws, set, lane, C, MB, RMAX, KC, p.nr, p.flags, obj, err_out, n_obj, set_flags, chosen, track_xy);
}


// ---------------------------------------------------------------------------------------------
// Frame-sets with thousands of candidate groups, several warps each.
//
// The number of groups of a frame-set is the sum over its roots of the product of the candidate counts per camera: on 8
// cameras x 16 markers the mean is about 700, one frame-set in a hundred has more than 3000, single roots reach tens of
// thousands.  One warp evaluates 32 groups per round, so with one warp per frame-set the kernel lasts as long as its
// heaviest frame-set while most warps idle.  The first kernel therefore finishes only the frame-sets of at most `chunk`
// groups and cuts every other one into items (frame-set, range of `chunk` groups); the second kernel hands the items to
// warps.  A warp prepares the frame-set again (cheap: about two rounds' worth), evaluates its range, and leaves the best
// group of every root the range touches in global memory; the warp that finishes a frame-set's last item folds the items'
// results together in ascending range order (strict "<": the earliest group wins ties, as np.argmin) and emits.
// The result is bit-identical to one warp walking the whole frame-set.
struct MatchItem { uint32_t set, chunk, n_chunks, first; };           // set = ~0u: void (the item list was full)
#define MATCH_PARTIAL_WORDS 6                                          // key, group, X, Y, Z, error
struct MatchSplit {
    unsigned* counters;                // [0] frame-sets claimed, [1] items allocated, [2] items claimed (zeroed before the first kernel)
    MatchItem* items;                  // [item_cap]; nullptr: every frame-set is finished by the warp that claimed it
    unsigned long long* partial;       // [item_cap][RMAX][MATCH_PARTIAL_WORDS]
    int* range;                        // [item_cap][2] first and last root the item's range touches
    unsigned* arrive;                  // [n_sets] finished items of the frame-set; the finisher re-arms it
    uint32_t chunk, item_cap;          // chunk: a multiple of 32
};

// first kernel: persistent warps claim frame-sets from a counter (the work per frame-set varies by orders of magnitude, a
// static assignment leaves the SMs idle behind the heaviest CTAs)
static __device__ __forceinline__ void match_sets_body(
    const CameraTables* __restrict__ tb, const WarpState& ws, int lane, const int32_t* blob_xy, const int32_t* blob_n, int n_sets,
    int C, int MB, int RMAX, int KC, uint32_t GMAX, const MatchSplit& sp, double* __restrict__ obj, double* __restrict__ err_out,
    int32_t* __restrict__ n_obj, int32_t* __restrict__ set_flags, int32_t* __restrict__ chosen, int32_t* __restrict__ track_xy,
    const int32_t* __restrict__ img_flags) {
    while (true) {
        unsigned s = 0;
        if (lane == 0) s = atomicAdd(sp.counters, 1u);
        s = __shfl_sync(FULL_MASK, s, 0);
        if (s >= (unsigned)n_sets) break;
        const int set = (int)s;
        const MatchPrep p = match_prepare_warp(tb, ws, blob_xy + (size_t)set * C * MB * 2, blob_n + (size_t)set * C, lane, C, MB, RMAX, KC, GMAX,
                                               img_flags ? img_flags + (size_t)set * C : nullptr);
        if (sp.items && p.total > sp.chunk) {
            const uint32_t nch = (p.total + sp.chunk - 1) / sp.chunk;
            unsigned first = 0;
            if (lane == 0) first = atomicAdd(sp.counters + 1, nch);
            first = __shfl_sync(FULL_MASK, first, 0);
            const bool fits = first <= sp.item_cap && nch <= sp.item_cap - first;
            for (uint32_t c = lane; c < nch && first + c < sp.item_cap; c += 32) {
                MatchItem it;
                it.set = fits ? (uint32_t)set : ~0u; it.chunk = c; it.n_chunks = nch; it.first = first;
                sp.items[first + c] = it;
            }
            if (fits) { __syncwarp(); continue; }
        }
        match_eval_range_warp(tb, ws, lane, C, MB, KC, p.nr, 0u, p.total);
        match_emit_warp(tb, ws, set, lane, C, MB, RMAX, KC, p.nr, p.flags, obj, err_out, n_obj, set_flags, chosen, track_xy);
        __syncwarp();
    }
}

// second kernel: persistent warps claim items
static __device__ __forceinline__ void match_chunks_body(
    const CameraTables* __restrict__ tb, const WarpState& ws, int lane, const int32_t* blob_xy, const int32_t* blob_n,
    int C, int MB, int RMAX, int KC, uint32_t GMAX, const MatchSplit& sp, double* __restrict__ obj, double* __restrict__ err_out,
    int32_t* __restrict__ n_obj, int32_t* __restrict__ set_flags, int32_t* __restrict__ chosen, int32_t* __restrict__ track_xy,
    const int32_t* __restrict__ img_flags) {
    unsigned n_items = __ldcg(sp.counters + 1);                      // final: the first kernel has finished
    if (n_items > sp.item_cap) n_items = sp.item_cap;
    while (true) {
        unsigned i = 0;
        if (lane == 0) i = atomicAdd(sp.counters + 2, 1u);
        i = __shfl_sync(FULL_MASK, i, 0);
        if (i >= n_items) break;
        const MatchItem it = sp.items[i];
        if (it.set == ~0u) continue;
        const int set = (int)it.set;
        const MatchPrep p = match_prepare_warp(tb, ws, blob_xy + (size_t)set * C * MB * 2, blob_n + (size_t)set * C, lane, C, MB, RMAX, KC, GMAX,
                                               img_flags ? img_flags + (size_t)set * C : nullptr);
        const uint32_t w_lo = it.chunk * sp.chunk;
        const uint32_t w_hi = p.total - w_lo < sp.chunk ? p.total : w_lo + sp.chunk;
        match_eval_range_warp(tb, ws, lane, C, MB, KC, p.nr, w_lo, w_hi);
        // roots of the first and the last group of the range (last r with gprefix[r] <= w)
        int r_lo, r_hi;
        {
            int lo = 0, hi = p.nr;
            while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (ws.gprefix[mid] <= w_lo) lo = mid; else hi = mid; }
            r_lo = lo;
            lo = r_lo; hi = p.nr;
            while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (ws.gprefix[mid] <= w_hi - 1u) lo = mid; else hi = mid; }
            r_hi = lo;
        }
        unsigned long long* mine = sp.partial + (size_t)i * RMAX * MATCH_PARTIAL_WORDS;
        for (int r = r_lo + lane; r <= r_hi; r += 32) {
            unsigned long long* q = mine + (size_t)r * MATCH_PARTIAL_WORDS;
            q[0] = ws.best_key[r];
            q[1] = (unsigned long long)ws.best_g[r];
            q[2] = (unsigned long long)__double_as_longlong(ws.best_xe[4 * r + 0]);
            q[3] = (unsigned long long)__double_as_longlong(ws.best_xe[4 * r + 1]);
            q[4] = (unsigned long long)__double_as_longlong(ws.best_xe[4 * r + 2]);
            q[5] = (unsigned long long)__double_as_longlong(ws.best_xe[4 * r + 3]);
        }
        if (lane == 0) { sp.range[2 * i] = r_lo; sp.range[2 * i + 1] = r_hi; }
        __threadfence();                                             // every lane: its stores before the arrival below
        __syncwarp();
        unsigned before = 0;
        if (lane == 0) before = atomicAdd(sp.arrive + set, 1u);
        before = __shfl_sync(FULL_MASK, before, 0);
        if (before != it.n_chunks - 1u) continue;

        // the frame-set's last item: fold the items' results in ascending range order, emit
        __threadfence();
        if (lane == 0) sp.arrive[set] = 0u;
        for (int r = lane; r < p.nr; r += 32) { ws.best_key[r] = ~0ull; ws.best_g[r] = 0u; }
        __syncwarp();
        for (uint32_t c = 0; c < it.n_chunks; ++c) {
            const size_t j = (size_t)it.first + c;
            const int a = __ldcg(sp.range + 2 * j), b = __ldcg(sp.range + 2 * j + 1);
            const unsigned long long* theirs = sp.partial + j * RMAX * MATCH_PARTIAL_WORDS;
            for (int r = a + lane; r <= b; r += 32) {
                const unsigned long long* q = theirs + (size_t)r * MATCH_PARTIAL_WORDS;
                const unsigned long long key = __ldcg(q);
                if (key < ws.best_key[r]) {
                    ws.best_key[r] = key;
                    ws.best_g[r] = (uint32_t)__ldcg(q + 1);
                    ws.best_xe[4 * r + 0] = __longlong_as_double((long long)__ldcg(q + 2));
                    ws.best_xe[4 * r + 1] = __longlong_as_double((long long)__ldcg(q + 3));
                    ws.best_xe[4 * r + 2] = __longlong_as_double((long long)__ldcg(q + 4));
                    ws.best_xe[4 * r + 3] = __longlong_as_double((long long)__ldcg(q + 5));
                }
            }
            __syncwarp();                                            // the next item may hand a root to another lane
        }
        match_emit_warp(tb, ws, set, lane, C, MB, RMAX, KC, p.nr, p.flags, obj, err_out, n_obj, set_flags, chosen, track_xy);
        __syncwarp();
    }
}

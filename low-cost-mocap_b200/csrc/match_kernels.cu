// S2 + S3 on sm_90a: epipolar correspondence search, DLT triangulation of every candidate
// group, reprojection error, per-root argmin.  One warp per frame-set; frame-sets with more than MOCAP_MATCH_CHUNK
// candidate groups are cut into ranges of groups that a second kernel hands to warps (match_device.cuh, MatchSplit).
//
// Replaces find_point_correspondance_and_object_points (reference
// computer_code/api/helpers.py:339-421) including its inner calls of triangulate_points
// (:330-336 -> :293-327) and calculate_reprojection_errors (:203-241), and, as a separate
// kernel, triangulate_points / calculate_reprojection_errors on explicit correspondences.
//
// The reference builds "roots" (camera-0 blobs, later unmatched blobs of other cameras) and
// for every further camera branches each root's candidate groups over the blobs closer than
// 5 px to the root's epipolar line, sorted by distance.  Groups of one root are therefore the
// Cartesian product of per-camera candidate lists, and the reference's group order is the
// mixed-radix number with the EARLIEST camera as least significant digit (helpers.py:394-400
// puts the newest camera outermost).  This kernel stores only the per-camera candidate lists
// and enumerates group indices; nothing is materialised.
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "geom.cuh"
#include "match_device.cuh"

__global__ void __launch_bounds__(128)
k_match_triangulate(const CameraTables* __restrict__ tb, const int32_t* blob_xy, const int32_t* blob_n,
                    const uint32_t* __restrict__ set_list, uint32_t* set_count, MatchSplit sp,
                    int n_sets, int C, int MB, int RMAX, int KC,
                    uint32_t GMAX, double* __restrict__ obj, double* __restrict__ err_out,
                    int32_t* __restrict__ n_obj, int32_t* __restrict__ set_flags, int32_t* __restrict__ chosen,
                    int32_t* __restrict__ track_xy, const int32_t* __restrict__ img_flags) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warps = blockDim.x >> 5;
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    WarpState ws = carve_warp_state(smem_raw + warp_state_bytes(RMAX, C, KC, MB) * wid, RMAX, C, KC, MB);
    if (set_list) {                                   // persistent walk over a worklist of frame-sets
        const unsigned n_work = *set_count;
        for (unsigned w = blockIdx.x * warps + wid; w < n_work; w += gridDim.x * warps) {
            const int set = (int)set_list[w];
            match_triangulate_warp(tb, ws, blob_xy + (size_t)set * C * MB * 2, blob_n + (size_t)set * C, set, lane,
                                   C, MB, RMAX, KC, GMAX, obj, err_out, n_obj, set_flags, chosen, track_xy,
                                   img_flags ? img_flags + (size_t)set * C : nullptr);
            __syncwarp();
        }
        __syncthreads();
        if (threadIdx.x == 0) {                           // the last CTA to finish re-arms the worklist
            __threadfence();
            if (atomicAdd(set_count + 1, 1u) == gridDim.x - 1) { set_count[0] = 0; set_count[1] = 0; }
        }
        return;
    }
    // persistent warps claim frame-sets from sp.counters[0]; frame-sets of more than sp.chunk candidate groups become
    // items for k_match_chunks (match_device.cuh)
    match_sets_body(tb, ws, lane, blob_xy, blob_n, n_sets, C, MB, RMAX, KC, GMAX, sp, obj, err_out, n_obj, set_flags, chosen, track_xy, img_flags);
}

// the items k_match_triangulate left: ranges of the candidate groups of the heavy frame-sets, one warp each
__global__ void __launch_bounds__(128)
k_match_chunks(const CameraTables* __restrict__ tb, const int32_t* blob_xy, const int32_t* blob_n, MatchSplit sp,
               int C, int MB, int RMAX, int KC, uint32_t GMAX, double* __restrict__ obj, double* __restrict__ err_out,
               int32_t* __restrict__ n_obj, int32_t* __restrict__ set_flags, int32_t* __restrict__ chosen,
               int32_t* __restrict__ track_xy, const int32_t* __restrict__ img_flags) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    WarpState ws = carve_warp_state(smem_raw + warp_state_bytes(RMAX, C, KC, MB) * wid, RMAX, C, KC, MB);
    match_chunks_body(tb, ws, lane, blob_xy, blob_n, C, MB, RMAX, KC, GMAX, sp, obj, err_out, n_obj, set_flags, chosen, track_xy, img_flags);
}

// ---------------------------------------------------------------------------------------------
// explicit correspondences: triangulate_points / calculate_reprojection_errors, one thread per point
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
k_triangulate_points(const CameraTables* __restrict__ tb, const double* __restrict__ obs,
                     const uint8_t* __restrict__ mask, int n_points, int C,
                     const double* __restrict__ X_in, double* __restrict__ X_out,
                     double* __restrict__ err_out, uint8_t* __restrict__ valid) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_points) return;
    const double* o = obs + (size_t)f * C * 2;
    const uint8_t* m = mask + (size_t)f * C;
    int nv = 0;
    for (int c = 0; c < C; ++c) nv += m[c] ? 1 : 0;
    if (nv <= 1) {                                             // helpers.py:300-301, 222-223
        if (valid) valid[f] = 0;
        if (X_out) { X_out[3 * f] = X_out[3 * f + 1] = X_out[3 * f + 2] = nan(""); }
        if (err_out) err_out[f] = nan("");
        return;
    }
    double X[3];
    if (X_in) { X[0] = X_in[3 * f]; X[1] = X_in[3 * f + 1]; X[2] = X_in[3 * f + 2]; }
    else {
        Sym4 B;
        sym4_zero(B);
        int k = 0;
        for (int c = 0; c < C; ++c)
            if (m[c]) { dlt_add_view(B, tb->Pkc[k][c], o[2 * c], o[2 * c + 1]); ++k; }
        dlt_solve(B, X);
    }
    if (X_out) { X_out[3 * f] = X[0]; X_out[3 * f + 1] = X[1]; X_out[3 * f + 2] = X[2]; }
    if (valid) valid[f] = 1;
    if (err_out) {
        double sq[2 * MOCAP_MAX_CAM];
        int k = 0;
        for (int c = 0; c < C; ++c)
            if (m[c]) {
                float u, v;
                project_like_cv(tb->R[c], tb->t[c], tb->fx[k], tb->fy[k], tb->cx[k], tb->cy[k], X, u, v);
                const double dx = DSUB(o[2 * c], (double)u), dy = DSUB(o[2 * c + 1], (double)v);
                sq[2 * k] = DMUL(dx, dx); sq[2 * k + 1] = DMUL(dy, dy);
                ++k;
            }
        // explicit correspondences arrive as object arrays in the reference's callers
        // (index.py:254,274; helpers.py:271): left fold
        err_out[f] = mean_like_numpy(sq, 2 * nv, false);
    }
}

// scratch of the chunked matcher, sized for the batch: items, their partial results, arrival counters
static int ensure_match_split(mocap_ctx* ctx, int n_sets) {
    // room for four items per frame-set, the partial results bounded by 512 MB; frame-sets that find the list full are
    // finished by the warp that claimed them
    long long want = (long long)n_sets * 4 > 4096 ? (long long)n_sets * 4 : 4096;
    const long long per_item = (long long)ctx->cfg.max_roots * MATCH_PARTIAL_WORDS * (long long)sizeof(unsigned long long);
    if (want * per_item > (512ll << 20)) want = (512ll << 20) / per_item;
    const int want_items = (int)want;
    if (n_sets <= ctx->match_cap_sets && want_items <= ctx->match_item_cap) return MOCAP_OK;
    const size_t items = (size_t)want_items;
    const int st = grow_carved(ctx, ctx->match_split, Drain::stream, [&](Layout& L) {
        ctx->d_match_arrive = L.take<unsigned>(n_sets);      // the finishers keep it zero
        L.zero_so_far();
        ctx->d_match_items = L.take<MatchItem>(items); ctx->d_match_range = L.take<int>(items * 2);
        ctx->d_match_partial = L.take<unsigned long long>(items * ctx->cfg.max_roots * MATCH_PARTIAL_WORDS);
    });
    ctx->match_cap_sets = st ? 0 : n_sets; ctx->match_item_cap = st ? 0 : want_items;
    return st;
}

int launch_match(mocap_ctx* ctx, const int32_t* blob_xy, const int32_t* blob_n, int n_sets,
                 double* obj, double* err, int32_t* n_obj, int32_t* set_flags, int32_t* chosen) {
    if (n_sets <= 0) return MOCAP_OK;
    const mocap_config& c = ctx->cfg;
    const int warps = 4;
    const size_t smem = match_smem_bytes(c, warps);
    const int full = ctx->num_sms * ctx->match_ctas_per_sm;
    int grid = (n_sets + warps - 1) / warps;
    if (grid > full) grid = full;
    MatchSplit sp;
    memset(&sp, 0, sizeof(sp));
    sp.counters = ctx->match_counter.as<unsigned>();
    if (ctx->match_chunk > 0) {
        const int st = ensure_match_split(ctx, n_sets);
        if (st) return st;
        sp.items = static_cast<MatchItem*>(ctx->d_match_items);
        sp.partial = ctx->d_match_partial; sp.range = ctx->d_match_range; sp.arrive = ctx->d_match_arrive;
        sp.chunk = (uint32_t)ctx->match_chunk; sp.item_cap = (uint32_t)ctx->match_item_cap;
    }
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->match_counter.get(), 0, 4 * sizeof(unsigned), ctx->stream));
    k_match_triangulate<<<grid, warps * 32, smem, ctx->stream>>>(ctx->d_tables, blob_xy, blob_n, nullptr, nullptr, sp, n_sets, c.n_cam,
                                                                 c.max_blobs, c.max_roots, c.max_cands,
                                                                 (uint32_t)c.max_groups, obj, err, n_obj, set_flags, chosen, ctx->track_xy_cur, ctx->img_flags_cur);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    if (sp.items) {
        // how many items there are is known on the device only: a full persistent grid, warps without an item leave at once
        k_match_chunks<<<full, warps * 32, smem, ctx->stream>>>(ctx->d_tables, blob_xy, blob_n, sp, c.n_cam, c.max_blobs, c.max_roots, c.max_cands,
                                                                (uint32_t)c.max_groups, obj, err, n_obj, set_flags, chosen, ctx->track_xy_cur, ctx->img_flags_cur);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    return MOCAP_OK;
}

int launch_match_list(mocap_ctx* ctx, const int32_t* blob_xy, const int32_t* blob_n, const uint32_t* set_list, uint32_t* set_count,
                      int n_sets_max, double* obj, double* err, int32_t* n_obj, int32_t* set_flags) {
    const mocap_config& c = ctx->cfg;
    const int warps = 4;
    const size_t smem = match_smem_bytes(c, warps);
    int grid = (n_sets_max + warps - 1) / warps;
    if (grid > ctx->num_sms) grid = ctx->num_sms;
    MatchSplit none;
    memset(&none, 0, sizeof(none));
    k_match_triangulate<<<grid, warps * 32, smem, ctx->stream>>>(ctx->d_tables, blob_xy, blob_n, set_list, set_count, none, n_sets_max, c.n_cam,
                                                                 c.max_blobs, c.max_roots, c.max_cands, (uint32_t)c.max_groups,
                                                                 obj, err, n_obj, set_flags, nullptr, ctx->track_xy_cur, ctx->d_img_flags);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    return MOCAP_OK;
}

int launch_triangulate(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                       const double* X_in, double* X, double* err, uint8_t* valid) {
    if (n_points <= 0) return MOCAP_OK;
    const int threads = 128;
    k_triangulate_points<<<(n_points + threads - 1) / threads, threads, 0, ctx->stream>>>(
        ctx->d_tables, obs, mask, n_points, ctx->cfg.n_cam, X_in, X, err, valid);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    return MOCAP_OK;
}

int match_kernels_init(mocap_ctx* ctx) {
    const size_t smem = match_smem_bytes(ctx->cfg, 4);
    if (smem > 200 * 1024) return mocap_fail(ctx, MOCAP_EINVAL, "matcher state needs %zu bytes of shared memory per CTA; lower max_roots/max_cands", smem);
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_match_triangulate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_match_triangulate, 128, smem));
    ctx->match_ctas_per_sm = per_sm > 0 ? per_sm : 1;
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_match_chunks, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int st = ctx->match_counter.grow(ctx, 4 * sizeof(unsigned), Drain::none);
    if (st) return st;
    // candidate groups per item of the chunked matcher (match_device.cuh); MOCAP_MATCH_CHUNK=0: one warp per frame-set throughout
    const char* ch = getenv("MOCAP_MATCH_CHUNK");
    int chunk = ch && ch[0] ? atoi(ch) : MOCAP_MATCH_CHUNK;
    if (chunk < 0) chunk = 0;
    ctx->match_chunk = (chunk + 31) / 32 * 32;
    return MOCAP_OK;
}

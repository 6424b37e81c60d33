// S1 + S2 + S3 in ONE persistent kernel (1-channel frames): the whole per-frame body of
// Cameras._camera_read (reference computer_code/api/helpers.py:84-103) in a single pass over HBM.
//
// Work is claimed dynamically, one "unit" (a contiguous slice of an image) per warp at a time:
//   stream    the warp thresholds its slice with 8 independent 128-bit streaming loads per lane and
//             appends the rare non-empty 16-pixel segments to the image's list (as k_threshold_segments)
//   last one  the warp that completes the LAST slice of an image (atomic counter, release/acquire by
//   reduces   __threadfence) reduces that image's segment list to blobs right away (warp-level
//             blob_reduce), while every other warp keeps streaming
//   last one  the warp that completes the LAST image of a frame-set runs the matcher + DLT +
//   matches   reprojection error for that frame-set (match_triangulate_warp)
// Nobody ever waits: there are no inter-warp spin loops, only "last arriver does the follow-up work",
// so the sparse stages hide under the HBM stream of the other warps of the SM instead of running as
// separate kernels after it.  Images / frame-sets beyond the warp-level capacities are put on
// worklists and finished by the full-size kernels (k_blob_reduce, k_match_triangulate) afterwards.
#include "fused_device.cuh"

size_t fused_slab_bytes(const mocap_config& c) {
    size_t a = sizeof(WarpSlab), b = warp_state_bytes(c.max_roots, c.n_cam, c.max_cands, c.max_blobs);
    size_t m = a > b ? a : b;
    return (m + 15) & ~(size_t)15;
}

int launch_pipeline_fused(mocap_ctx* ctx, const uint8_t* frames, int n_sets, int channels, int threshold, const SetOut& out) {
    if (n_sets <= 0) return MOCAP_OK;
    const mocap_config& c = ctx->cfg;
    FusedParams P;
    memset(&P, 0, sizeof(P));
    P.frames = reinterpret_cast<const uint4*>(frames);
    P.n_sets = n_sets; P.C = c.n_cam; P.W = c.width; P.H = c.height;
    P.seg_per_image = c.width * c.height / MOCAP_SEG_PX;
    P.u4_per_image = P.seg_per_image * (channels == 3 ? 3 : 1);
    P.threshold = threshold;
    const int iters_total = (P.u4_per_image + FUSED_SEGS_PER_ITER - 1) / FUSED_SEGS_PER_ITER;
    P.units_per_image = (iters_total + 15) / 16;             // ~16 iterations (64 KB) per unit
    P.iters_per_unit = (iters_total + P.units_per_image - 1) / P.units_per_image;
    P.total_units = (long long)n_sets * c.n_cam * P.units_per_image;
    P.tc = thresh_const(threshold);
    P.E = c.max_segments;
    P.seg_count = ctx->d_seg_count; P.seg_list = ctx->d_seg_list;
    P.img_done = ctx->d_img_done; P.set_done = ctx->d_set_done; P.set_defer = ctx->d_set_done + ctx->cap_images;
    P.unit_counter = ctx->d_unit_counter;
    P.blob_xy = ctx->d_blob_xy; P.blob_n = ctx->d_blob_n; P.img_flags = ctx->d_img_flags;
    P.img_worklist = ctx->d_worklist; P.img_work_count = ctx->d_work_count;
    P.set_worklist = ctx->d_set_worklist; P.set_work_count = ctx->d_work_count + 2;
    P.tb = ctx->d_tables;
    P.MB = c.max_blobs; P.RMAX = c.max_roots; P.KC = c.max_cands; P.GMAX = (uint32_t)c.max_groups;
    P.obj = out.obj; P.err = out.err; P.n_obj = out.n; P.set_flags = out.flags; P.track_xy = out.track_xy;
    P.slab_bytes = fused_slab_bytes(c);
    const size_t smem = P.slab_bytes * FUSED_WARPS;
    const bool wide = moments_wide(c);

    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_unit_counter, 0, sizeof(unsigned long long), ctx->stream));
    int st = timing_begin(ctx);
    if (st) return st;
    const int grid = ctx->num_sms * ctx->fused_ctas_per_sm;
    if (channels == 3) {                                     // H x W x 3 interleaved: the layout _find_dot receives
        if (wide) {
            if (P.tc.use_and) k_pipeline_fused<true, true, true><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
            else k_pipeline_fused<true, false, true><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
        } else {
            if (P.tc.use_and) k_pipeline_fused<false, true, true><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
            else k_pipeline_fused<false, false, true><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
        }
    } else if (wide) {
        if (P.tc.use_and) k_pipeline_fused<true, true><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
        else k_pipeline_fused<true, false><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
    } else {
        if (P.tc.use_and) k_pipeline_fused<false, true><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
        else k_pipeline_fused<false, false><<<grid, FUSED_WARPS * 32, smem, ctx->stream>>>(P);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    if ((st = timing_end(ctx)) != MOCAP_OK) return st;
    ctx->launches += 1;
    // slow path for whatever exceeded the warp-level capacities (normally nothing: both kernels
    // read an empty worklist and exit)
    if ((st = launch_blob_fallback(ctx, ctx->d_blob_xy, ctx->d_blob_n, nullptr, ctx->d_img_flags, n_sets * ctx->cfg.n_cam)) != MOCAP_OK)
        return st;
    return launch_match_list(ctx, ctx->d_blob_xy, ctx->d_blob_n, ctx->d_set_worklist, ctx->d_work_count + 2, n_sets, out, ctx->d_img_flags);
}

int fused_kernel_init(mocap_ctx* ctx) {
    const size_t smem = fused_slab_bytes(ctx->cfg) * FUSED_WARPS;
    if (smem > 110 * 1024) { ctx->use_fused = 0; return MOCAP_OK; }    // matcher state too large: three-kernel pipeline
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_pipeline_fused<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;      // persistent grid = what is actually co-resident
    CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pipeline_fused<false, false>, FUSED_WARPS * 32, smem));
    if (per_sm < 1) { ctx->use_fused = 0; return MOCAP_OK; }
    ctx->fused_ctas_per_sm = per_sm;
    return MOCAP_OK;
}

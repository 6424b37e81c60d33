// The detection overlay _find_dot draws into every captured frame (reference computer_code/api/helpers.py:148,156-157):
// contours, then the centre labels and plus marks, in place on the frames (drawing code: overlay.cuh).
//
//   k_overlay_gray      cv2's RGB2GRAY of the undrawn frames, for the batched entry (the live loop passes the grey
//                       plane the preprocessing kernel already made for S1);
//   k_overlay_contours  one thread per run of 4 pixels: the contour colour where ov_border holds -- the only stage that
//                       touches every pixel (1 byte read per pixel, a 3-byte write per contour pixel);
//   k_overlay_marks     one warp per image: the lanes take (blob, label character) items and the pluses.  Items of one
//                       image overlap only in pixels they all paint the mark colour, so their order does not matter.
// In triangulate mode, after those, the epipolar lines find_point_correspondance_and_object_points draws into camera
// i >= 1 for every root that exists before camera i (helpers.py:359-365, drawlines :497-504), in the reference's order
// (camera by camera, roots in creation order, a later line over an earlier one):
//   k_overlay_epilines  the matcher's own prepare step (match_prepare_warp) rebuilds a frame-set's roots, epiline_f32
//                       their float32 lines.  Pass 0, one warp per frame-set, counts its lines; pass 1, one warp per
//                       (frame-set, camera i >= 1), draws camera i's, the lanes splitting each line's pixels with a
//                       __syncwarp between lines, line n of the session in palette[n % L]: n = the context's counter +
//                       the lines of the group's earlier frame-sets + those of the frame-set's earlier cameras;
//   k_overlay_epiadvance  moves the counter on by the group's lines.
#include <vector>
#include "common.cuh"
#include "match_device.cuh"
#include "overlay.cuh"

static int overlay_frames(mocap_ctx* ctx, uint8_t* frames, int n_images, const int32_t* blob_xy, const int32_t* blob_n);

#define OV_RUN 4                        // pixels per thread of k_overlay_contours (W is a multiple of 16)
#define OV_ITEMS (OV_MAX_LABEL + 1)     // per blob: one item per label character, one for the plus

__global__ void __launch_bounds__(256)
k_overlay_gray(const uint8_t* __restrict__ frames, size_t n_px, uint8_t* __restrict__ gray) {
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n_px) gray[p] = (uint8_t)ov_gray(frames + p * 3);
}

__global__ void __launch_bounds__(256)
k_overlay_contours(const uint8_t* __restrict__ gray, uint8_t* __restrict__ frames, int n_images, int W, int H) {
    const int runs = W / OV_RUN;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)n_images * H * runs) return;
    const int x0 = (int)(t % runs) * OV_RUN;
    const size_t row = t / runs;                           // image * H + y
    const int y = (int)(row % H);
    const size_t img = row / H;
    const uint8_t* g = gray + img * W * H;
    uint8_t* f = frames + img * W * H * 3;
#pragma unroll
    for (int k = 0; k < OV_RUN; ++k)
        if (ov_border(g, W, H, x0 + k, y)) ov_put(f, W, H, x0 + k, y, OV_CONTOUR_0, OV_CONTOUR_1, OV_CONTOUR_2);
}

__global__ void __launch_bounds__(128)
k_overlay_marks(const int32_t* __restrict__ blob_xy, const int32_t* __restrict__ blob_n, int MB, uint8_t* __restrict__ frames,
                int n_images, int W, int H) {
    const int img = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (img >= n_images) return;
    const int n = blob_n[img] < MB ? blob_n[img] : MB;
    const int32_t* xy = blob_xy + (size_t)img * MB * 2;
    uint8_t* f = frames + (size_t)img * W * H * 3;
    for (int it = lane; it < n * OV_ITEMS; it += 32) {
        const int b = it / OV_ITEMS, k = it % OV_ITEMS;
        if (k == OV_MAX_LABEL) ov_plus(f, W, H, xy[2 * b], xy[2 * b + 1]);
        else ov_label_char(f, W, H, xy[2 * b], xy[2 * b + 1], k);
    }
}

__global__ void __launch_bounds__(32)
k_overlay_epilines(const CameraTables* __restrict__ tb, const int32_t* __restrict__ blob_xy, const int32_t* __restrict__ blob_n,
                   int n_sets, int C, int MB, int RMAX, int KC, uint32_t GMAX, uint8_t* __restrict__ frames, int W, int H,
                   const uint8_t* __restrict__ palette, int L, const unsigned long long* __restrict__ counter,
                   uint32_t* __restrict__ counts, int pass) {
    extern __shared__ __align__(16) unsigned char ov_smem[];
    const int set = blockIdx.x, lane = threadIdx.x, only = pass ? (int)blockIdx.y + 1 : 0;
    if (set >= n_sets) return;
    const WarpState ws = carve_warp_state(ov_smem, RMAX, C, KC, MB);
    const MatchPrep prep = match_prepare_warp(tb, ws, blob_xy + (size_t)set * C * MB * 2, blob_n + (size_t)set * C, lane,
                                              C, MB, RMAX, KC, GMAX, nullptr);
    // roots are made camera by camera: the roots that exist before camera i are the first before[i]
    int before = 0;
    uint32_t total = 0;
    unsigned long long n = 0;
    if (pass == 1) {
        for (int s = lane; s < set; s += 32) n += counts[s];
#pragma unroll 1
        for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(FULL_MASK, n, o);
        n += *counter;
    }
    for (int i = 1; i < C; ++i) {
        while (before < prep.nr && ws.rcam[before] < i) ++before;
        total += (uint32_t)before;
        if (i != only) { n += (unsigned long long)before; continue; }
        uint8_t* f = frames + ((size_t)set * C + i) * W * H * 3;
        for (int j = 0; j < before; ++j, ++n) {
            const int rc = ws.rcam[j];
            double a, b, c;
            epiline_f32(tb->F[rc][i], (double)ws.xy_s[(rc * MB + ws.rpt[j]) * 2], (double)ws.xy_s[(rc * MB + ws.rpt[j]) * 2 + 1], a, b, c);
            int64_t y0, y1;
            if (ov_epiline_ends((float)a, (float)b, (float)c, W, &y0, &y1)) {
                const uint8_t* col = palette + (size_t)(n % (unsigned long long)L) * 3;
                ov_line(f, W, H, 0, y0, W, y1, col[0], col[1], col[2], lane, 32);
            }
            __syncwarp();
        }
    }
    if (pass == 0 && lane == 0) counts[set] = total;
}

__global__ void k_overlay_epiadvance(const uint32_t* __restrict__ counts, int n_sets, unsigned long long* __restrict__ counter) {
    unsigned long long n = 0;
    for (int s = threadIdx.x; s < n_sets; s += 32) n += counts[s];
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(FULL_MASK, n, o);
    if (threadIdx.x == 0) *counter += n;
}

// the epipolar lines of n_sets frame-sets of frames [C][W][H][3] with their S1 blob lists
int launch_epilines(mocap_ctx* ctx, uint8_t* frames, int n_sets, const int32_t* blob_xy, const int32_t* blob_n) {
    const mocap_config& g = ctx->cfg;
    if (n_sets <= 0 || g.n_cam < 2) return MOCAP_OK;
    if (n_sets > ctx->line_counts_cap) {
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        cudaFree(ctx->d_line_counts);
        ctx->d_line_counts = nullptr; ctx->line_counts_cap = 0;
        CUDA_TRY(ctx, cudaMalloc(&ctx->d_line_counts, (size_t)n_sets * sizeof(uint32_t)));
        ctx->line_counts_cap = n_sets;
    }
    const size_t smem = warp_state_bytes(g.max_roots, g.n_cam, g.max_cands, g.max_blobs);
    for (int pass = 0; pass < 2; ++pass) {
        k_overlay_epilines<<<dim3(n_sets, pass ? g.n_cam - 1 : 1), 32, smem, ctx->stream>>>(ctx->d_tables, blob_xy, blob_n, n_sets, g.n_cam, g.max_blobs, g.max_roots,
                                                              g.max_cands, (uint32_t)g.max_groups, frames, g.width, g.height, ctx->d_palette,
                                                              ctx->palette_len, ctx->d_line_counter, ctx->d_line_counts, pass);
        CUDA_TRY(ctx, cudaGetLastError());
    }
    k_overlay_epiadvance<<<1, 32, 0, ctx->stream>>>(ctx->d_line_counts, n_sets, ctx->d_line_counter);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 3;
    return MOCAP_OK;
}

// the overlay of n_images frames [W][H][3] (the context's size) from their grey planes and S1 blob lists
int launch_overlay(mocap_ctx* ctx, const uint8_t* gray, uint8_t* frames, int n_images, const int32_t* blob_xy, const int32_t* blob_n) {
    if (n_images <= 0) return MOCAP_OK;
    const int W = ctx->cfg.width, H = ctx->cfg.height;
    const size_t threads = (size_t)n_images * H * (W / OV_RUN);
    k_overlay_contours<<<(unsigned)((threads + 255) / 256), 256, 0, ctx->stream>>>(gray, frames, n_images, W, H);
    CUDA_TRY(ctx, cudaGetLastError());
    k_overlay_marks<<<(n_images + 3) / 4, 128, 0, ctx->stream>>>(blob_xy, blob_n, ctx->cfg.max_blobs, frames, n_images, W, H);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 2;
    return MOCAP_OK;
}

extern "C" {

int mocap_set_overlay(mocap_ctx* ctx, int on, uint32_t seed, int palette_len) {
    if (!ctx) return MOCAP_EINVAL;
    if (palette_len < 1 || palette_len > MOCAP_OVERLAY_MAX_PALETTE)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_set_overlay: palette_len %d is not in 1..%d", palette_len, MOCAP_OVERLAY_MAX_PALETTE);
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    std::vector<uint8_t> pal((size_t)palette_len * 3);
    ov_palette(seed, palette_len, pal.data());
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (!ctx->d_palette) CUDA_TRY(ctx, cudaMalloc(&ctx->d_palette, (size_t)MOCAP_OVERLAY_MAX_PALETTE * 3));
    if (!ctx->d_line_counter) CUDA_TRY(ctx, cudaMalloc(&ctx->d_line_counter, sizeof(unsigned long long)));
    const mocap_config& g = ctx->cfg;
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_overlay_epilines, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)warp_state_bytes(g.max_roots, g.n_cam, g.max_cands, g.max_blobs)));
    CUDA_TRY(ctx, cudaMemcpy(ctx->d_palette, pal.data(), pal.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(ctx, cudaMemset(ctx->d_line_counter, 0, sizeof(unsigned long long)));
    ctx->palette_len = palette_len;
    ctx->overlay_on = on ? 1 : 0;
    return MOCAP_OK;
}

int mocap_overlay_dev(mocap_ctx* ctx, uint8_t* frames, int n_sets, const int32_t* blob_xy, const int32_t* blob_n, int mode) {
    if (!ctx) return MOCAP_EINVAL;
    if (!frames || !blob_xy || !blob_n || n_sets < 0 || mode < 1 || (mode & ~(MOCAP_LIVE_CAPTURE | MOCAP_LIVE_TRIANGULATE)))
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_overlay_dev: bad argument (mode: CAPTURE and/or TRIANGULATE)");
    if ((mode & MOCAP_LIVE_TRIANGULATE) && !ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    if ((mode & MOCAP_LIVE_TRIANGULATE) && !ctx->d_palette)
        return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_overlay has not been called (the epipolar lines need its palette)");
    if (n_sets == 0) return MOCAP_OK;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    int st = MOCAP_OK;
    if ((mode & MOCAP_LIVE_CAPTURE) && (st = overlay_frames(ctx, frames, n_sets * ctx->cfg.n_cam, blob_xy, blob_n)) != MOCAP_OK) return st;
    if (mode & MOCAP_LIVE_TRIANGULATE) return launch_epilines(ctx, frames, n_sets, blob_xy, blob_n);
    return MOCAP_OK;
}

}  // extern "C"

// contours and marks of n_images undrawn frames: the grey plane first, in groups that fit the scratch
static int overlay_frames(mocap_ctx* ctx, uint8_t* frames, int n_images, const int32_t* blob_xy, const int32_t* blob_n) {
    const size_t plane = (size_t)ctx->cfg.width * ctx->cfg.height;
    const int group = (int)((64ull << 20) / plane > 0 ? (64ull << 20) / plane : 1);     // images per grey scratch fill
    int st = ensure_scratch(ctx, (size_t)(n_images < group ? n_images : group) * plane);
    if (st) return st;
    uint8_t* gray = static_cast<uint8_t*>(ctx->d_scratch);
    for (int i0 = 0; i0 < n_images; i0 += group) {
        const int n = n_images - i0 < group ? n_images - i0 : group;
        uint8_t* f = frames + (size_t)i0 * plane * 3;
        const size_t px = (size_t)n * plane;
        k_overlay_gray<<<(unsigned)((px + 255) / 256), 256, 0, ctx->stream>>>(f, px, gray);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        if ((st = launch_overlay(ctx, gray, f, n, blob_xy + (size_t)i0 * ctx->cfg.max_blobs * 2, blob_n + i0)) != MOCAP_OK) return st;
    }
    return MOCAP_OK;
}

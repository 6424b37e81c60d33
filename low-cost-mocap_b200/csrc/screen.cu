// Per-view screening of explicit correspondences between bundle-adjustment rounds (rule: screen.cuh).
//
// k_screen_observations: one warp per track.  Each CTA first builds the C x C projection matrices K_k [R_c | t_c] of
// the CURRENT poses (device R, t -- the buffers mocap_bundle_adjust_dev updates in place; the context's camera tables
// hold the poses of the last mocap_set_cameras and are read for the intrinsics only) in shared memory.  Then, per
// track, the lanes own view pairs (<= 120 at 16 cameras: <= 4 rounds), each one 2-view DLT and <= 16 projections; the
// winner is the warp maximum of a packed (support, ~pair) key.  The refit and the final check are computed by every
// lane (the same DLT in ascending camera order, so the same bits as the host build) and split over the lanes by view
// for the projections.  The number of rows is read from device memory, so it can come from
// mocap_tracks_to_observations_dev without a host round trip.  No synchronisation.
#include <math.h>
#include "common.cuh"
#include "screen.cuh"

static_assert(SCREEN_MAX_CAM == MOCAP_MAX_CAM, "screen.cuh sizes its tables for MOCAP_MAX_CAM cameras");

#define SCREEN_WARPS 8

__global__ void __launch_bounds__(SCREEN_WARPS * 32)
k_screen_observations(const CameraTables* __restrict__ tb, const double* __restrict__ obs, const uint8_t* __restrict__ mask_in,
                      int n_max, const int32_t* __restrict__ n_dev, const double* __restrict__ R, const double* __restrict__ t,
                      int C, double thr2, uint8_t* __restrict__ mask_out, int32_t* __restrict__ stats) {
    __shared__ ScreenCams cams;
    for (int e = threadIdx.x; e < C * C; e += blockDim.x) {
        const int k = e / C, c = e - k * C;
        screen_set_P(cams, k, c, tb->Kmat[k], R + 9 * c, t + 3 * c);
    }
    for (int c = threadIdx.x; c < C; c += blockDim.x) screen_set_cam(cams, c, R + 9 * c, t + 3 * c, tb->fx[c], tb->fy[c], tb->cx[c], tb->cy[c]);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int n = n_dev ? max(0, min(*n_dev, n_max)) : n_max;
    int v_in = 0, v_kept = 0, emptied = 0;
    for (int f = blockIdx.x * SCREEN_WARPS + (threadIdx.x >> 5); f < n; f += gridDim.x * SCREEN_WARPS) {
        const double* o = obs + (size_t)f * C * 2;
        const unsigned S = __ballot_sync(0xffffffffu, lane < C && mask_in[(size_t)f * C + lane] != 0);
        const int nv = __popc(S);
        unsigned out = S;
        if (nv >= 2) {
            unsigned my_key = 0u, my_sup = 0u;
            for (int p = lane; p < nv * (nv - 1) / 2; p += 32) {
                const unsigned sup = screen_support(cams, o, C, screen_pair(S, p), S, thr2);
                const unsigned key = screen_key(__popc(sup), p);
                if (key > my_key) { my_key = key; my_sup = sup; }
            }
            unsigned best = my_key;
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, off));
            const int src = __ffs(__ballot_sync(0xffffffffu, my_key == best)) - 1;
            const unsigned W = __shfl_sync(0xffffffffu, my_sup, src);
            out = screen_refit(S, W, [&](unsigned T, unsigned Q) {
                double X[3];
                screen_point(cams, o, T, C, X);
                const bool ok = lane < C && ((Q >> lane) & 1u) && screen_err2(cams, o, T, lane, X) <= thr2;
                return __ballot_sync(0xffffffffu, ok);
            });
        }
        if (lane < C) mask_out[(size_t)f * C + lane] = (uint8_t)((out >> lane) & 1u);
        v_in += nv; v_kept += __popc(out); emptied += (nv >= 2 && out == 0u) ? 1 : 0;
    }
    if (stats && lane == 0 && v_in) {
        atomicAdd(stats + 0, v_in);
        atomicAdd(stats + 1, v_kept);
        atomicAdd(stats + 2, v_in - v_kept);
        atomicAdd(stats + 3, emptied);
    }
}

// arguments of both entry points; everything is refused before anything is enqueued
static int screen_check(mocap_ctx* ctx, const double* obs, const uint8_t* mask_in, int n_points_max, const double* R, const double* t,
                        double threshold_px, const uint8_t* mask_out, const char* who) {
    if (!obs || !mask_in || !R || !t || !mask_out || n_points_max <= 0)
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: bad argument", who);
    if (mask_out == mask_in) return mocap_fail(ctx, MOCAP_EINVAL, "%s: mask_out must not be mask_in (screening always starts from the caller's mask)", who);
    if (!(threshold_px > 0.0) || !isfinite(threshold_px))
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: threshold_px must be positive and finite (got %g)", who, threshold_px);
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    return MOCAP_OK;
}

static int screen_launch(mocap_ctx* ctx, const double* obs, const uint8_t* mask_in, int n_points_max, const int32_t* n_points,
                         const double* R, const double* t, double threshold_px, uint8_t* mask_out, int32_t* stats) {
    cudaStream_t s = ctx->stream;
    if (stats) CUDA_TRY(ctx, cudaMemsetAsync(stats, 0, 4 * sizeof(int32_t), s));
    const int blocks = (n_points_max + SCREEN_WARPS - 1) / SCREEN_WARPS;
    const int grid = blocks < 4 * ctx->num_sms ? blocks : 4 * ctx->num_sms;
    k_screen_observations<<<grid, SCREEN_WARPS * 32, 0, s>>>(ctx->d_tables, obs, mask_in, n_points_max, n_points, R, t, ctx->cfg.n_cam,
                                                              threshold_px * threshold_px, mask_out, stats);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    return MOCAP_OK;
}

extern "C" {

int mocap_screen_observations_dev(mocap_ctx* ctx, const double* obs, const uint8_t* mask_in, int n_points_max, const int32_t* n_points,
                                  const double* R, const double* t, double threshold_px, uint8_t* mask_out, int32_t* stats) {
    if (!ctx) return MOCAP_EINVAL;
    int st = screen_check(ctx, obs, mask_in, n_points_max, R, t, threshold_px, mask_out, "mocap_screen_observations_dev");
    if (st) return st;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return screen_launch(ctx, obs, mask_in, n_points_max, n_points, R, t, threshold_px, mask_out, stats);
}

int mocap_screen_observations_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask_in, int n_points_max, const int32_t* n_points,
                                   const double* R, const double* t, double threshold_px, uint8_t* mask_out, int32_t* stats) {
    if (!ctx) return MOCAP_EINVAL;
    int st = screen_check(ctx, obs, mask_in, n_points_max, R, t, threshold_px, mask_out, "mocap_screen_observations_host");
    if (st) return st;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    const int C = ctx->cfg.n_cam;
    const int n = n_points ? (*n_points < 0 ? 0 : *n_points < n_points_max ? *n_points : n_points_max) : n_points_max;
    const size_t rows = n > 0 ? (size_t)n : 1;
    double *d_obs, *d_R, *d_t;
    uint8_t *d_in, *d_out;
    int32_t* d_stats;
    st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
        d_obs = L.take<double>(rows * C * 2); d_in = L.take<uint8_t>(rows * C); d_out = L.take<uint8_t>(rows * C);
        d_R = L.take<double>((size_t)C * 9); d_t = L.take<double>((size_t)C * 3); d_stats = L.take<int32_t>(4);
    });
    if (st) return st;
    cudaStream_t s = ctx->stream;
    if (n > 0) {
        CUDA_TRY(ctx, cudaMemcpyAsync(d_obs, obs, (size_t)n * C * 2 * 8, cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_in, mask_in, (size_t)n * C, cudaMemcpyHostToDevice, s));
    } else {
        CUDA_TRY(ctx, cudaMemsetAsync(d_in, 0, C, s));           // one row without views: nothing to screen, zero stats
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(d_R, R, (size_t)C * 9 * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_t, t, (size_t)C * 3 * 8, cudaMemcpyHostToDevice, s));
    st = screen_launch(ctx, d_obs, d_in, (int)rows, nullptr, d_R, d_t, threshold_px, d_out, d_stats);
    if (st) return st;
    int32_t h_stats[4];
    if (n > 0) CUDA_TRY(ctx, cudaMemcpyAsync(mask_out, d_out, (size_t)n * C, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(h_stats, d_stats, sizeof(h_stats), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (stats) memcpy(stats, h_stats, sizeof(h_stats));
    return MOCAP_OK;
}

}  // extern "C"

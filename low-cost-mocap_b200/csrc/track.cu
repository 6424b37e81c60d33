// Drone tracking on the device (step code and semantics: track.cuh).  Two launches per batch of frame-sets, no
// synchronisation, on the context's stream:
//
// k_track_scan: one CTA, one warp per drone.  The warp walks the batch's frame-sets in order (the Kalman recursion is
//   sequential per drone); per frame-set its lanes gather the drone's candidates from the locate_objects output by
//   ballot, split the 9 x 9 products of the predict / correct steps over the entries and the association over the
//   candidates.  It writes pos, present and chosen, and appends the low-pass inputs of each present frame-set (the
//   posterior velocity and the chosen object's heading) to the drone's history rows, which carry the last
//   TRACK_HIST samples over to the next batch.  A pending reset is applied before the first frame-set.  A frame-set
//   whose call entry is 0 (call != NULL) is skipped: absent outputs, and neither the clock nor the history moves.
// k_track_lowpass: one thread per (frame-set, drone, channel); each runs its window of <= 300 samples from zero state.
#include <math.h>
#include "common.cuh"
#include "track.cuh"

struct mocap_tracker {
    mocap_ctx*  ctx;
    int         num_objects;
    TrackDrone* d_state;        // [num_objects]
    double*     d_hist;         // [num_objects * TRACK_CHANNELS][stride]
    int2*       d_slot;         // [cap][num_objects]: {history index of the sample, window length (0: absent)}
    int         cap;            // frame-sets per batch the buffers hold
    int         reset_pending;
    double      reset_time;
};

__global__ void __launch_bounds__(32 * TRACK_MAX_DRONES)
k_track_scan(TrackDrone* __restrict__ state, double* __restrict__ hist, int stride, const double* __restrict__ objects,
             const int32_t* __restrict__ drone_index, const int32_t* __restrict__ n_objects, int max_objects,
             const double* __restrict__ timestamps, const uint8_t* __restrict__ call, int n_sets, int reset, double reset_time,
             float* __restrict__ pos,
             uint8_t* __restrict__ present, int32_t* __restrict__ chosen, int2* __restrict__ slot) {
    __shared__ TrackWork work[TRACK_MAX_DRONES];
    __shared__ TrackDrone drones[TRACK_MAX_DRONES];
    const int d = threadIdx.x >> 5, lane = threadIdx.x & 31, D = blockDim.x >> 5;
    TrackWork& W = work[d];
    TrackDrone& S = drones[d];
    {
        const int* src = reinterpret_cast<const int*>(state + d);
        int* dst = reinterpret_cast<int*>(&S);
        for (int i = lane; i < (int)(sizeof(TrackDrone) / sizeof(int)); i += 32) dst[i] = src[i];
    }
    __syncwarp();
    if (reset && lane == 0) track_reset(S, reset_time);
    __syncwarp();
    for (int i = lane; i < 9; i += 32) W.x[i] = S.x[i];
    for (int i = lane; i < 81; i += 32) W.P[i] = S.P[i];
    // keep the last TRACK_HIST samples of the previous batch at the front of the rows (ascending chunks: the
    // destination never overtakes the source)
    int hist_len = S.hist_len;
    const int keep = min(hist_len, TRACK_HIST), shift = hist_len - keep;
    if (shift > 0)
        for (int ch = 0; ch < TRACK_CHANNELS; ++ch) {
            double* row = hist + (size_t)(d * TRACK_CHANNELS + ch) * stride;
            for (int i0 = 0; i0 < keep; i0 += 32) {
                const double v = i0 + lane < keep ? row[shift + i0 + lane] : 0.0;
                __syncwarp();
                if (i0 + lane < keep) row[i0 + lane] = v;
                __syncwarp();
            }
        }
    hist_len = keep;
    int k = S.k;
    double prev_time = S.prev_time;
    __syncwarp();

    for (int s = 0; s < n_sets; ++s) {
        const size_t o = (size_t)s * D + d;
        if (call && !call[s]) {
            if (lane < 3) pos[3 * o + lane] = 0.0f;
            if (lane == 0) { present[o] = 0; chosen[o] = -1; slot[o] = make_int2(0, 0); }
            continue;
        }
        const double t = timestamps[s];
        const double dt = DSUB(t, prev_time);
        prev_time = t;
        const int n = min(max(n_objects[s], 0), max_objects);
        const double* obj = objects + (size_t)s * max_objects * 5;
        const int32_t* di = drone_index + (size_t)s * max_objects;
        int first = -1;
        for (int c0 = 0; c0 < n && first < 0; c0 += 32) {
            const unsigned hit = __ballot_sync(0xffffffffu, c0 + lane < n && di[c0 + lane] == d);
            if (hit) first = c0 + __ffs(hit) - 1;
        }
        if (first < 0) {
            if (lane < 3) pos[3 * o + lane] = 0.0f;
            if (lane == 0) { present[o] = 0; chosen[o] = -1; slot[o] = make_int2(0, 0); }
            continue;
        }
        if (lane == 0) track_init(W, obj + (size_t)first * 5);
        __syncwarp();
        float fdt, fh;
        track_dt_terms(dt, fdt, fh);
        track_predict_a(W, fdt, fh, lane, 32);
        __syncwarp();
        track_predict_b(W, fdt, fh, lane, 32);
        __syncwarp();
        // nearest candidate, first minimum: each lane scans its candidates in order, then the warp keeps the smaller
        // distance and, between equal ones, the smaller row
        double best = INFINITY;
        int bj = n;
        for (int j = first + lane; j < n; j += 32)
            if (di[j] == d) {
                const double dist = track_dist(obj + (size_t)j * 5, W.x);
                if (dist < best) { best = dist; bj = j; }
            }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, off);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, off);
            if (ob < best || (ob == best && oj < bj)) { best = ob; bj = oj; }
        }
        if (bj >= n) bj = first;           // every distance NaN: np.argmin's first entry
        const double* cand = obj + (size_t)bj * 5;
        if (lane == 0) track_measure(W, S, cand, dt);
        __syncwarp();
        track_gain(W, lane, 32);
        __syncwarp();
        track_correct(W, lane, 32);
        __syncwarp();
        if (lane < 9) W.x[lane] = W.xn[lane];
        __syncwarp();
        if (lane < 3) pos[3 * o + lane] = W.x[lane];
        if (lane < 3) hist[(size_t)(d * TRACK_CHANNELS + lane) * stride + hist_len] = (double)W.x[3 + lane];
        if (lane == 3) hist[(size_t)(d * TRACK_CHANNELS + 3) * stride + hist_len] = cand[3];
        k = track_next_call(k);
        if (lane == 0) { present[o] = 1; chosen[o] = bj; slot[o] = make_int2(hist_len, track_window(k)); }
        ++hist_len;
    }
    __syncwarp();
    if (lane == 0) { S.k = k; S.hist_len = hist_len; S.prev_time = prev_time; }
    for (int i = lane; i < 9; i += 32) S.x[i] = W.x[i];
    for (int i = lane; i < 81; i += 32) S.P[i] = W.P[i];
    __syncwarp();
    {
        const int* src = reinterpret_cast<const int*>(&S);
        int* dst = reinterpret_cast<int*>(state + d);
        for (int i = lane; i < (int)(sizeof(TrackDrone) / sizeof(int)); i += 32) dst[i] = src[i];
    }
}

__global__ void __launch_bounds__(256)
k_track_lowpass(const double* __restrict__ hist, int stride, const int2* __restrict__ slot, int n_sets, int D,
                float* __restrict__ vel, double* __restrict__ heading) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_sets * D * TRACK_CHANNELS) return;
    const int ch = e % TRACK_CHANNELS, o = e / TRACK_CHANNELS, d = o % D;
    const int2 sl = slot[o];
    double y = 0.0;
    if (sl.y > 0) y = track_lowpass(hist + (size_t)(d * TRACK_CHANNELS + ch) * stride + sl.x - sl.y + 1, sl.y);
    if (ch < 3) vel[3 * o + ch] = TF32(y);
    else heading[o] = y;
}

mocap_ctx* tracker_context(const mocap_tracker* tr) { return tr->ctx; }
int tracker_num_objects(const mocap_tracker* tr) { return tr->num_objects; }

static size_t hist_stride(int cap) { return (size_t)TRACK_HIST + (size_t)cap; }

// buffers for batches of n_sets frame-sets; a larger batch reallocates them (after the stream drains) and keeps the
// history rows
static int tracker_reserve(mocap_tracker* tr, int n_sets) {
    if (n_sets <= tr->cap) return MOCAP_OK;
    mocap_ctx* ctx = tr->ctx;
    int cap = tr->cap ? tr->cap : 1024;
    while (cap < n_sets) cap *= 2;
    const size_t rows = (size_t)tr->num_objects * TRACK_CHANNELS;
    double* hist = nullptr;
    int2* slot = nullptr;
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(ctx, cudaMalloc(&hist, rows * hist_stride(cap) * sizeof(double)));
    if (cudaMalloc(&slot, (size_t)cap * tr->num_objects * sizeof(int2)) != cudaSuccess) {
        cudaFree(hist);
        return mocap_fail(ctx, MOCAP_ECUDA, "mocap_track_objects_dev: out of device memory for %d frame-sets", n_sets);
    }
    if (tr->d_hist)
        CUDA_TRY(ctx, cudaMemcpy2D(hist, hist_stride(cap) * sizeof(double), tr->d_hist, hist_stride(tr->cap) * sizeof(double),
                                   hist_stride(tr->cap) * sizeof(double), rows, cudaMemcpyDeviceToDevice));
    cudaFree(tr->d_hist);
    cudaFree(tr->d_slot);
    tr->d_hist = hist;
    tr->d_slot = slot;
    tr->cap = cap;
    return MOCAP_OK;
}

extern "C" {

int mocap_tracker_create(mocap_ctx* ctx, int num_objects, mocap_tracker** out) {
    if (!ctx) return MOCAP_EINVAL;
    if (!out) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_tracker_create: bad argument");
    *out = nullptr;
    if (num_objects < 1 || num_objects > TRACK_MAX_DRONES)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_tracker_create: num_objects must be 1 .. %d (got %d)", TRACK_MAX_DRONES, num_objects);
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    mocap_tracker* tr = new mocap_tracker();
    tr->ctx = ctx;
    tr->num_objects = num_objects;
    TrackDrone init[TRACK_MAX_DRONES];
    memset(init, 0, sizeof(init));
    for (int d = 0; d < num_objects; ++d) init[d].prev_int = 1;    // prev_positions starts as the list [0, 0, 0]
    if (cudaMalloc(&tr->d_state, num_objects * sizeof(TrackDrone)) != cudaSuccess ||
        cudaMemcpy(tr->d_state, init, num_objects * sizeof(TrackDrone), cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(tr->d_state);
        delete tr;
        return mocap_fail(ctx, MOCAP_ECUDA, "mocap_tracker_create: device allocation failed");
    }
    *out = tr;
    return MOCAP_OK;
}

void mocap_tracker_destroy(mocap_tracker* tr) {
    if (!tr) return;
    cudaSetDevice(tr->ctx->cfg.device);
    cudaStreamSynchronize(tr->ctx->stream);
    cudaFree(tr->d_state);
    cudaFree(tr->d_hist);
    cudaFree(tr->d_slot);
    delete tr;
}

int mocap_tracker_reset(mocap_tracker* tr, double prev_time) {
    if (!tr) return MOCAP_EINVAL;
    if (!isfinite(prev_time)) return mocap_fail(tr->ctx, MOCAP_EINVAL, "mocap_tracker_reset: prev_time must be finite");
    tr->reset_pending = 1;      // applied by the next batch before its first frame-set
    tr->reset_time = prev_time;
    return MOCAP_OK;
}

int mocap_track_objects_dev(mocap_tracker* tr, const double* objects, const int32_t* drone_index, const int32_t* n_objects,
                            int max_objects, const double* timestamps, int n_frame_sets, float* pos, float* vel,
                            double* heading, uint8_t* present, int32_t* chosen) {
    return mocap_track_objects_gated_dev(tr, objects, drone_index, n_objects, max_objects, timestamps, nullptr, n_frame_sets, pos,
                                         vel, heading, present, chosen);
}

int mocap_track_objects_gated_dev(mocap_tracker* tr, const double* objects, const int32_t* drone_index, const int32_t* n_objects,
                                  int max_objects, const double* timestamps, const uint8_t* call, int n_frame_sets, float* pos,
                                  float* vel, double* heading, uint8_t* present, int32_t* chosen) {
    if (!tr) return MOCAP_EINVAL;
    mocap_ctx* ctx = tr->ctx;
    if (!objects || !drone_index || !n_objects || !timestamps || !pos || !vel || !heading || !present || !chosen)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_track_objects_dev: bad argument");
    if (max_objects < 1 || n_frame_sets < 1)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_track_objects_dev: max_objects and n_frame_sets must be >= 1 (got %d, %d)",
                          max_objects, n_frame_sets);
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    int st = tracker_reserve(tr, n_frame_sets);
    if (st) return st;
    const int D = tr->num_objects;
    const int stride = (int)hist_stride(tr->cap);
    k_track_scan<<<1, 32 * D, 0, ctx->stream>>>(tr->d_state, tr->d_hist, stride, objects, drone_index, n_objects, max_objects,
                                                timestamps, call, n_frame_sets, tr->reset_pending, tr->reset_time, pos, present, chosen,
                                                tr->d_slot);
    CUDA_TRY(ctx, cudaGetLastError());
    tr->reset_pending = 0;
    const int threads = n_frame_sets * D * TRACK_CHANNELS;
    k_track_lowpass<<<(threads + 255) / 256, 256, 0, ctx->stream>>>(tr->d_hist, stride, tr->d_slot, n_frame_sets, D, vel, heading);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 2;
    return MOCAP_OK;
}

}  // extern "C"

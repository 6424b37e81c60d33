// The live capture loop on the device: Cameras._camera_read (reference computer_code/api/helpers.py:68-135) for a
// batch of reads, from the camera driver's raw frames to the tracker's filtered drone states.
//
// Every stage is an existing launcher; this file adds k_live_blobs and the call sequence:
//   run_raw_groups (preproc.cu): per launch group, k_preprocess -> S1 (mode CAPTURE) or S1+S2+S3 (TRIANGULATE, the
//     matcher writing n / obj / err / flags of the result) -> k_live_blobs (per-read step code: live.cuh);
//   then, over all reads, k_locate_objects and the gated tracker (LOCATE), called = the reads the reference makes a
//   predict_location call on.
// Each stage writes its own slice of the one result buffer, so the host form needs one copy back.
#include "common.cuh"
#include "live.cuh"

static_assert(LIVE_CAPTURE == MOCAP_LIVE_CAPTURE && LIVE_TRIANGULATE == MOCAP_LIVE_TRIANGULATE && LIVE_LOCATE == MOCAP_LIVE_LOCATE,
              "live.cuh mirrors the MOCAP_LIVE_* bits");

#define LIVE_THRESHOLD 51      // cv.threshold(grey, 255*0.2, 255, THRESH_BINARY) on uint8 == pix > 51 (helpers.py:146)

// one thread per read of the launch group; blob lists of the group's images as S1 left them in the context
__global__ void __launch_bounds__(128)
k_live_blobs(const int32_t* __restrict__ blob_xy, const int32_t* __restrict__ blob_n, const int32_t* __restrict__ img_flags,
             int n_sets, int C, int MB, int S, int have_blobs, LiveOut L, uint8_t* __restrict__ frames) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_sets) return;
    const int32_t* xy = blob_xy + (size_t)r * C * MB * 2;
    live_read(C, MB, xy, blob_n + (size_t)r * C, img_flags + (size_t)r * C, have_blobs, L.mode & LIVE_LOCATE,
              L.mode & LIVE_TRIANGULATE, L.blob_n + (size_t)r * C, L.first + (size_t)r * C * 2, L.gate + r, L.called + r, L.flags + r);
    if (frames && have_blobs)
        for (int c = 0; c < C; ++c)
            live_dots(MB, xy + (size_t)c * MB * 2, blob_n[(size_t)r * C + c], S, frames + ((size_t)r * C + c) * S * S * 3);
}

int launch_live_blobs(mocap_ctx* ctx, const LiveOut& live, int s0, int n_sets, int have_blobs, uint8_t* frames) {
    if (n_sets <= 0) return MOCAP_OK;
    const int C = ctx->cfg.n_cam;
    LiveOut L = live;
    L.flags += s0; L.gate += s0; L.called += s0;
    L.blob_n += (size_t)s0 * C; L.first += (size_t)s0 * C * 2;
    k_live_blobs<<<(n_sets + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_blob_xy, ctx->d_blob_n, ctx->d_img_flags, n_sets, C,
                                                                 ctx->cfg.max_blobs, ctx->cfg.width, have_blobs, L,
                                                                 (live.mode & LIVE_CAPTURE) ? frames : nullptr);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    return MOCAP_OK;
}

static uint64_t slice(uint64_t& at, uint64_t bytes) {
    const uint64_t o = at;
    at = (at + bytes + 15) & ~(uint64_t)15;
    return o;
}

static void live_offsets(const mocap_config& c, int R, int D, mocap_live_offsets* L) {
    const uint64_t r = (uint64_t)R, C = (uint64_t)c.n_cam, RM = (uint64_t)c.max_roots, d = (uint64_t)D;
    uint64_t at = 0;
    L->obj = slice(at, r * RM * 3 * 8);
    L->err = slice(at, r * RM * 8);
    L->objects = slice(at, r * RM * 5 * 8);
    L->heading = slice(at, r * d * 8);
    L->pos = slice(at, r * d * 3 * 4);
    L->vel = slice(at, r * d * 3 * 4);
    L->flags = slice(at, r * 4);
    L->blob_n = slice(at, r * C * 4);
    L->first = slice(at, r * C * 2 * 4);
    L->n = slice(at, r * 4);
    L->n_objects = slice(at, r * 4);
    L->drone_index = slice(at, r * RM * 4);
    L->chosen = slice(at, r * d * 4);
    L->gate = slice(at, r);
    L->called = slice(at, r);
    L->present = slice(at, r * d);
    L->total = at;
}

// the checks the entry points make before anything is launched or copied
int live_check(mocap_ctx* ctx, mocap_tracker* tr, const void* raw, int n_reads, int mode, const double* timestamps,
               const void* result, const char* who) {
    if (!raw || !result || n_reads < 0) return mocap_fail(ctx, MOCAP_EINVAL, "%s: bad argument", who);
    if (mode != 0 && mode != LIVE_CAPTURE && mode != (LIVE_CAPTURE | LIVE_TRIANGULATE) &&
        mode != (LIVE_CAPTURE | LIVE_TRIANGULATE | LIVE_LOCATE))
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: mode %d is not 0, CAPTURE, CAPTURE|TRIANGULATE or CAPTURE|TRIANGULATE|LOCATE "
                                             "(the reference triangulates only while capturing, and locates only while triangulating)", who, mode);
    if ((mode & LIVE_LOCATE) && (!tr || !timestamps))
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: LOCATE needs a tracker and timestamps", who);
    if (tr && tracker_context(tr) != ctx) return mocap_fail(ctx, MOCAP_EINVAL, "%s: the tracker belongs to another context", who);
    if (!ctx->pp_in_w) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_preprocess has not been called");
    if ((mode & LIVE_TRIANGULATE) && !ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    return MOCAP_OK;
}

static int live_run(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode, const double* timestamps,
                    uint8_t* frames, void* result) {
    if (n_reads == 0) return MOCAP_OK;
    mocap_live_offsets L;
    live_offsets(ctx->cfg, n_reads, tr ? tracker_num_objects(tr) : 0, &L);
    uint8_t* base = static_cast<uint8_t*>(result);
    LiveOut live;
    live.flags = reinterpret_cast<int32_t*>(base + L.flags);
    live.gate = base + L.gate;
    live.blob_n = reinterpret_cast<int32_t*>(base + L.blob_n);
    live.first = reinterpret_cast<int32_t*>(base + L.first);
    live.called = base + L.called;
    live.mode = mode;
    double* obj = reinterpret_cast<double*>(base + L.obj);
    double* err = reinterpret_cast<double*>(base + L.err);
    int32_t* n = reinterpret_cast<int32_t*>(base + L.n);
    const int stages = (mode & LIVE_TRIANGULATE) ? RAW_MATCH : (mode & LIVE_CAPTURE) ? RAW_DETECT : RAW_PREPROCESS;
    int st = run_raw_groups(ctx, raw, n_reads, LIVE_THRESHOLD, stages, frames, obj, err, n, live.flags, &live);
    if (st || !(mode & LIVE_LOCATE)) return st;
    const int M = ctx->cfg.max_roots;          // one object per point at most: nothing is dropped (the reference is unbounded)
    double* objects = reinterpret_cast<double*>(base + L.objects);
    int32_t* drone_index = reinterpret_cast<int32_t*>(base + L.drone_index);
    int32_t* n_objects = reinterpret_cast<int32_t*>(base + L.n_objects);
    st = launch_locate(ctx, obj, err, n, n_reads, M, objects, drone_index, n_objects);
    if (st) return st;
    return mocap_track_objects_gated_dev(tr, objects, drone_index, n_objects, M, timestamps, live.called, n_reads,
                                         reinterpret_cast<float*>(base + L.pos), reinterpret_cast<float*>(base + L.vel),
                                         reinterpret_cast<double*>(base + L.heading), base + L.present,
                                         reinterpret_cast<int32_t*>(base + L.chosen));
}

extern "C" {

int mocap_live_layout(mocap_ctx* ctx, int n_reads, int num_objects, mocap_live_offsets* layout) {
    if (!ctx) return MOCAP_EINVAL;
    if (!layout || n_reads < 0 || num_objects < 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_live_layout: bad argument");
    live_offsets(ctx->cfg, n_reads, num_objects, layout);
    return MOCAP_OK;
}

int mocap_live_dev(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode, const double* timestamps,
                   uint8_t* frames, void* result) {
    if (!ctx) return MOCAP_EINVAL;
    int st = live_check(ctx, tr, raw, n_reads, mode, timestamps, result, "mocap_live_dev");
    if (st) return st;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return live_run(ctx, tr, raw, n_reads, mode, timestamps, frames, result);
}

int mocap_live_host(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode, const double* timestamps,
                    uint8_t* frames, void* result) {
    if (!ctx) return MOCAP_EINVAL;
    int st = live_check(ctx, tr, raw, n_reads, mode, timestamps, result, "mocap_live_host");
    if (st || n_reads == 0) return st;
    LiveHostRun run;
    if ((st = live_host_run(ctx, tr, raw, n_reads, mode, timestamps, frames != nullptr, 0, &run)) != MOCAP_OK) return st;
    return live_host_finish(ctx, run, frames, result, nullptr, nullptr);
}

}  // extern "C"

// mocap_live_host up to the chain: staging in, live_run.  The processed frames stay on the device at run->d_frames when
// keep_frames; extra_bytes more of page-locked staging are kept for live_host_finish.
int live_host_run(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode, const double* timestamps,
                  int keep_frames, size_t extra_bytes, LiveHostRun* run) {
    int st;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    const int C = ctx->cfg.n_cam, S = ctx->cfg.width;
    mocap_live_offsets& L = run->L;
    live_offsets(ctx->cfg, n_reads, tr ? tracker_num_objects(tr) : 0, &L);
    const size_t raw_bytes = (size_t)n_reads * C * ctx->pp_in_w * ctx->pp_in_h * 3;
    run->frame_copy = keep_frames ? (size_t)n_reads * C * S * S * 3 : 0;
    run->extra_bytes = extra_bytes;
    double* d_ts;
    uint8_t *d_raw, *d_extra;
    // device buffers and their page-locked twins, the same layout in both; the stream has drained if a device buffer grew
    if ((st = grow_carved(ctx, ctx->live_in, Drain::stream, [&](Layout& R) {
             d_ts = R.take<double>((mode & LIVE_LOCATE) ? n_reads : 0); d_raw = R.take<uint8_t>(raw_bytes); })) ||
        (st = ctx->live_in_host.grow(ctx, ctx->live_in.bytes(), Drain::none)) ||
        (st = grow_carved(ctx, ctx->live_out, Drain::stream, [&](Layout& R) {
             R.take<uint8_t>(L.total);                             // the result, at offset 0
             run->d_frames = R.take<uint8_t>(run->frame_copy); d_extra = R.take<uint8_t>(extra_bytes); })) ||
        (st = ctx->live_out_host.grow(ctx, ctx->live_out.bytes(), Drain::none)))
        return st;
    run->frame_off = run->d_frames - ctx->live_out.as<uint8_t>();
    run->extra_off = d_extra - ctx->live_out.as<uint8_t>();
    if (!keep_frames) run->d_frames = nullptr;
    // the staging buffers are free here: the previous call returned after its synchronisation
    uint8_t* h_in = ctx->live_in_host.as<uint8_t>();
    const size_t raw_off = d_raw - ctx->live_in.as<uint8_t>();
    if (mode & LIVE_LOCATE) memcpy(h_in, timestamps, (size_t)n_reads * sizeof(double));
    memcpy(h_in + raw_off, raw, raw_bytes);
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->live_in.get(), h_in, raw_off + raw_bytes, cudaMemcpyHostToDevice, ctx->stream));
    return live_run(ctx, tr, d_raw, n_reads, mode, (mode & LIVE_LOCATE) ? d_ts : nullptr, run->d_frames, ctx->live_out.get());
}

// the rest of mocap_live_host: the result, the frames (frames != NULL) and run.extra_bytes from the device pointer
// `extra` back to the host, one synchronisation
int live_host_finish(mocap_ctx* ctx, const LiveHostRun& run, uint8_t* frames, void* result, const void* extra, void* extra_out) {
    uint8_t* h_out = ctx->live_out_host.as<uint8_t>();
    CUDA_TRY(ctx, cudaMemcpyAsync(h_out, ctx->live_out.get(), run.L.total, cudaMemcpyDeviceToHost, ctx->stream));
    if (frames) CUDA_TRY(ctx, cudaMemcpyAsync(h_out + run.frame_off, run.d_frames, run.frame_copy, cudaMemcpyDeviceToHost, ctx->stream));
    if (run.extra_bytes) CUDA_TRY(ctx, cudaMemcpyAsync(h_out + run.extra_off, extra, run.extra_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(result, h_out, run.L.total);
    if (frames) memcpy(frames, h_out + run.frame_off, run.frame_copy);
    if (run.extra_bytes) memcpy(extra_out, h_out + run.extra_off, run.extra_bytes);
    return MOCAP_OK;
}

// C ABI of libmocap_b200.so (see include/mocap_b200.h for the contract and the
// reference functions each entry point replaces).
#include <stdarg.h>
#include <stdlib.h>
#include <math.h>
#include <new>
#include "common.cuh"
#include "camera_tables.h"

int blob_kernels_init(mocap_ctx* ctx);
int match_kernels_init(mocap_ctx* ctx);
int fused_kernel_init(mocap_ctx* ctx);
int ba_dev_init(mocap_ctx* ctx);

int mocap_fail(mocap_ctx* ctx, int code, const char* fmt, ...) {
    if (ctx) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
        va_end(ap);
    }
    return code;
}

// ---- scratch management ------------------------------------------------------------------
int ensure_images(mocap_ctx* ctx, int n_images) {
    if (n_images <= ctx->cap_images) return MOCAP_OK;
    const size_t n = (size_t)n_images;
    int st = grow_carved(ctx, ctx->images, Drain::stream, [&](Layout& L) {
        ctx->d_seg_count = L.take<uint32_t>(n); ctx->d_work_count = L.take<uint32_t>(4);     // kept zero by the kernels afterwards
        ctx->d_img_done = L.take<uint32_t>(n); ctx->d_set_done = L.take<uint32_t>(2 * n);
        L.zero_so_far();
        ctx->d_seg_list = L.take<uint32_t>(n * ctx->cfg.max_segments); ctx->d_worklist = L.take<uint32_t>(n);
        ctx->d_set_worklist = L.take<uint32_t>(n); ctx->d_unit_counter = L.take<unsigned long long>(1);
        ctx->d_blob_xy = L.take<int32_t>(n * ctx->cfg.max_blobs * 2); ctx->d_blob_n = L.take<int32_t>(n); ctx->d_img_flags = L.take<int32_t>(n);
    });
    ctx->cap_images = st ? 0 : n_images;
    return st;
}

static int ensure_sets(mocap_ctx* ctx, int n_sets) {
    if (n_sets <= ctx->cap_sets) return MOCAP_OK;
    const size_t n = (size_t)n_sets, R = ctx->cfg.max_roots;
    int st = grow_carved(ctx, ctx->sets, Drain::stream, [&](Layout& L) {
        ctx->d_obj = L.take<double>(n * R * 3); ctx->d_err = L.take<double>(n * R);
        ctx->d_nobj = L.take<int32_t>(n); ctx->d_setflags = L.take<int32_t>(n);
    });
    ctx->cap_sets = st ? 0 : n_sets;
    return st;
}

// Single-pass kernel or three-kernel pipeline for this batch of 1-channel frames?  The single-pass kernel wins
// while the sparse stages are light (config 2: 4.34 ms against 4.70 ms per 10 000 frame-sets on an H100 SXM at a
// 400 W power limit); with many blobs per frame-set the sparse stages interleaved with the stream loop on every SM
// hold back the stream (config 3 shape: 5.68 ms against 5.29 ms per 4000 frame-sets), so batches that follow a heavy
// batch take the three-kernel pipeline.  The blob count of the previous batch arrives through mapped host memory
// (written by the last CTA of the blob fallback kernel): no synchronisation, a stale or torn value only steers
// this heuristic, both pipelines give the same results.
bool pick_fused(const mocap_ctx* ctx) {
    if (!ctx->use_fused) return false;
    if (!ctx->pipeline_auto) return true;
    const volatile unsigned long long* h_stat = ctx->stat_host.as<volatile unsigned long long>();
    const unsigned long long blobs = h_stat[0], images = h_stat[1];
    if (images == 0) return true;
    return (double)blobs * ctx->cfg.n_cam <= (double)MOCAP_HEAVY_BLOBS_PER_SET * (double)images;
}

// Launch groups bound the detection scratch (max_segments * 4 B of segment list per image) at any batch size: 65 536
// images for the single-pass kernel, 4096 frame-sets for the three-kernel pipeline.
int run_sets(mocap_ctx* ctx, const uint8_t* frames, int n_sets, int channels, int threshold, bool fused, const SetOut& out,
             cudaEvent_t frames_read) {
    const int C = ctx->cfg.n_cam;
    const size_t set_bytes = (size_t)C * ctx->cfg.width * ctx->cfg.height * channels;
    const int group = fused ? (65536 / C > 0 ? 65536 / C : 1) : 4096;
    int st = ensure_images(ctx, (n_sets < group ? n_sets : group) * C);
    if (st) return st;
    for (int s0 = 0; s0 < n_sets; s0 += group) {
        const int ns = (n_sets - s0 < group) ? n_sets - s0 : group;
        const uint8_t* f = frames + (size_t)s0 * set_bytes;
        const SetOut o = out.at(ctx->cfg, s0);      // frame-set indices inside a launch group start at 0
        st = fused ? launch_pipeline_fused(ctx, f, ns, channels, threshold, o)
                   : launch_detect(ctx, f, ns * C, channels, threshold, ctx->d_blob_xy, ctx->d_blob_n, nullptr, ctx->d_img_flags);
        if (st) return st;
        if (frames_read) CUDA_TRY(ctx, cudaEventRecord(frames_read, ctx->stream));
        if (!fused && (st = launch_match(ctx, ctx->d_blob_xy, ctx->d_blob_n, ns, o, ctx->d_img_flags, nullptr)) != MOCAP_OK) return st;
    }
    return MOCAP_OK;
}

extern "C" {

const char* mocap_status_string(int status) {
    switch (status) {
        case MOCAP_OK: return "ok";
        case MOCAP_EINVAL: return "invalid argument";
        case MOCAP_ENODEV: return "no usable CUDA device (libmocap_b200 needs an sm_90 (H100) GPU; there is no CPU fallback)";
        case MOCAP_ECUDA: return "CUDA runtime error";
        case MOCAP_ENOMEM: return "out of memory";
        case MOCAP_ESTATE: return "call order error (cameras not set?)";
        default: return "unknown status";
    }
}

void mocap_default_config(mocap_config* cfg, int n_cam, int width, int height) {
    cfg->device = 0;
    cfg->n_cam = n_cam;
    cfg->width = width;
    cfg->height = height;
    cfg->max_blobs = 32;
    cfg->max_segments = 1024;
    cfg->max_roots = 64;
    cfg->max_cands = 8;
    cfg->max_groups = 4096;
}

const char* mocap_last_error(const mocap_ctx* ctx) { return ctx ? ctx->err : "no context"; }

static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

int mocap_create(mocap_ctx** out, const mocap_config* cfg) {
    if (!out || !cfg) return MOCAP_EINVAL;
    *out = nullptr;
    if (cfg->n_cam < 1 || cfg->n_cam > MOCAP_MAX_CAM || cfg->width < 16 || cfg->width % MOCAP_SEG_PX != 0 ||
        cfg->height < 1 || cfg->max_blobs < 1 || cfg->max_blobs > MOCAP_MAX_BLOBS ||
        !is_pow2(cfg->max_segments) || cfg->max_segments < 64 || cfg->max_segments > 4096 ||
        cfg->max_roots < 1 || cfg->max_roots > MOCAP_MAX_ROOTS || cfg->max_cands < 1 || cfg->max_cands > MOCAP_MAX_CANDS ||
        cfg->max_groups < 1 || (long long)cfg->width * cfg->height / MOCAP_SEG_PX > 65535)
        return MOCAP_EINVAL;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0 || cfg->device < 0 || cfg->device >= n_dev) {
        cudaGetLastError();
        return MOCAP_ENODEV;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess) return MOCAP_ENODEV;
    if (prop.major != 9 || prop.minor != 0) return MOCAP_ENODEV;     // the fatbin holds sm_90a code only
    if (cudaSetDevice(cfg->device) != cudaSuccess) return MOCAP_ENODEV;

    mocap_ctx* ctx = new (std::nothrow) mocap_ctx();
    if (!ctx) return MOCAP_ENOMEM;
    ctx->cfg = *cfg;
    ctx->num_sms = prop.multiProcessorCount;
    ctx->h_tables.n_cam = cfg->n_cam;
    int st = MOCAP_OK;
    do {
        if (ctx->tables.grow(ctx, sizeof(CameraTables), Drain::none) != MOCAP_OK) { st = MOCAP_ENOMEM; break; }
        ctx->d_tables = ctx->tables.as<CameraTables>();
        if (cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { st = MOCAP_ECUDA; break; }
        if (cudaStreamCreateWithFlags(&ctx->copy_stream2, cudaStreamNonBlocking) != cudaSuccess) { st = MOCAP_ECUDA; break; }
        for (int k = 0; k < 2 * 64; ++k)
            if (cudaEventCreate(&ctx->tim_ev[k]) != cudaSuccess) { st = MOCAP_ECUDA; break; }
        if (st) break;
        for (int k = 0; k < 2; ++k) {
            if (cudaEventCreateWithFlags(&ctx->stage_free[k], cudaEventDisableTiming) != cudaSuccess) { st = MOCAP_ECUDA; break; }
            if (cudaEventCreateWithFlags(&ctx->copied[k], cudaEventDisableTiming) != cudaSuccess) { st = MOCAP_ECUDA; break; }
        }
        if (st) break;
        if ((st = blob_kernels_init(ctx)) != MOCAP_OK) break;
        if ((st = match_kernels_init(ctx)) != MOCAP_OK) break;
        {
            // MOCAP_PIPELINE = split | fused pins the pipeline (A/B measurements); unset: single-pass kernel,
            // except for batches of heavy frame-sets (see pick_fused)
            const char* mode = getenv("MOCAP_PIPELINE");
            ctx->use_fused = (mode && strcmp(mode, "split") == 0) ? 0 : 1;
            ctx->pipeline_auto = (mode && mode[0]) ? 0 : 1;
        }
        {
            if (ctx->stat_host.grow(ctx, 16, Drain::none, 16, cudaHostAllocMapped) != MOCAP_OK) { st = MOCAP_ENOMEM; break; }
            void* d = nullptr;
            if (cudaHostGetDevicePointer(&d, ctx->stat_host.get(), 0) != cudaSuccess) { st = MOCAP_ECUDA; break; }
            ctx->d_stat_host = static_cast<unsigned long long*>(d);
            if (ctx->stat_acc.grow(ctx, 8, Drain::none, 8) != MOCAP_OK) { st = MOCAP_ENOMEM; break; }
        }
        if ((st = fused_kernel_init(ctx)) != MOCAP_OK) break;
        if ((st = ba_dev_init(ctx)) != MOCAP_OK) break;
    } while (0);
    if (st != MOCAP_OK) { mocap_destroy(ctx); return st; }
    *out = ctx;
    return MOCAP_OK;
}

void mocap_destroy(mocap_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->cfg.device);
    cudaDeviceSynchronize();
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->copy_stream2) cudaStreamDestroy(ctx->copy_stream2);
    for (int k = 0; k < 2 * 64; ++k) if (ctx->tim_ev[k]) cudaEventDestroy(ctx->tim_ev[k]);
    for (int k = 0; k < 2; ++k) if (ctx->stage_free[k]) cudaEventDestroy(ctx->stage_free[k]);
    for (int k = 0; k < 2; ++k) if (ctx->copied[k]) cudaEventDestroy(ctx->copied[k]);
    delete ctx;
}

int mocap_set_stream(mocap_ctx* ctx, void* cuda_stream) {
    if (!ctx) return MOCAP_EINVAL;
    ctx->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    return MOCAP_OK;
}

int mocap_set_large_holes(mocap_ctx* ctx, int on) {
    if (!ctx) return MOCAP_EINVAL;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return blob_set_large_holes(ctx, on);
}

// ---- host-side camera tables: camera_tables.h ---------------------------------------------
int mocap_set_cameras(mocap_ctx* ctx, const double* K, const double* R, const double* t) {
    if (!ctx || !K || !R || !t) return MOCAP_EINVAL;
    const int C = ctx->cfg.n_cam;
    CameraTables& T = ctx->h_tables;
    build_camera_tables(T, C, K, R, t);
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_tables, &T, sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));      // T lives in pageable memory of the ctx
    ctx->cameras_set = true;
    return MOCAP_OK;
}

int mocap_set_world_transform(mocap_ctx* ctx, const double* M) {
    if (!ctx) return MOCAP_EINVAL;
    CameraTables& T = ctx->h_tables;
    T.use_world = M ? 1 : 0;
    if (M) memcpy(T.world, M, 16 * sizeof(double));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_tables, &T, sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return MOCAP_OK;
}

// ---- S1 ------------------------------------------------------------------------------------
int mocap_detect_dev(mocap_ctx* ctx, const uint8_t* frames, int n_images, int channels, int threshold,
                     int32_t* blob_xy, int32_t* blob_n, int64_t* blob_mom, int32_t* img_flags) {
    if (!ctx) return MOCAP_EINVAL;
    if (!frames || !blob_xy || !blob_n || n_images < 0 || (channels != 1 && channels != 3))
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_detect_dev: bad argument");
    if ((reinterpret_cast<uintptr_t>(frames) & 15u) != 0)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_detect_dev: frames must be 16-byte aligned");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    int st = ensure_images(ctx, n_images);
    if (st) return st;
    return launch_detect(ctx, frames, n_images, channels, threshold, blob_xy, blob_n, blob_mom, img_flags);
}

// ---- S2+S3 ---------------------------------------------------------------------------------
int mocap_match_triangulate_dev(mocap_ctx* ctx, const int32_t* blob_xy, const int32_t* blob_n, int n_frame_sets,
                                double* obj, double* err, int32_t* n_obj, int32_t* set_flags, int32_t* chosen) {
    if (!ctx) return MOCAP_EINVAL;
    if (!blob_xy || !blob_n || !obj || !err || !n_obj || n_frame_sets < 0)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_match_triangulate_dev: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return launch_match(ctx, blob_xy, blob_n, n_frame_sets, SetOut{obj, err, n_obj, set_flags, nullptr}, nullptr, chosen);
}

// ---- S1+S2+S3 ------------------------------------------------------------------------------
int mocap_pipeline_dev(mocap_ctx* ctx, const uint8_t* frames, int n_frame_sets, int channels, int threshold,
                       double* obj, double* err, int32_t* n_obj, int32_t* set_flags) {
    return mocap_pipeline_tracks_dev(ctx, frames, n_frame_sets, channels, threshold, obj, err, n_obj, set_flags, nullptr);
}

int mocap_pipeline_tracks_dev(mocap_ctx* ctx, const uint8_t* frames, int n_frame_sets, int channels, int threshold,
                              double* obj, double* err, int32_t* n_obj, int32_t* set_flags, int32_t* track_xy) {
    if (!ctx) return MOCAP_EINVAL;
    if (!frames || !obj || !err || !n_obj || n_frame_sets < 0 || (channels != 1 && channels != 3))
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_pipeline_dev: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return run_sets(ctx, frames, n_frame_sets, channels, threshold, pick_fused(ctx), SetOut{obj, err, n_obj, set_flags, track_xy}, nullptr);
}

int mocap_pipeline_host(mocap_ctx* ctx, const uint8_t* frames, int n_frame_sets, int channels, int threshold,
                        double* obj, double* err, int32_t* n_obj, int32_t* set_flags) {
    if (!ctx) return MOCAP_EINVAL;
    if (!frames || !obj || !err || !n_obj || n_frame_sets < 0 || (channels != 1 && channels != 3))
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_pipeline_host: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    const int C = ctx->cfg.n_cam, RM = ctx->cfg.max_roots;
    const size_t set_bytes = (size_t)C * ctx->cfg.width * ctx->cfg.height * channels;
    int chunk = (int)((size_t)(256u << 20) / set_bytes);      // ~256 MB per staging buffer
    if (chunk < 1) chunk = 1;
    if (chunk > n_frame_sets) chunk = n_frame_sets > 0 ? n_frame_sets : 1;
    const size_t need = (size_t)chunk * set_bytes;
    int st = grow_carved(ctx, ctx->stage, Drain::device, [&](Layout& L) {   // the copy streams use them too
        for (int k = 0; k < 2; ++k) ctx->d_stage[k] = L.take<uint8_t>(need);
    });
    if (st) return st;
    st = ensure_sets(ctx, n_frame_sets);
    if (st) return st;
    cudaEvent_t* copied = ctx->copied;
    // the copies must not start before earlier work on the caller's stream has finished with the staging buffers
    CUDA_TRY(ctx, cudaEventRecord(copied[0], ctx->stream));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->copy_stream, copied[0], 0));
    CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->copy_stream2, copied[0], 0));
    const bool fused = pick_fused(ctx);
    const SetOut out{ctx->d_obj, ctx->d_err, ctx->d_nobj, ctx->d_setflags, nullptr};
    int k = 0, n_chunks = 0;
    for (int s0 = 0; s0 < n_frame_sets; s0 += chunk, k ^= 1, ++n_chunks) {
        const int ns = (n_frame_sets - s0 < chunk) ? n_frame_sets - s0 : chunk;
        cudaStream_t cs = k ? ctx->copy_stream2 : ctx->copy_stream;
        if (n_chunks >= 2) CUDA_TRY(ctx, cudaStreamWaitEvent(cs, ctx->stage_free[k], 0));
        CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_stage[k], frames + (size_t)s0 * set_bytes, (size_t)ns * set_bytes,
                                      cudaMemcpyHostToDevice, cs));
        CUDA_TRY(ctx, cudaEventRecord(copied[k], cs));
        CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->stream, copied[k], 0));
        if ((st = run_sets(ctx, ctx->d_stage[k], ns, channels, threshold, fused, out.at(ctx->cfg, s0), ctx->stage_free[k])) != MOCAP_OK)
            return st;
    }
    const size_t n = (size_t)n_frame_sets;
    CUDA_TRY(ctx, cudaMemcpyAsync(obj, ctx->d_obj, n * RM * 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(err, ctx->d_err, n * RM * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(n_obj, ctx->d_nobj, n * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (set_flags) CUDA_TRY(ctx, cudaMemcpyAsync(set_flags, ctx->d_setflags, n * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return MOCAP_OK;
}

int mocap_locate_objects_dev(mocap_ctx* ctx, const double* obj, const double* err, const int32_t* n_obj, int n_frame_sets,
                             int max_objects, double* objects, int32_t* drone_index, int32_t* n_objects) {
    if (!ctx) return MOCAP_EINVAL;
    if (!obj || !err || !n_obj || !objects || !drone_index || !n_objects || n_frame_sets < 0 || max_objects < 1)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_locate_objects_dev: bad argument");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return launch_locate(ctx, obj, err, n_obj, n_frame_sets, max_objects, objects, drone_index, n_objects);
}

// ---- S3 on explicit correspondences ----------------------------------------------------------
int mocap_triangulate_dev(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                          double* X, double* err, uint8_t* valid) {
    if (!ctx) return MOCAP_EINVAL;
    if (!obs || !mask || !X || n_points < 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_triangulate_dev: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return launch_triangulate(ctx, obs, mask, n_points, nullptr, X, err, valid);
}

static int tri_host_common(mocap_ctx* ctx, const double* obs, const uint8_t* mask, const double* X_in, int n_points,
                           double* X, double* err, uint8_t* valid) {
    if (!ctx) return MOCAP_EINVAL;
    if (!obs || !mask || n_points < 0) return mocap_fail(ctx, MOCAP_EINVAL, "triangulate: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    if (n_points == 0) return MOCAP_OK;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    const int C = ctx->cfg.n_cam;
    const size_t n = (size_t)n_points;
    const size_t b_obs = n * C * 2 * sizeof(double), b_X = n * 3 * sizeof(double), b_err = n * sizeof(double);
    double *d_obs, *d_X, *d_Xin, *d_err;
    uint8_t *d_mask, *d_valid;
    int st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
        d_obs = L.take<double>(n * C * 2); d_X = L.take<double>(n * 3); d_Xin = L.take<double>(n * 3);
        d_err = L.take<double>(n); d_mask = L.take<uint8_t>(n * C); d_valid = L.take<uint8_t>(n);
    });
    if (st) return st;
    CUDA_TRY(ctx, cudaMemcpyAsync(d_obs, obs, b_obs, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_mask, mask, n * C, cudaMemcpyHostToDevice, ctx->stream));
    if (X_in) CUDA_TRY(ctx, cudaMemcpyAsync(d_Xin, X_in, b_X, cudaMemcpyHostToDevice, ctx->stream));
    st = launch_triangulate(ctx, d_obs, d_mask, n_points, X_in ? d_Xin : nullptr, d_X, d_err, d_valid);
    if (st) return st;
    if (X) CUDA_TRY(ctx, cudaMemcpyAsync(X, d_X, b_X, cudaMemcpyDeviceToHost, ctx->stream));
    if (err) CUDA_TRY(ctx, cudaMemcpyAsync(err, d_err, b_err, cudaMemcpyDeviceToHost, ctx->stream));
    if (valid) CUDA_TRY(ctx, cudaMemcpyAsync(valid, d_valid, n, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    return MOCAP_OK;
}

int mocap_triangulate_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                           double* X, double* err, uint8_t* valid) {
    if (ctx && !X) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_triangulate_host: X is NULL");
    return tri_host_common(ctx, obs, mask, nullptr, n_points, X, err, valid);
}

int mocap_reprojection_errors_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, const double* X,
                                   int n_points, double* err, uint8_t* valid) {
    if (ctx && (!X || !err)) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_reprojection_errors_host: NULL argument");
    return tri_host_common(ctx, obs, mask, X, n_points, nullptr, err, valid);
}

// ---- misc ------------------------------------------------------------------------------------
int mocap_host_alloc(void** out, uint64_t bytes) {
    if (!out) return MOCAP_EINVAL;
    *out = nullptr;
    if (cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return MOCAP_ENOMEM; }
    return MOCAP_OK;
}
void mocap_host_free(void* p) { if (p) cudaFreeHost(p); }

uint64_t mocap_launch_count(const mocap_ctx* ctx) { return ctx ? ctx->launches : 0; }

int mocap_enable_kernel_timing(mocap_ctx* ctx, int on) {
    if (!ctx) return MOCAP_EINVAL;
    ctx->timing_on = on ? 1 : 0;
    return MOCAP_OK;
}
int mocap_detect_kernel_ms(mocap_ctx* ctx, int reset, double* avg_ms, int* n_launches) {
    if (!ctx) return MOCAP_EINVAL;
    const int st = timing_flush(ctx);
    if (st) return st;
    if (avg_ms) *avg_ms = ctx->detect_ms_n ? ctx->detect_ms_sum / ctx->detect_ms_n : 0.0;
    if (n_launches) *n_launches = ctx->detect_ms_n;
    if (reset) { ctx->detect_ms_sum = 0.0; ctx->detect_ms_n = 0; }
    return MOCAP_OK;
}

}  // extern "C"

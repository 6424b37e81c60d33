// SURVEY.md section 8(f) "next" #2: capture-side preprocessing, the step right before S1.
//
// Replaces the per-camera body of Cameras._camera_read (reference computer_code/api/helpers.py:70-82):
//   rot90 -> make_square (zero pad to a square + 8-row feather, helpers.py:507-523) -> cv.undistort ->
//   cv.GaussianBlur 9x9 (sigma 0) -> cv.filter2D with the 5x5 sharpening kernel -> cvtColor RGB2BGR
// as ONE kernel per batch of frames: every CTA produces a 64x64 output tile and keeps all
// intermediates in shared memory, so a raw frame is read once and the processed frame written once
// (the reference makes five full passes over every frame on the CPU).
//
// Every stage follows OpenCV's 8-bit arithmetic exactly (each verified bit-for-bit against cv2 4.13):
//   undistort   initUndistortRectifyMap in double -> fixed-point map (1/32 px) -> bilinear remap with
//               integer weights (32-fx)(32-fy)*32 ... summing to 2^15, (acc + 2^14) >> 15,
//               BORDER_CONSTANT 0.  The map is built once per session on the host.
//   GaussianBlur 9x9, sigma 0 -> sigma 1.7 -> the fixed-point kernel [4 13 30 51 60 51 30 13 4]/256,
//               separable, 16.16 accumulation, (acc + 2^15) >> 16, BORDER_REFLECT_101
//   filter2D    integer correlation with the 5x5 kernel, BORDER_REFLECT_101, saturate to [0, 255]
#include <vector>
#include "common.cuh"
#include "preproc_tile.cuh"

// undistortion map per camera: m1 int16 [S][S][2] integer source coordinates (x, y), read by the kernel as
//                            one 32-bit word per pixel;  m2 uint16 [S][S]   (fy << 5) | fx, the 1/32 px fractions
//
// One CTA = one 64x64 output tile (preproc_tile.cuh) of TWO consecutive frames of one camera: the gather decodes
// the camera's map once per pixel and applies it to both frames; then, frame by frame, the two blur passes
// channel by channel (the transposed Q8.8 plane holds one channel) and the 5x5 filter; stages separated by
// barriers.  45 KB of shared memory and 42 registers: 5 CTAs resident per SM, so one CTA's gather overlaps its
// neighbours' filter stages.  Measured alternatives (8000 frames 320x240x3): one frame per CTA, 28 KB, 8 CTAs:
// -9 %; blur of all three channels at once, 48 KB, 4 CTAs: -14 %; 64x32 tiles with 2 / 3 / 4 frames: -12 / -8 / -16 %.
// blockIdx.z = frame group * C + camera; frame k of the group is image ((group * PP_F + k) * C + camera): the
// PP_F frames a CTA handles belong to ONE camera, so the gather decodes that camera's map once per pixel.
__global__ void __launch_bounds__(256)
k_preprocess(const uint8_t* __restrict__ raw_frames, int n_images, int C, int in_w, int in_h, int S, const int* __restrict__ rotation,
             const int32_t* __restrict__ m1, const uint16_t* __restrict__ m2, uint8_t* __restrict__ out, uint8_t* __restrict__ gray,
             int word_stores) {
    __shared__ __align__(16) uint8_t smem[PP_SMEM_BYTES];
    uint8_t* U = smem;                                                  // PP_F frames; G of a frame reuses its U
    uint32_t* GhT = reinterpret_cast<uint32_t*>(smem + PP_F * PP_U_BYTES);
    const int cam = blockIdx.z % C, group = blockIdx.z / C;
    const int x0 = blockIdx.x * PP_TX, y0 = blockIdx.y * PP_TY;
    PPFrame f;
    f.n_frames = 0;
#pragma unroll
    for (int k = 0; k < PP_F; ++k) {
        const long long img = (long long)(group * PP_F + k) * C + cam;
        const bool in = img < n_images;
        f.raw[k] = in ? raw_frames + (size_t)img * in_w * in_h * 3 : nullptr;
        f.out[k] = (in && out) ? out + (size_t)img * S * S * 3 : nullptr;
        f.gray[k] = (in && gray) ? gray + (size_t)img * S * S : nullptr;
        f.n_frames += in ? 1 : 0;
    }
    f.m1 = m1; f.m2 = m2; f.map_offset = cam * S * S;
    f.in_w = in_w; f.in_h = in_h; f.S = S; f.rot = rotation[cam]; f.ay = (S - in_h) / 2;
    f.word_stores = word_stores;
    // the thread index is made opaque: knowing it is below 1024 the compiler narrows the item arithmetic of
    // the stages to 16 bits, which costs more mask/extend instructions than it saves
    int tid = threadIdx.x;
    asm volatile("" : "+r"(tid));
    const int nt = 256;
    pp_stage_undistort(f, U, x0, y0, tid, nt);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PP_F; ++k) {
        if (k >= f.n_frames) break;
        uint8_t* Uk = U + k * PP_U_BYTES;                               // G over U (dead after the horizontal pass)
        for (int c0 = 0; c0 < 3; c0 += PP_GHT_CH) {
            pp_stage_blur_h(Uk, GhT, c0, tid, nt);
            __syncthreads();
            pp_stage_blur_v(GhT, Uk, c0, tid, nt);
            __syncthreads();
        }
        pp_stage_sharpen_store(f, k, Uk, x0, y0, tid, nt);              // the next frame's horizontal pass may start
    }                                                                   // meanwhile: it writes GhT, reads its own U
}

// cv.initUndistortRectifyMap(K, dist, I, K, (S, S), CV_16SC2): per output pixel the source position
// in 1/32 px (double arithmetic, round half to even).  dist = k1 k2 p1 p2 k3.
static void build_undistort_map(const double* K, const double* dist, int S, int16_t* m1, uint16_t* m2) {
    const double fx = K[0], fy = K[4], u0 = K[2], v0 = K[5];
    const double k1 = dist[0], k2 = dist[1], p1 = dist[2], p2 = dist[3], k3 = dist[4];
    // inverse of the (upper triangular) new camera matrix
    const double ir0 = 1.0 / fx, ir1 = -K[1] / (fx * fy), ir2 = (K[1] * v0 - u0 * fy) / (fx * fy);
    const double ir4 = 1.0 / fy, ir5 = -v0 / fy;
    for (int i = 0; i < S; ++i) {
        const double xr = i * ir1 + ir2, yr = i * ir4 + ir5;
        for (int j = 0; j < S; ++j) {
            const double x = xr + j * ir0, y = yr;
            const double x2 = x * x, y2 = y * y, r2 = x2 + y2, _2xy = 2 * x * y;
            const double kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / 1.0;
            const double xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2);
            const double yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy;
            const double u = fx * xd + u0, v = fy * yd + v0;
            const long iu = lrint(u * 32.0), iv = lrint(v * 32.0);
            long qx = iu >> 5, qy = iv >> 5;
            if (qx < -32768) qx = -32768; if (qx > 32767) qx = 32767;
            if (qy < -32768) qy = -32768; if (qy > 32767) qy = 32767;
            m1[((size_t)i * S + j) * 2] = (int16_t)qx;
            m1[((size_t)i * S + j) * 2 + 1] = (int16_t)qy;
            m2[(size_t)i * S + j] = (uint16_t)(((iv & 31) << 5) | (iu & 31));
        }
    }
}

// processed frames and/or the grayscale plane S1 derives from them
static int launch_preprocess(mocap_ctx* ctx, const uint8_t* raw_frames, int n_images, uint8_t* out_frames, uint8_t* gray) {
    const int S = ctx->cfg.width, C = ctx->cfg.n_cam;
    const int groups_per_launch = 65535 / C > 0 ? 65535 / C : 1;           // gridDim.z <= 65535
    const int per_launch = groups_per_launch * PP_F * C;                    // whole frame-sets, whole groups
    for (int i0 = 0; i0 < n_images; i0 += per_launch) {
        const int n = n_images - i0 < per_launch ? n_images - i0 : per_launch;
        const int sets = (n + C - 1) / C, groups = (sets + PP_F - 1) / PP_F;
        uint8_t* o = out_frames ? out_frames + (size_t)i0 * S * S * 3 : nullptr;
        uint8_t* g = gray ? gray + (size_t)i0 * S * S : nullptr;
        const int word_stores = (S % 4 == 0) && (reinterpret_cast<uintptr_t>(o) % 4 == 0) && (reinterpret_cast<uintptr_t>(g) % 4 == 0);
        k_preprocess<<<dim3((S + PP_TX - 1) / PP_TX, (S + PP_TY - 1) / PP_TY, groups * C), 256, 0, ctx->stream>>>(
            raw_frames + (size_t)i0 * ctx->pp_in_w * ctx->pp_in_h * 3, n, C, ctx->pp_in_w, ctx->pp_in_h, S, ctx->pp_rot.as<int>(),
            ctx->pp_m1.as<const int32_t>(), ctx->pp_m2.as<uint16_t>(), o, g, word_stores);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
    }
    return MOCAP_OK;
}

// The launch-group loop of the raw-frame entry points (mocap_pipeline_raw_dev, mocap_live_dev).  The preprocessing
// kernel also emits the grayscale plane _find_dot would derive from the processed frame (helpers.py:144), so S1-S3 run
// on 1 byte per pixel through the single-pass pipeline kernel; the processed BGR frames are only written when the
// caller asks for them.  stages: RAW_PREPROCESS, RAW_DETECT (+ S1, blob lists left in the context's d_blob_xy /
// d_blob_n / d_img_flags) or RAW_MATCH (+ S2+S3 into obj / err / n_obj / set_flags, the blob lists left as well).
// live != NULL: k_live_blobs after each group's S1 (live.cu), and the detection overlay (overlay.cu) when the context
// draws it.
int run_raw_groups(mocap_ctx* ctx, const uint8_t* raw_frames, int n_frame_sets, int threshold, int stages, uint8_t* processed,
                   double* obj, double* err, int32_t* n_obj, int32_t* set_flags, const LiveOut* live) {
    const int C = ctx->cfg.n_cam, S = ctx->cfg.width;
    const size_t gray_bytes = (size_t)S * S;
    const int chunk = 4096 / C > 0 ? 4096 / C : 1;             // frame-sets per launch group (bounded scratch)
    // the grey plane stays in the scratch through S1-S3, k_live_blobs and the overlay: none of them uses the scratch
    uint8_t* gray;
    int st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) { gray = L.take<uint8_t>((size_t)chunk * C * gray_bytes); });
    if (st) return st;
    if (stages == RAW_DETECT && (st = ensure_images(ctx, (n_frame_sets < chunk ? n_frame_sets : chunk) * C)) != MOCAP_OK) return st;
    for (int s0 = 0; s0 < n_frame_sets; s0 += chunk) {
        const int ns = n_frame_sets - s0 < chunk ? n_frame_sets - s0 : chunk;
        uint8_t* out = processed ? processed + (size_t)s0 * C * gray_bytes * 3 : nullptr;
        st = launch_preprocess(ctx, raw_frames + (size_t)s0 * C * ctx->pp_in_w * ctx->pp_in_h * 3, ns * C, out,
                               stages == RAW_PREPROCESS ? nullptr : gray);
        if (st) return st;
        if (stages == RAW_MATCH)
            st = mocap_pipeline_dev(ctx, gray, ns, 1, threshold, obj + (size_t)s0 * ctx->cfg.max_roots * 3, err + (size_t)s0 * ctx->cfg.max_roots,
                                    n_obj + s0, set_flags ? set_flags + s0 : nullptr);
        else if (stages == RAW_DETECT)
            st = launch_detect(ctx, gray, ns * C, 1, threshold, ctx->d_blob_xy, ctx->d_blob_n, nullptr, ctx->d_img_flags);
        if (st) return st;
        if (live && (st = launch_live_blobs(ctx, *live, s0, ns, stages != RAW_PREPROCESS, out)) != MOCAP_OK) return st;
        // the overlay over k_live_blobs's dots, while this group's grey plane is still in the scratch
        if (live && ctx->overlay_on && out && (live->mode & MOCAP_LIVE_CAPTURE)) {
            if ((st = launch_overlay(ctx, gray, out, ns * C, ctx->d_blob_xy, ctx->d_blob_n)) != MOCAP_OK) return st;
            if ((live->mode & MOCAP_LIVE_TRIANGULATE) && (st = launch_epilines(ctx, out, ns, ctx->d_blob_xy, ctx->d_blob_n)) != MOCAP_OK)
                return st;
        }
    }
    return MOCAP_OK;
}

extern "C" {

int mocap_set_preprocess(mocap_ctx* ctx, int in_width, int in_height, const int* rotation, const double* K, const double* dist) {
    if (!ctx) return MOCAP_EINVAL;
    const int C = ctx->cfg.n_cam, S = ctx->cfg.width;
    if ((long long)C * S * S >= (1ll << 31) || (long long)in_width * in_height * 3 >= (1ll << 31))
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_set_preprocess: frames too large for 32-bit pixel indices");
    if (!rotation || !K || !dist || ctx->cfg.height != S || in_width != S || in_height > S - 16 || in_height < 1)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_set_preprocess: the context must be square (width == height == raw width) and the raw frame "
                                             "landscape with at least 8 pad rows above and below (the reference's make_square only works for that)");
    for (int c = 0; c < C; ++c)
        if (rotation[c] != 0 && rotation[c] != 2)
            return mocap_fail(ctx, MOCAP_EINVAL, "mocap_set_preprocess: rotation must be 0 or 2 (a quarter turn makes the frame portrait, which make_square cannot feather)");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    std::vector<int16_t> m1((size_t)C * S * S * 2);
    std::vector<uint16_t> m2((size_t)C * S * S);
    for (int c = 0; c < C; ++c) build_undistort_map(K + 9 * c, dist + 5 * c, S, m1.data() + (size_t)c * S * S * 2, m2.data() + (size_t)c * S * S);
    CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    // unset until all three maps are on the device, and unset with no maps if any step fails
    ctx->pp_in_w = ctx->pp_in_h = 0;
    ctx->pp_m1.reset(); ctx->pp_m2.reset(); ctx->pp_rot.reset();
    const void* host[3] = {m1.data(), m2.data(), rotation};
    const size_t bytes[3] = {m1.size() * sizeof(int16_t), m2.size() * sizeof(uint16_t), C * sizeof(int)};
    DeviceBuffer* maps[3] = {&ctx->pp_m1, &ctx->pp_m2, &ctx->pp_rot};
    for (int k = 0; k < 3; ++k) {
        int st = maps[k]->grow(ctx, bytes[k], Drain::none);
        if (!st && cudaMemcpy(maps[k]->get(), host[k], bytes[k], cudaMemcpyHostToDevice) != cudaSuccess)
            st = mocap_fail(ctx, MOCAP_ECUDA, "mocap_set_preprocess: cudaMemcpy failed: %s", cudaGetErrorString(cudaGetLastError()));
        if (st) { for (DeviceBuffer* m : maps) m->reset(); return st; }
    }
    ctx->pp_in_w = in_width; ctx->pp_in_h = in_height;
    return MOCAP_OK;
}

int mocap_get_undistort_map(mocap_ctx* ctx, int cam, int16_t* m1, uint16_t* m2) {
    if (!ctx) return MOCAP_EINVAL;
    const int S = ctx->cfg.width;
    if (!ctx->pp_in_w || cam < 0 || cam >= ctx->cfg.n_cam || !m1 || !m2) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_get_undistort_map: no preprocessing set / bad argument");
    CUDA_TRY(ctx, cudaMemcpy(m1, ctx->pp_m1.as<int16_t>() + (size_t)cam * S * S * 2, (size_t)S * S * 2 * sizeof(int16_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(ctx, cudaMemcpy(m2, ctx->pp_m2.as<uint16_t>() + (size_t)cam * S * S, (size_t)S * S * sizeof(uint16_t), cudaMemcpyDeviceToHost));
    return MOCAP_OK;
}

int mocap_preprocess_dev(mocap_ctx* ctx, const uint8_t* raw_frames, int n_images, uint8_t* out_frames) {
    if (!ctx) return MOCAP_EINVAL;
    if (!raw_frames || !out_frames || n_images < 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_preprocess_dev: bad argument");
    if (!ctx->pp_in_w) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_preprocess has not been called");
    if (n_images == 0) return MOCAP_OK;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return launch_preprocess(ctx, raw_frames, n_images, out_frames, nullptr);
}

int mocap_pipeline_raw_dev(mocap_ctx* ctx, const uint8_t* raw_frames, int n_frame_sets, int threshold, uint8_t* processed,
                           double* obj, double* err, int32_t* n_obj, int32_t* set_flags) {
    if (!ctx) return MOCAP_EINVAL;
    if (!raw_frames || !obj || !err || !n_obj || n_frame_sets < 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_pipeline_raw_dev: bad argument");
    if (!ctx->pp_in_w) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_preprocess has not been called");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called");
    if (n_frame_sets == 0) return MOCAP_OK;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    return run_raw_groups(ctx, raw_frames, n_frame_sets, threshold, RAW_MATCH, processed, obj, err, n_obj, set_flags, nullptr);
}

}  // extern "C"

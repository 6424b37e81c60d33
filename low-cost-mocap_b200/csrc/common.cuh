// Shared declarations of libmocap_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <vector>
#include "../../include/mocap_b200.h"
#include "ctx_memory.h"

#define MOCAP_MAX_CAM        16
#define MOCAP_MAX_BLOBS      64
#define MOCAP_MAX_ROOTS      128
#define MOCAP_MAX_CANDS      16
#define MOCAP_ACC_CAP        256     // blobs accumulated per image before max_blobs truncation
#define MOCAP_SEG_PX         16      // pixels per threshold segment (one 128-bit load of 1-channel data)

// Camera tables, device resident (built on the host by mocap_set_cameras).
struct CameraTables {
    double Pkc[MOCAP_MAX_CAM][MOCAP_MAX_CAM][12];  // Pkc[k][c] = K_k [R_c|t_c]  (helpers.py:305-308 uses K of the k-th PRESENT view)
    double F[MOCAP_MAX_CAM][MOCAP_MAX_CAM][9];     // F[r][c]: line in camera c of a point in camera r (helpers.py:362)
    double R[MOCAP_MAX_CAM][9];
    double t[MOCAP_MAX_CAM][3];
    double fx[MOCAP_MAX_CAM], fy[MOCAP_MAX_CAM], cx[MOCAP_MAX_CAM], cy[MOCAP_MAX_CAM];  // cv.projectPoints reads these four of K
    double Kmat[MOCAP_MAX_CAM][9];                 // full intrinsics (S4 rebuilds K_k [R|t] for trial poses)
    double world[16];                              // to_world_coords_matrix (helpers.py:99)
    int    use_world;
    int    n_cam;
};

struct mocap_ctx {
    mocap_config cfg;
    cudaStream_t stream;
    cudaStream_t copy_stream;
    cudaStream_t copy_stream2;   // staging buffers alternate between two copy streams (two copy engines in flight)
    char         err[512];
    bool         cameras_set;
    DeviceBuffer  tables; CameraTables* d_tables;      // d_tables = tables
    CameraTables  h_tables;
    // detection scratch, sized for cap_images; the first four regions are self-resetting counters, zeroed when it grows
    DeviceBuffer images;
    int       cap_images;
    uint32_t* d_seg_count;
    uint32_t* d_work_count;   // [4]: image worklist count + finished-CTA counter, set worklist count + finished-CTA counter
    uint32_t* d_img_done;     // fused kernel: finished units per image (self-resetting)
    uint32_t* d_set_done;     // fused kernel: [2*cap_images] finished images per set, then deferred marks
    uint32_t* d_seg_list;
    uint32_t* d_worklist;     // images deferred by the warp-level blob kernel
    uint32_t* d_set_worklist; // frame-sets deferred by the fused kernel
    unsigned long long* d_unit_counter;
    int32_t*  d_blob_xy;
    int32_t*  d_blob_n;
    int32_t*  d_img_flags;
    int       fused_ctas_per_sm;
    int       pipeline_auto;     // MOCAP_PIPELINE unset: heavy batches (many blobs per frame-set) take the three-kernel pipeline
    DeviceBuffer stat_acc;                           // device accumulator of the blob statistic
    PinnedBuffer stat_host;                          // mapped: {blobs, images} of the last batch, written by the GPU
    unsigned long long* d_stat_host;                 // device alias of stat_host
    int       use_fused;      // 1: single fused pipeline kernel for 1-channel frames (default)
    DeviceBuffer hole_win;    // mocap_set_large_holes: the whole-image windows of k_blob_reduce's CTAs; empty = off
    int       overlay_on;       // mocap_set_overlay: the live entry points draw the detection overlay (overlay.cu)
    DeviceBuffer palette; int palette_len;         // the epipolar lines' colours [palette_len][3]
    DeviceBuffer line_counter;                     // epipolar lines drawn since mocap_set_overlay
    DeviceBuffer line_counts;                      // lines per frame-set of a launch group
    // host-path staging: both buffers in one allocation
    DeviceBuffer stage;
    uint8_t*  d_stage[2];
    cudaEvent_t stage_free[2]; cudaEvent_t copied[2];   // per staging buffer: its kernel has finished / its copy has landed
    DeviceBuffer sets;
    double*   d_obj; double* d_err; int32_t* d_nobj; int32_t* d_setflags;
    int       cap_sets;
    // Generic scratch of the *_host entry points, the calibration and the grey planes of the raw-frame chain.  A
    // function that holds pointers carved from it must not call another user of it: that call may grow it (the
    // pointers dangle) or overwrite it.
    DeviceBuffer scratch;
    // S4 on the device (ba_dev.cu): workspace of k_ba_solve, launch shape
    DeviceBuffer ba_ws; int ba_threads; int ba_grid; size_t ba_smem;
    DeviceBuffer match_counter; int match_ctas_per_sm;  // k_match_triangulate: claim counters [4], resident CTAs per SM
    // chunked matcher (match_device.cuh MatchSplit): arrivals per frame-set (zeroed when it grows), items, their partial
    // results, the roots each touches
    DeviceBuffer match_split;
    unsigned* d_match_arrive; void* d_match_items; unsigned long long* d_match_partial; int* d_match_range;
    int match_chunk, match_item_cap, match_cap_sets;
    // capture-side preprocessing (SURVEY 8(f) #2); pp_in_w != 0 once mocap_set_preprocess has put all three maps on the device
    DeviceBuffer pp_m1, pp_m2, pp_rot; int pp_in_w, pp_in_h;
    // mocap_live_host staging: device and page-locked host buffers of {timestamps, raw frames} and {result, frames}
    DeviceBuffer live_in, live_out;
    PinnedBuffer live_in_host, live_out_host;
    // JPEG encoder (jpeg.cu): device tables + header per (width, height, quality), scratch of a group of images, and
    // mocap_live_jpeg_host's device output and page-locked staging
    DeviceBuffer jpeg_cfg[16]; int jpeg_cfg_key[16][3]; int jpeg_cfg_n;
    DeviceBuffer jpeg_scratch, jpeg_out;
    PinnedBuffer jpeg_host;
    // accounting
    uint64_t  launches;
    int       timing_on;
    cudaEvent_t tim_ev[2 * 64];   // pairs bracketing k_threshold_segments, resolved lazily
    int       tim_used;
    double    detect_ms_sum;
    int       detect_ms_n;
    int       num_sms;
};

int mocap_fail(mocap_ctx* ctx, int code, const char* fmt, ...);
#define CUDA_TRY(ctx, call)                                                              \
    do {                                                                                 \
        cudaError_t e__ = (call);                                                        \
        if (e__ != cudaSuccess)                                                          \
            return mocap_fail((ctx), MOCAP_ECUDA, "%s failed: %s (%s:%d)", #call,        \
                              cudaGetErrorString(e__), __FILE__, __LINE__);              \
    } while (0)

// What S2+S3 write per frame-set: obj [n][max_roots][3], err [n][max_roots], n [n], flags [n] (may be null) and the
// winners' pixels track_xy [n][max_roots][n_cam][2] (may be null).  at(): the same record from frame-set s0 on.
struct SetOut {
    double* obj; double* err; int32_t* n; int32_t* flags; int32_t* track_xy;
    SetOut at(const mocap_config& c, int s0) const {
        const size_t s = (size_t)s0, R = (size_t)c.max_roots;
        return {obj + s * R * 3, err + s * R, n + s, flags ? flags + s : nullptr, track_xy ? track_xy + s * R * c.n_cam * 2 : nullptr};
    }
};

// kernel launchers (each returns a MOCAP_* status; all enqueue on ctx->stream)
int launch_detect(mocap_ctx* ctx, const uint8_t* frames, int n_images, int channels, int threshold,
                  int32_t* blob_xy, int32_t* blob_n, int64_t* blob_mom, int32_t* img_flags);
// img_flags (may be null): the images' S1 flags, folded into each frame-set's flags; chosen (may be null)
int launch_match(mocap_ctx* ctx, const int32_t* blob_xy, const int32_t* blob_n, int n_sets, const SetOut& out,
                 const int32_t* img_flags, int32_t* chosen);
int launch_triangulate(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                       const double* X_in, double* X, double* err, uint8_t* valid);
int ensure_images(mocap_ctx* ctx, int n_images);
// the live loop's per-read outputs k_live_blobs writes (slices of the mocap_live_dev result, indexed by read)
struct LiveOut {
    int32_t* flags; uint8_t* gate; int32_t* blob_n; int32_t* first; uint8_t* called;
    int mode;                   // MOCAP_LIVE_* bits
};
int launch_live_blobs(mocap_ctx* ctx, const LiveOut& live, int s0, int n_sets, int have_blobs, uint8_t* frames);
// the detection overlay of n_images frames of the context's size from their grey planes and blob lists, and the
// matcher's epipolar lines into n_sets frame-sets of them (overlay.cu)
int launch_overlay(mocap_ctx* ctx, const uint8_t* gray, uint8_t* frames, int n_images, const int32_t* blob_xy, const int32_t* blob_n);
int launch_epilines(mocap_ctx* ctx, uint8_t* frames, int n_sets, const int32_t* blob_xy, const int32_t* blob_n);
// mocap_live_host in two halves (live.cu), so that mocap_live_jpeg_host runs the same chain: live_check; live_host_run
// (staging in, the chain; the frames stay on the device when keep_frames); live_host_finish (result, frames and
// extra_bytes of device data back, one synchronisation).  frame_off, extra_off: where the frames and the extra bytes
// sit in the output staging (the result is at 0).
struct LiveHostRun {
    mocap_live_offsets L;
    size_t frame_copy, extra_bytes, frame_off, extra_off;
    uint8_t* d_frames;
};
int live_check(mocap_ctx* ctx, mocap_tracker* tr, const void* raw, int n_reads, int mode, const double* timestamps,
               const void* result, const char* who);
int live_host_run(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode, const double* timestamps,
                  int keep_frames, size_t extra_bytes, LiveHostRun* run);
int live_host_finish(mocap_ctx* ctx, const LiveHostRun& run, uint8_t* frames, void* result, const void* extra, void* extra_out);
// the JPEG encoder (jpeg.cu): mocap_encode_jpeg_dev after its checks
int jpeg_encode(mocap_ctx* ctx, const uint8_t* images, int n_images, int tiles, int tile_w, int tile_h, int quality,
                uint8_t* out, uint64_t out_stride, int32_t* out_len);
#define MOCAP_JPEG_CONFIGS 16                     // (width, height, quality) configurations cached per context
#define JPEG_CONFIG_BYTES  3200                   // JpegTables + the header, padded (jpeg.cuh)
// raw frames -> preprocessing [-> S1 [-> S2+S3]] per launch group (preproc.cu)
enum { RAW_PREPROCESS = 0, RAW_DETECT = 1, RAW_MATCH = 2 };
int run_raw_groups(mocap_ctx* ctx, const uint8_t* raw_frames, int n_frame_sets, int threshold, int stages, uint8_t* processed,
                   double* obj, double* err, int32_t* n_obj, int32_t* set_flags, const LiveOut* live);
// the context and drone count of a tracker (track.cu)
mocap_ctx* tracker_context(const mocap_tracker* tr);
int tracker_num_objects(const mocap_tracker* tr);
int launch_locate(mocap_ctx* ctx, const double* obj, const double* err, const int32_t* n_obj, int n_sets,
                  int max_objects, double* out, int32_t* drone_index, int32_t* n_out);
int launch_blob_fallback(mocap_ctx* ctx, int32_t* blob_xy, int32_t* blob_n, int64_t* blob_mom, int32_t* img_flags, int n_images);
int blob_set_large_holes(mocap_ctx* ctx, int on);
// frame-sets with more blobs than this (average of the previous batch) are cheaper through the three-kernel
// pipeline: the matcher's large code then runs in a kernel of its own instead of evicting the stream loop
#define MOCAP_HEAVY_BLOBS_PER_SET 48
// candidate groups per work item of the chunked matcher: frame-sets with more are evaluated by several warps
#define MOCAP_MATCH_CHUNK 512
int launch_match_list(mocap_ctx* ctx, const int32_t* blob_xy, const int32_t* blob_n, const uint32_t* set_list, uint32_t* set_count,
                      int n_sets_max, const SetOut& out, const int32_t* img_flags);
int launch_pipeline_fused(mocap_ctx* ctx, const uint8_t* frames, int n_sets, int channels, int threshold, const SetOut& out);
// S1-S3 of n_sets frame-sets through the single-pass kernel (fused) or the three-kernel pipeline, launch group by
// launch group; frames_read (may be null) is recorded after the last launch that reads a group's frames (api.cu)
int run_sets(mocap_ctx* ctx, const uint8_t* frames, int n_sets, int channels, int threshold, bool fused, const SetOut& out,
             cudaEvent_t frames_read);
bool pick_fused(const mocap_ctx* ctx);
// the S1 launchers' shared pieces: the moment sums of a frame this size may exceed 32 bits (the kernels' WIDE variant);
// mocap_enable_kernel_timing's event pair around the stream kernel (no-ops while timing is off); the pairs' read-out
inline bool moments_wide(const mocap_config& c) {
    const long long mx = c.width > c.height ? c.width : c.height;
    return 6ll * mx * c.width * c.height >= (1ll << 32);
}
int timing_begin(mocap_ctx* ctx);
int timing_end(mocap_ctx* ctx);
int timing_flush(mocap_ctx* ctx);
// The cold-start calibration's pair table (calib_ransac.cu): for camera pairs (a[k], b[k]) their common observations
// {x_a, y_a, x_b, y_b} in frame order, cast to float32 as the reference casts them (index.py:243-244), pair k at
// [off[k], off[k+1]).  adjacent_pairs: the chain's table, pairs (c, c+1), failing with MOCAP_EINVAL where a pair has
// fewer than 8 common observations.  scatter_pairs: a mask over the table -> out [n_points][P], 0 where a frame is not
// common to the pair.
struct PairTable {
    std::vector<int> a, b;
    std::vector<float4> pts;
    std::vector<int> off;
    int pairs() const { return (int)a.size(); }
    int count(int k) const { return off[k + 1] - off[k]; }
    int max_count() const { int x = 0; for (int k = 0; k < pairs(); ++k) x = count(k) > x ? count(k) : x; return x; }
};
PairTable pair_table(const double* obs, const uint8_t* mask, int n_points, int C, const std::vector<int>& a, const std::vector<int>& b);
int adjacent_pairs(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points, const char* who, PairTable& tab);
void scatter_pairs(const PairTable& tab, const uint8_t* mask, int n_points, int C, const uint8_t* sel, uint8_t* out);
// cold-start pose chain over the adjacent table (calib_init.cu): per pair an 8-point F started from init_inl (over the
// table; NULL = all common observations) and re-fitted on its Sampson inliers at thr2, E, the cheirality vote and the
// chain; inl_out (may be NULL) [n_points][C-1] the final Sampson sets
int calibrate_chain(mocap_ctx* ctx, const PairTable& tab, const uint8_t* mask, int n_points, const double* F_given,
                    const uint8_t* init_inl, double thr2, double* R, double* t, double* F_used, int* votes, uint8_t* inl_out);
// RANSAC fundamental matrices over a pair table (calib_ransac.cu).  ransac_check_options fills o (opt NULL = defaults) or
// fails with MOCAP_EINVAL.  ransac_run: pair p's samples are drawn from the hash of (seed, p, ...).  Out: F_best [P][9],
// inl over the table, keys [P] (0: no sample of that pair gave a model).  Three launches, one synchronisation.
// Scratch: dominated by P * hypotheses * 27 doubles of models.
int ransac_check_options(mocap_ctx* ctx, const mocap_ransac_options* opt, mocap_ransac_options* o, const char* who);
int ransac_run(mocap_ctx* ctx, const PairTable& tab, const mocap_ransac_options& o, double* F_best, uint8_t* inl, unsigned long long* keys);
// The 8-point re-fits of every pair of a table at once (calib_graph.cu).  PairDev: the table on the device and the
// stages' buffers, carved by take(); the caller copies pts and off up.  fit_pairs: per pair the Hartley transform of
// its fit set inl (host, over the table), k_epipolar_normal_pairs, calib_pose::fit_from_normal; F [P][9] (host) is
// overwritten where ok[p] = 1 and left where the eigen problem fails.  select_pairs: k_sampson_pairs under F at thr2,
// the selection sel (host, over the table) out.  One launch and one synchronisation each.
struct PairDev {
    float4* pts; int* off; uint8_t* inl; double *T, *n45, *F;
    void take(Layout& L, const PairTable& tab) {
        const size_t P = tab.pairs(), total = tab.pts.size();
        pts = L.take<float4>(total); off = L.take<int>(P + 1); inl = L.take<uint8_t>(total);
        T = L.take<double>(P * 6); n45 = L.take<double>(P * 45); F = L.take<double>(P * 9);
    }
};
int fit_pairs(mocap_ctx* ctx, const PairTable& tab, const PairDev& d, const uint8_t* inl, double* F, uint8_t* ok);
int select_pairs(mocap_ctx* ctx, const PairTable& tab, const PairDev& d, const double* F, double thr2, uint8_t* sel);

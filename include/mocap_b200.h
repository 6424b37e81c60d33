/*
 * mocap_b200.h -- C ABI of libmocap_b200.so: the H100 (sm_90a) multi-view
 * marker-tracking core that stands in for the per-frame geometry path of
 * jyjblrd/Low-Cost-Mocap, computer_code/api/helpers.py.
 *
 * The reference has no FFI of its own: its hot path is five module-level Python
 * functions.  Each entry point below names the reference function (file:line,
 * relative to the reference repository) it replaces; the Python mirror that
 * re-creates the reference signatures on top of this ABI lives in
 * low-cost-mocap_b200/api.py and the binding a maintainer adds is shown in
 * INTEGRATION.md.
 *
 * Conventions
 *   - plain C, plain pointers and sizes; no torch / numpy types.
 *   - every function returns MOCAP_OK (0) or a negative MOCAP_E* code;
 *     mocap_last_error(ctx) gives the text of the last failure of that ctx.
 *   - "_dev" entry points take DEVICE pointers and only enqueue work on the
 *     context's stream (mocap_set_stream); they never synchronise.
 *     "_host" entry points take HOST pointers, copy in/out and return when the
 *     results are in the host buffers.
 *   - one context per host thread (the reference's Cameras singleton is
 *     unsynchronised, Singleton.py:3); contexts are independent.  A context owns scratch
 *     (segment lists, counters, blob lists) shared by all of its calls: use it from ONE
 *     stream at a time -- before pointing it at another stream with mocap_set_stream, the
 *     work already enqueued through it must have finished or be ordered before the new
 *     stream's work (event).  The bundle-adjustment entry points use a workspace of their
 *     own and may run on a second stream next to the pipeline entry points.
 *   - there is no CPU fallback: without a CUDA device every call fails with
 *     MOCAP_ENODEV.
 *
 * Layouts (row-major, innermost last)
 *   frames      uint8  [n_frame_sets][n_cam][H][W]        (channels == 1)
 *               uint8  [n_frame_sets][n_cam][H][W][3]     (channels == 3, the
 *               layout Cameras._find_dot receives, helpers.py:143)
 *   blob_xy     int32  [n_images][max_blobs][2]   (x, y) = int(m10/m00), int(m01/m00)
 *   blob_n      int32  [n_images]                 n_images = n_frame_sets * n_cam
 *   blob_mom    int64  [n_images][max_blobs][4]   {2*m00, 6*m10, 6*m01, pixel count}; the pixel count of a
 *                                                 blob is its 8-connected area, that of a hole contour the size
 *                                                 of the region the hole encloses: its 4-connected component of
 *                                                 the complement of the blob around it, nested blobs included
 *   img_flags   int32  [n_images]                 MOCAP_F_* bits
 *   obj         double [n_frame_sets][max_roots][3]
 *   err         double [n_frame_sets][max_roots]  mean squared reprojection error, px^2
 *   n_obj       int32  [n_frame_sets]
 *   set_flags   int32  [n_frame_sets]             MOCAP_F_* bits
 *   chosen      int32  [n_frame_sets][max_roots][n_cam]  blob index per camera of the
 *                                                 winning correspondence, -1 = no view
 */
#ifndef MOCAP_B200_H
#define MOCAP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MOCAP_OK          0
#define MOCAP_EINVAL     -1   /* bad argument                                  */
#define MOCAP_ENODEV     -2   /* no usable CUDA device / wrong architecture    */
#define MOCAP_ECUDA      -3   /* a CUDA runtime call failed                    */
#define MOCAP_ENOMEM     -4
#define MOCAP_ESTATE     -5   /* e.g. cameras not set                          */

/* per-image / per-frame-set overflow flags (results for that unit are truncated) */
#define MOCAP_F_SEGMENTS  1   /* more above-threshold 16-px segments than max_segments */
#define MOCAP_F_BLOBS     2   /* more blobs than max_blobs                               */
#define MOCAP_F_ROOTS     4   /* more roots than max_roots                               */
#define MOCAP_F_CANDS     8   /* more than max_cands candidates on one epipolar line     */
#define MOCAP_F_GROUPS   16   /* more than max_groups candidate groups for one root      */
#define MOCAP_F_HOLES    32   /* per image, not an overflow.  Blobs with holes are reproduced as cv.findContours(RETR_TREE) +
                                 cv.moments treat them (helpers.py:147-158): one more contour -- one more point -- per hole, the
                                 outer contour's moments over the FILLED blob, cv2's hierarchy order.  The bit is left only
                                 when that slow path could not run.  By default: a holed blob wider or taller than 62
                                 pixels, or more than 64 holes in the image.  With mocap_set_large_holes(ctx, 1): more
                                 than 64 holes in the image only (a holed blob of any size is reproduced).  The image then
                                 carries, for every blob of it, holed or not, one centre and the moments of the polygon
                                 through its own set pixels, in descending raster order of the blob's first pixel, as an
                                 image without holes does. */

#if defined(__GNUC__)
#define MOCAP_API __attribute__((visibility("default")))
#else
#define MOCAP_API
#endif

typedef struct mocap_ctx mocap_ctx;

typedef struct mocap_config {
    int device;         /* CUDA device ordinal                                            */
    int n_cam;          /* cameras per frame-set (1..16)                                   */
    int width;          /* image width, multiple of 16 (640)                              */
    int height;         /* image height (480)                                             */
    int max_blobs;      /* blobs kept per image (<= 64)                                   */
    int max_segments;   /* above-threshold 16-px segments handled per image (power of two, 64..4096) */
    int max_roots;      /* roots per frame-set in the matcher (<= 128)                    */
    int max_cands;      /* candidates kept per (root, camera) (<= 16)                     */
    int max_groups;     /* candidate groups evaluated per root                            */
} mocap_config;

/* Fills *cfg with defaults for n_cam cameras of width x height. */
MOCAP_API void mocap_default_config(mocap_config* cfg, int n_cam, int width, int height);

MOCAP_API int  mocap_create(mocap_ctx** out, const mocap_config* cfg);
MOCAP_API void mocap_destroy(mocap_ctx* ctx);
MOCAP_API const char* mocap_last_error(const mocap_ctx* ctx);
/* Text for a status when no context exists (mocap_create failed). */
MOCAP_API const char* mocap_status_string(int status);

/* cudaStream_t on which all *_dev work is enqueued (NULL = the legacy default stream). */
MOCAP_API int mocap_set_stream(mocap_ctx* ctx, void* cuda_stream);

/* Camera model of the session.  HOST pointers: K[n_cam][9], R[n_cam][9], t[n_cam][3],
 * row-major doubles.  Replaces the state the reference keeps in
 * Cameras.camera_params (helpers.py:19-22,188-193) and in the camera_poses list
 * every hot-path function receives (helpers.py:293,339; set at helpers.py:171-175).
 * Builds on the host, once: P_kc = K_k [R_c|t_c] (helpers.py:305-308,351-355) and the
 * fundamental matrices F_rc of every ordered camera pair
 * (cv.sfm.fundamentalFromProjections, helpers.py:362). */
MOCAP_API int mocap_set_cameras(mocap_ctx* ctx, const double* K, const double* R, const double* t);

/* Optional epilogue of the matcher: object points leave in world coordinates
 * (helpers.py:96-103: flip x,y; 4x4 to_world_coords_matrix; dehomogenise; swap y,z).
 * M = NULL switches it off (default).  HOST pointer, 16 doubles row-major. */
MOCAP_API int mocap_set_world_transform(mocap_ctx* ctx, const double* M);

/* S1 -- replaces Cameras._find_dot (helpers.py:143-163) for n_images images at once:
 * gray (cvtColor RGB2GRAY when channels == 3), pix > threshold, 8-connected blobs,
 * contour-polygon moments, centre = int(m10/m00), int(m01/m00); zero-area blobs are
 * dropped; blobs leave in cv.findContours order (descending raster position of the
 * blob's first pixel).  blob_mom and img_flags may be NULL. */
MOCAP_API int mocap_detect_dev(mocap_ctx* ctx, const uint8_t* frames, int n_images, int channels,
                     int threshold, int32_t* blob_xy, int32_t* blob_n,
                     int64_t* blob_mom, int32_t* img_flags);

/* Holed blobs wider or taller than 62 pixels in S1 (every entry point that runs S1).  cv.findContours(RETR_TREE) +
 * cv.moments (helpers.py:147-158) give such a blob a contour per hole and fill its outer one, whatever its size; by
 * default (off) S1 reproduces that for holed blobs up to 62 x 62 pixels only and flags an image with a larger one
 * (MOCAP_F_HOLES).  on != 0 allocates a whole-image window for the slow path, four bitmaps of (height + 2) x
 * ceil((width + 2) / 64) 64-bit words per SM (166 KB per SM at 640 x 480, 409 KB at 1024 x 768), and larger holed
 * blobs are reproduced too: only more than 64 holes in one image leave the flag.  on == 0 frees it.  Results of images
 * the default already reproduces do not change.  Synchronises the context's stream; MOCAP_ENOMEM when the allocation
 * fails (the setting is then off). */
MOCAP_API int mocap_set_large_holes(mocap_ctx* ctx, int on);

/* S2+S3 -- replaces find_point_correspondance_and_object_points (helpers.py:339-421),
 * incl. the triangulate_points / calculate_reprojection_errors calls inside it
 * (helpers.py:408-419), for n_frame_sets frame-sets at once.  Input is the output of
 * mocap_detect_dev.  chosen and set_flags may be NULL. */
MOCAP_API int mocap_match_triangulate_dev(mocap_ctx* ctx, const int32_t* blob_xy, const int32_t* blob_n,
                                int n_frame_sets, double* obj, double* err, int32_t* n_obj,
                                int32_t* set_flags, int32_t* chosen);

/* S1+S2+S3 back to back on the context's stream, intermediate blob lists kept in
 * context-owned device memory: the per-frame body of Cameras._camera_read
 * (helpers.py:84-103) without capture/preprocessing. */
MOCAP_API int mocap_pipeline_dev(mocap_ctx* ctx, const uint8_t* frames, int n_frame_sets, int channels,
                       int threshold, double* obj, double* err, int32_t* n_obj, int32_t* set_flags);

/* mocap_pipeline_dev that also leaves, for every emitted point, the pixel of the winning correspondence in each
 * camera: track_xy int32 [n_frame_sets][max_roots][n_cam][2], (-1, -1) where the camera has no view (NULL: not
 * written).  This is the (F, C, 2) image_points array with None entries that bundle_adjustment receives
 * (helpers.py:244, index.py:272), per triangulated point. */
MOCAP_API int mocap_pipeline_tracks_dev(mocap_ctx* ctx, const uint8_t* frames, int n_frame_sets, int channels,
                              int threshold, double* obj, double* err, int32_t* n_obj, int32_t* set_flags,
                              int32_t* track_xy);

/* Same with HOST buffers: frames are copied to the device in chunks overlapped with
 * compute, results copied back; returns after the results are in the host buffers.
 * For best speed pass page-locked memory (mocap_host_alloc). */
MOCAP_API int mocap_pipeline_host(mocap_ctx* ctx, const uint8_t* frames, int n_frame_sets, int channels,
                        int threshold, double* obj, double* err, int32_t* n_obj, int32_t* set_flags);

/* Capture-side preprocessing -- replaces the per-camera body of Cameras._camera_read before S1
 * (helpers.py:70-82): rot90, make_square (zero pad + 8-row feather, helpers.py:507-523), cv.undistort,
 * cv.GaussianBlur 9x9, cv.filter2D with the 5x5 sharpening kernel, cvtColor RGB2BGR -- in one kernel,
 * bit-exact with cv2's 8-bit arithmetic.  The context must be square: width == height == in_width (the
 * reference's make_square only handles landscape frames padded top and bottom).  HOST pointers:
 * rotation int [n_cam] (0 or 2, camera-params.json "rotation"), K double [n_cam][9], dist double
 * [n_cam][5] = k1 k2 p1 p2 k3 (camera-params.json "distortion_coef"). */
MOCAP_API int mocap_set_preprocess(mocap_ctx* ctx, int in_width, int in_height, const int* rotation,
                         const double* K, const double* dist);
/* raw uint8 [n_images][in_height][in_width][3] -> out uint8 [n_images][S][S][3].  DEVICE pointers.
 * n_images = n_frame_sets * n_cam (camera index = image index mod n_cam). */
MOCAP_API int mocap_preprocess_dev(mocap_ctx* ctx, const uint8_t* raw_frames, int n_images, uint8_t* out_frames);
/* The whole per-frame body of Cameras._camera_read (helpers.py:70-103) for n_frame_sets frame-sets of RAW
 * camera frames: preprocessing (as mocap_preprocess_dev) -> S1 -> S2+S3.  The preprocessing kernel also
 * emits the grey plane _find_dot's cvtColor(RGB2GRAY) would derive from the processed frame
 * (helpers.py:144), so S1-S3 read 1 byte per pixel; results are those of S1 on the 3-channel frames.
 * processed (uint8 [n_images][S][S][3], the frames the reference goes on to JPEG-encode) may be NULL when
 * the caller does not display them (then they are never written).  DEVICE pointers. */
MOCAP_API int mocap_pipeline_raw_dev(mocap_ctx* ctx, const uint8_t* raw_frames, int n_frame_sets, int threshold,
                           uint8_t* processed, double* obj, double* err, int32_t* n_obj, int32_t* set_flags);
/* The fixed-point undistortion map of one camera as built by mocap_set_preprocess (the tables
 * cv.initUndistortRectifyMap(..., CV_16SC2) returns): m1 int16 [S][S][2], m2 uint16 [S][S].  HOST pointers. */
MOCAP_API int mocap_get_undistort_map(mocap_ctx* ctx, int cam, int16_t* m1, uint16_t* m2);

/* Tracking hand-off -- replaces locate_objects (helpers.py:424-480) for n_frame_sets frame-sets at
 * once: marker triplets (two markers 0.15 apart, a third 0.095 from both, tolerance 0.025) -> object
 * records.  Input is the matcher's output (obj/err/n_obj, with the world transform set if the caller
 * wants world coordinates as the reference does).  objects double [n_frame_sets][max_objects][5] =
 * {x, y, z, heading, error}; drone_index int32 [n_frame_sets][max_objects]; n_objects int32
 * [n_frame_sets].  A frame-set's first min(n_obj, max_roots) points are read (n_obj <= 0: none).  A frame-set can hold up
 * to one object per point; objects beyond max_objects (>= 1) are dropped in scan order, n_objects is clamped to
 * max_objects and record slots at or beyond n_objects are left unwritten.  DEVICE pointers. */
MOCAP_API int mocap_locate_objects_dev(mocap_ctx* ctx, const double* obj, const double* err, const int32_t* n_obj,
                             int n_frame_sets, int max_objects, double* objects, int32_t* drone_index,
                             int32_t* n_objects);

/* Drone tracking -- replaces KalmanFilter.predict_location (KalmanFilter.py:50-100, with its LowPassFilter.py
 * filters) for n_frame_sets frame-sets at once; each frame-set is one predict_location call at its timestamp.  A
 * tracker holds device-resident state for num_objects (1 .. 8) drones on one context and enqueues on the context's
 * stream; create it after the context's stream is set as wanted, destroy it before the context.
 *   mocap_tracker_reset(tr, prev_time): the reference's reset() with prev_time = its time.time() - 20: the next
 *   present step of every drone re-initialises at its first candidate and prev_positions returns to zero; the
 *   covariance and the low-pass histories are kept.  Applied by the next mocap_track_objects_dev call.
 *   mocap_track_objects_dev: objects / drone_index / n_objects / max_objects are mocap_locate_objects_dev's outputs,
 *   timestamps double [n_frame_sets] in seconds (a frame-set with no objects only advances time).  Outputs per
 *   frame-set and drone: pos float [n_frame_sets][num_objects][3], vel float [..][3] (low-pass filtered), heading
 *   double [..] (low-pass filtered), present uint8 [..] (1 where the reference returns a record for the drone),
 *   chosen int32 [..] (the object row the drone was associated with, -1 if absent); pos / vel / heading are 0 where
 *   present is 0.  DEVICE pointers, two launches, never synchronises (the first batch larger than the tracker's
 *   buffers waits for the stream while they grow).  A NULL pointer, max_objects < 1 or n_frame_sets < 1 returns
 *   MOCAP_EINVAL before any launch. */
typedef struct mocap_tracker mocap_tracker;
MOCAP_API int  mocap_tracker_create(mocap_ctx* ctx, int num_objects, mocap_tracker** out);
MOCAP_API void mocap_tracker_destroy(mocap_tracker* tr);
MOCAP_API int  mocap_tracker_reset(mocap_tracker* tr, double prev_time);
MOCAP_API int  mocap_track_objects_dev(mocap_tracker* tr, const double* objects, const int32_t* drone_index,
                                       const int32_t* n_objects, int max_objects, const double* timestamps,
                                       int n_frame_sets, float* pos, float* vel, double* heading, uint8_t* present,
                                       int32_t* chosen);
/* mocap_track_objects_dev with a gate: call uint8 [n_frame_sets] (DEVICE).  A frame-set whose call entry is 0 is not a
 * predict_location call -- the reference makes none on a read where no camera saw a blob (helpers.py:90,106): the
 * tracker's clock, call index and low-pass histories do not move, and its outputs are present = 0, chosen = -1 and
 * zeros.  call == NULL: every frame-set is a call (= mocap_track_objects_dev). */
MOCAP_API int  mocap_track_objects_gated_dev(mocap_tracker* tr, const double* objects, const int32_t* drone_index,
                                             const int32_t* n_objects, int max_objects, const double* timestamps,
                                             const uint8_t* call, int n_frame_sets, float* pos, float* vel, double* heading,
                                             uint8_t* present, int32_t* chosen);

/* The live capture loop -- replaces Cameras._camera_read (helpers.py:68-135) from the raw frames of the camera driver
 * to the filtered drone states, for n_reads reads at once (a read is one call of _camera_read; n_reads = 1 in the
 * live loop, more to replay a recorded session).  The context must have had mocap_set_preprocess; the read's chain is
 * the existing stages: preprocessing -> S1 -> k_live_blobs (capture payload, gate, flags, dots) -> S2+S3 with the
 * world transform -> locate_objects -> the gated tracker.
 *   mode: bits of MOCAP_LIVE_*, following the reference's nesting (helpers.py:84-106): 0 = preprocessing only;
 *   CAPTURE = S1 (needs no cameras: the reference has no poses yet in capture mode); CAPTURE|TRIANGULATE = also S2+S3
 *   (needs mocap_set_cameras); CAPTURE|TRIANGULATE|LOCATE = also the locator and the tracker (needs tr, created on
 *   this context, and timestamps).  Any other combination returns MOCAP_EINVAL before any launch.
 *   raw uint8 [n_reads][n_cam][in_h][in_w][3]; timestamps double [n_reads] (the clock reading of each read, locate
 *   mode only, may be NULL otherwise); frames uint8 [n_reads][n_cam][S][S][3] or NULL: the processed frames, with a
 *   1-px (100, 255, 100) dot at every blob centre when CAPTURE is set (what the drop-in _find_dot draws).
 *   result: ONE device buffer of mocap_live_layout(ctx, n_reads, tr ? num_objects : 0).total bytes, struct of arrays
 *   over the reads, each slice written by the stage that computes it (byte offsets in mocap_live_layout):
 *     flags      int32  [R]          OR of the read's images' MOCAP_F_* bits and its frame-set flags
 *     gate       uint8  [R]          1 where some camera has at least one blob (helpers.py:90); 0 in mode 0
 *     blob_n     int32  [R][C]       blobs per camera (0 in mode 0)
 *     first      int32  [R][C][2]    first blob centre per camera, (-1, -1) if none (helpers.py:92)
 *     n          int32  [R]          TRIANGULATE: points of the matcher (helpers.py:94)
 *     obj        double [R][RM][3]   ... in world coordinates when a world transform is set (helpers.py:96-103)
 *     err        double [R][RM]
 *     n_objects  int32  [R]          LOCATE: locate_objects (helpers.py:105), M = max_roots records per read
 *     objects    double [R][M][5]    {x, y, z, heading, error}
 *     drone_index int32 [R][M]
 *     called     uint8  [R]          LOCATE: 1 where the read is a predict_location call (= gate)
 *     pos        float  [R][D][3]    LOCATE: the tracker's outputs (mocap_track_objects_gated_dev with call = called)
 *     vel        float  [R][D][3]
 *     heading    double [R][D]
 *     present    uint8  [R][D]
 *     chosen     int32  [R][D]
 *   Slices a mode does not compute, and record slots beyond n / n_objects, are left unwritten.  DEVICE pointers,
 *   never synchronises, allocates only while the context's scratch grows to the batch size. */
#define MOCAP_LIVE_CAPTURE     1
#define MOCAP_LIVE_TRIANGULATE 2
#define MOCAP_LIVE_LOCATE      4
typedef struct mocap_live_offsets {
    uint64_t flags, gate, blob_n, first, n, obj, err, n_objects, objects, drone_index, called, pos, vel, heading, present,
             chosen;
    uint64_t total;     /* bytes of the result buffer; every slice starts on a 16-byte boundary */
} mocap_live_offsets;
MOCAP_API int  mocap_live_layout(mocap_ctx* ctx, int n_reads, int num_objects, mocap_live_offsets* layout);
MOCAP_API int  mocap_live_dev(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode,
                              const double* timestamps, uint8_t* frames, void* result);
/* The same with HOST raw / timestamps / frames / result: one host-to-device copy (timestamps and raw frames through
 * page-locked staging the context owns), the device chain, one device-to-host copy of the result and one of the frames
 * (if asked for), one synchronisation. */
MOCAP_API int  mocap_live_host(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode,
                               const double* timestamps, uint8_t* frames, void* result);

/* Baseline JPEG encoding -- the camera stream's cv.imencode('.jpg', frames) (index.py:55-56), byte for byte what
 * cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality]) returns with libjpeg-turbo: 3-channel BGR input,
 * 4:2:0, the standard (Annex K) Huffman tables, JFIF 1.01, no restart markers.
 * mocap_jpeg_bound: worst-case bytes of one width x height image, header and EOI included (0 for a size outside
 * 1..65500).
 * mocap_encode_jpeg_dev: images uint8 [n_images][tile_h][tiles * tile_w][3], stored as the frames side by side are
 *   stored one after another, [n_images][tiles][tile_h][tile_w][3] -- np.hstack of `tiles` frames without the copy;
 *   tiles = 1 is a plain image.  out uint8 [n_images][out_stride]: image i's JPEG from out + i * out_stride;
 *   out_len int32 [n_images]: its length, or -1 when it does not fit out_stride (then nothing of it is written).
 *   quality 1..100; any other, n_images < 0, tiles, tile_w or tile_h < 1, or a side over 65500 give MOCAP_EINVAL before
 *   any launch.  DEVICE pointers, the context's stream, never synchronises; 4 launches per group of images (a group is
 *   as many as fit 256 MB of scratch, about 8 bytes per pixel).
 * mocap_live_jpeg_host: mocap_live_host (same chain, same outputs), plus the JPEG of each read's processed frames side
 *   by side (np.hstack, helpers.py:141; with the dots in capture mode) at `quality`: HOST jpeg uint8
 *   [n_reads][jpeg_stride], jpeg_len int32 [n_reads]; frames may be NULL.  Copies back exactly the JPEG bytes.  Two
 *   synchronisations: one for the result, the frames and the lengths, one for the bytes.  A JPEG longer than
 *   jpeg_stride returns MOCAP_EINVAL after the first (jpeg is then not written; result and frames are). */
MOCAP_API uint64_t mocap_jpeg_bound(int width, int height);
MOCAP_API int  mocap_encode_jpeg_dev(mocap_ctx* ctx, const uint8_t* images, int n_images, int tiles, int tile_w, int tile_h,
                                     int quality, uint8_t* out, uint64_t out_stride, int32_t* out_len);
MOCAP_API int  mocap_live_jpeg_host(mocap_ctx* ctx, mocap_tracker* tr, const uint8_t* raw, int n_reads, int mode,
                                    const double* timestamps, uint8_t* frames, void* result,
                                    int quality, uint8_t* jpeg, uint64_t jpeg_stride, int32_t* jpeg_len);

/* S3 -- replaces triangulate_points (helpers.py:330-336) and
 * calculate_reprojection_errors (helpers.py:203-211) on explicit correspondences.
 * obs double [n_points][n_cam][2], mask uint8 [n_points][n_cam] (0 = [None, None]).
 * X double [n_points][3], err double [n_points], valid uint8 [n_points]
 * (0 where the reference returns [None]*3 / None, i.e. fewer than two views).
 * err may be NULL.  DEVICE pointers. */
MOCAP_API int mocap_triangulate_dev(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                          double* X, double* err, uint8_t* valid);
/* HOST-pointer convenience form of the above. */
MOCAP_API int mocap_triangulate_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                           double* X, double* err, uint8_t* valid);
/* calculate_reprojection_errors for GIVEN points (helpers.py:203-241). HOST pointers. */
MOCAP_API int mocap_reprojection_errors_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask,
                                   const double* X, int n_points, double* err, uint8_t* valid);

/* Cold-start extrinsics -- replaces the body of calculate_camera_pose up to its bundle_adjustment call
 * (index.py:229-270): per adjacent camera pair a fundamental matrix from the common observations,
 * E = K1^T F K0 (cv.sfm.essentialFromFundamental with the intrinsics of cameras 0 and 1), the four
 * motions of cv.sfm.motionFromEssential, the reference's cheirality vote and the pose chain.  The
 * reference's F comes from cv.findFundamentalMat(FM_RANSAC) (seeded, repeatable); here F is a
 * normalised 8-point estimate re-fitted twice on its 1 px Sampson inliers, or -- F_given != NULL --
 * supplied by the caller (double [n_cam-1][9], x2^T F x1 = 0).  HOST pointers: obs/mask as for
 * mocap_bundle_adjust_host; R [n_cam][9], t [n_cam][3] out; F_used [n_cam-1][9] and votes
 * [n_cam-1][4] (points in front of the cameras per candidate) may be NULL. */
MOCAP_API int mocap_calibrate_init_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                              const double* F_given, double* R, double* t, double* F_used, int* votes);

/* Robust form of the above: each pair's F comes from RANSAC, as the reference's cv.findFundamentalMat(FM_RANSAC,
 * 1 px, 0.99999) does (index.py:246), so that mismatched points (a stray reflection recorded in capture-points mode)
 * do not pull the fit.  For all C-1 pairs at once, on the device: `hypotheses` 7-point samples per pair drawn from
 * a counter-based hash of (seed, pair, hypothesis) -- the result does not depend on the launch geometry, and is
 * repeatable for a given seed -- every model scored with cv2's fundamental-matrix error (the larger squared
 * distance to the two epipolar lines) against threshold_px^2, and per pair the model with the most inliers (ties:
 * the lowest hypothesis, then root).  The normalised 8-point fit and its Sampson re-selection rounds (at
 * threshold_px) then start from that model's inliers instead of from all points; E, the cheirality vote (over all
 * common observations, as index.py:253-257) and the chain are those of mocap_calibrate_init_host.  cv2's sample
 * sequence is not replayed: parity is defined downstream of F.  HOST pointers; opt NULL = defaults; R, t, F_used,
 * votes as above; inliers uint8 [n_points][n_cam-1] (may be NULL): 1 where the point is in the pair's final fit
 * set, 0 elsewhere and where the frame is not common to the pair.  Bad options, or a pair with fewer than 8 common
 * observations, return MOCAP_EINVAL before anything is launched. */
typedef struct mocap_ransac_options {
    double   threshold_px;   /* 1.0 (index.py:246)                              */
    int      hypotheses;     /* 2048 per pair, 1 .. 65536                        */
    uint64_t seed;           /* 0                                                */
} mocap_ransac_options;
MOCAP_API void mocap_ransac_default_options(mocap_ransac_options* opt);
MOCAP_API int  mocap_calibrate_init_ransac_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                      const mocap_ransac_options* opt, double* R, double* t, double* F_used,
                                      int* votes, uint8_t* inliers);
/* The RANSAC stage of the above alone: per adjacent pair the winning model F [n_cam-1][9] (unit Frobenius norm,
 * x2^T F x1 = 0) and its inliers uint8 [n_points][n_cam-1] (may be NULL) at threshold_px, before any refinement.
 * Three kernel launches whatever the number of cameras.  Needs no intrinsics.  HOST pointers. */
MOCAP_API int  mocap_fundamental_ransac_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                   const mocap_ransac_options* opt, double* F, uint8_t* inliers);

/* Pose-graph cold start: every camera placed from every overlapping pair instead of the chain of adjacent pairs.
 * It computes what the reference's calculate-camera-pose handler computes (index.py:229-270) -- the camera poses in
 * camera 0's frame with |t_1| = 1, from 2D tracks and the intrinsics -- and departs from it deliberately:
 *   - every pair (a < b) with at least min_common common observations is used, not only (c, c+1): one bad pair no
 *     longer breaks the cameras after it;
 *   - each pair's F comes from RANSAC (as mocap_calibrate_init_ransac_host, pair p of the pair table drawing its
 *     samples from (seed, p)), re-fitted by 8-point rounds on its Sampson inliers;
 *   - E = K_b^T F K_a with each pair's own intrinsics (the reference uses those of cameras 0 and 1, index.py:247), and
 *     the four motions are judged in the pair's own frame, P_a = K_a [I|0], P_b = K_b [R|t], counting the inliers in
 *     front of both cameras (the reference triangulates with camera a's accumulated pose on one side and the relative
 *     candidate on the other, index.py:253-262, which can pick a twisted motion);
 *   - a pair is dropped with fewer than min_inliers points in front or a median triangulation angle below
 *     min_angle_deg; rotations by weighted chordal averaging with Cauchy re-weighting, pairs off by more than
 *     rot_outlier_deg dropped;
 *   - translations from the bearing constraints of every track with the rotations known (the reference chains
 *     t_{c+1} = t_c + R_c t_rel with unit baselines, index.py:264-265), irls_rounds rounds of Cauchy weights at 4 px;
 *     a view enters if it is an inlier of at least 2 used pairs (1 where its camera has one used pair).
 * HOST pointers.  ropt / gopt NULL = defaults.  R [n_cam][9], t [n_cam][3] out.  pairs (capacity n_cam(n_cam-1)/2,
 * may be NULL) receives one record per pair of the pair table, *n_pairs (may be NULL) their number.  support uint8
 * [n_points][n_cam] (may be NULL): 1 where the view's final weight is >= 0.5 on a track that keeps at least 2 such
 * views -- a first bundle-adjustment mask.  Bad options, too few common observations to link every camera to camera 0
 * or more than 16 cameras return MOCAP_EINVAL before any launch; if the pairs that pass the checks no longer link every
 * camera, MOCAP_EINVAL names the cameras.  Device scratch grows with pairs x hypotheses x 27 doubles (53 MB at 120
 * pairs x 2048, 425 MB at 16384); MOCAP_ECUDA if it cannot be allocated.  Two calls with the same inputs give the same
 * bits. */
typedef struct mocap_graph_options {
    int    min_common;        /* 30: common observations for a pair to enter the table, >= 8 */
    int    min_inliers;       /* 30: inliers in front of both cameras for a pair to be used   */
    double min_angle_deg;     /* 2.0: median triangulation angle for a pair to be used        */
    double rot_outlier_deg;   /* 5.0: rotation residual above which a pair is dropped         */
    int    irls_rounds;       /* 4: translation solves, 1 .. 64                               */
} mocap_graph_options;
typedef struct mocap_graph_pair {
    int    a, b;              /* cameras, a < b                                               */
    int    common;            /* common observations                                          */
    int    inliers;           /* Sampson inliers of the re-fitted F                           */
    int    candidate;         /* chosen motion 0..3 of E, -1 if none                           */
    int    in_front;          /* inliers in front of both cameras under it                    */
    double median_angle_deg;  /* median triangulation angle of those                          */
    double rot_residual_deg;  /* angle between R_b R_a^T and the pair's R_ab (NaN: no motion) */
    int    used;              /* 1 if the pair placed the rotations and chose the views       */
} mocap_graph_pair;
MOCAP_API void mocap_graph_default_options(mocap_graph_options* opt);
MOCAP_API int  mocap_calibrate_graph_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                const mocap_ransac_options* ropt, const mocap_graph_options* gopt, double* R, double* t,
                                mocap_graph_pair* pairs, int* n_pairs, uint8_t* support);

/* S4 -- replaces bundle_adjustment (helpers.py:244-290): robust (Cauchy) trust-region
 * least squares over the poses of cameras 1..C-1 (rotation vector + translation;
 * camera 0 pinned at (I,0); the reference's focal parameters are dead, helpers.py:267-270),
 * residual_j = float32(mean squared reprojection error of point j after DLT
 * re-triangulation with the trial poses).  HOST pointers; R,t are in/out. */
typedef struct mocap_ba_options {
    double ftol;        /* 1e-2  (helpers.py:288)                */
    double xtol;        /* 1e-8  (scipy default)                 */
    double gtol;        /* 1e-8  (scipy default)                 */
    int    max_nfev;    /* 0 -> 100 * n_params (scipy default)   */
    int    jacobian;    /* 0: 2-point finite differences of the float32 residuals -- exactly what scipy
                              differentiates for the reference (percent-level quantisation noise,
                              SURVEY.md section 7); 1 (default): the same differences taken before the
                              float32 cast */
    int    prefit;      /* 1 (default): first run a classic Levenberg-Marquardt bundle adjustment over
                              poses AND points (analytic Jacobians, per-point 3x3 blocks eliminated by
                              Schur complement, dense reduced camera system) on the plain squared
                              reprojection error, then polish on the reference objective; 0: reference
                              iteration only */
    int    prefit_max_iter;  /* 50 */
    int    engine;      /* 0 (default): the whole solve in ONE persistent, grid-synchronous kernel (k_ba_solve): no host round
                              trips; 1: host-stepped (optimiser control on the host, one launch per phase, a stream
                              synchronisation per step) -- the same algorithm, kept as a cross-check */
} mocap_ba_options;

typedef struct mocap_ba_report {
    double cost_initial;   /* reference objective 0.5 * sum log1p(r^2) at the start   */
    double cost_final;     /* ... at the returned poses                                */
    double optimality;     /* ||J^T f||_inf at the end                                 */
    int    n_iterations;   /* trust-region iterations on the reference objective       */
    int    n_fev;          /* residual-vector evaluations (each = n_points DLTs)       */
    int    status;         /* scipy-style: 0 max_nfev, 1 gtol, 2 ftol, 3 xtol, 4 both  */
    int    n_residuals;
    double prefit_cost_initial;  /* 0.5 * sum of squared pixel residuals before / after the prefit */
    double prefit_cost_final;
    int    prefit_iterations;
    int    n_launches;     /* kernels launched by this call                            */
    int    n_tr_solves;    /* device-resident solve: trust-region sub-problems solved, and ... */
    int    n_tr_newton;    /* ... Newton iterations on the damping alpha they took in total (<= 10 each)  */
    float  phase_ms[8];    /* device-resident solve only: wall time per phase, CTA 0's clock --
                              0 set-up and control, 1 prefit: reduced camera system (Schur complement), 2 prefit: dense solve,
                              3 prefit: back-substitution + trial cost, 4 polish: finite-difference Jacobian + normal equations,
                              5 polish: tridiagonalisation, 6 polish: trust-region sub-problems, 7 polish: trial evaluations */
} mocap_ba_report;

MOCAP_API void mocap_ba_default_options(mocap_ba_options* opt);
MOCAP_API int  mocap_bundle_adjust_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                              double* R, double* t, const mocap_ba_options* opt,
                              mocap_ba_report* report);
/* The same with DEVICE buffers, stream-ordered, never synchronises: ONE cooperative launch of k_ba_solve runs the
 * whole bundle adjustment (residuals, Jacobians, Schur complement, the <= 90 x 90 dense solves, step control).
 * obs double [n_points_max][n_cam][2], mask uint8 [n_points_max][n_cam]; n_points (device int32, may be NULL =
 * n_points_max) is read by the kernel, so the count can come from mocap_tracks_to_observations_dev without a
 * host round trip; R [n_cam][9], t [n_cam][3] device doubles in/out; opt is a HOST pointer (NULL = defaults; the
 * engine field is ignored); report is a DEVICE pointer (may be NULL; status -3: no point with two views). */
MOCAP_API int  mocap_bundle_adjust_dev(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points_max,
                             const int32_t* n_points, double* R, double* t, const mocap_ba_options* opt,
                             mocap_ba_report* report);
/* CTA budget G of k_ba_solve for this context (1 .. number of SMs; 0 = the default, one per SM).  A single solve
 * (mocap_bundle_adjust_dev) runs on all G CTAs; a batch of K solves (mocap_bundle_adjust_batch_dev) splits them,
 * problem k getting G / K + (k < G % K).  One solve is a cooperative grid whose serial sections (dense solves,
 * tridiagonalisation) leave most CTAs waiting at the grid barrier, so INDEPENDENT solves -- the reference runs one
 * bundle_adjustment per recorded batch (index.py:249-276), a session with several batches has several -- finish sooner
 * side by side, in one batched call or as K contexts on K streams with G = SMs / K each (measured on an H100 SXM at a
 * 400 W power limit, a config-3 step of S1-S3 over 4000 frame-sets plus 4 solves of 8 cameras x 18 800 points:
 * 13.6 ms with the solves in turn on 132 CTAs, 11.3 ms as 2 x 66, 10.4 ms as 4 x 33 on four contexts).
 * Results depend on the number of CTAs a solve runs on only in the rounding of its sums, and are reproducible for
 * a given number. */
MOCAP_API int  mocap_set_ba_grid(mocap_ctx* ctx, int n_ctas);

/* One problem of a batched bundle adjustment: the arguments of mocap_bundle_adjust_dev that differ per solve.
 * DEVICE pointers; n_points may be NULL (= n_points_max), report may be NULL. */
#define MOCAP_BA_MAX_BATCH 16
typedef struct mocap_ba_problem {
    const double*    obs;          /* [n_points_max][n_cam][2]                                   */
    const uint8_t*   mask;         /* [n_points_max][n_cam]                                      */
    int              n_points_max;
    const int32_t*   n_points;     /* device int32, read by the kernel                           */
    double*          R;            /* [n_cam][9] in/out                                          */
    double*          t;            /* [n_cam][3] in/out                                          */
    mocap_ba_report* report;
} mocap_ba_problem;
/* n_problems (1 .. MOCAP_BA_MAX_BATCH, and at most the context's CTA budget, mocap_set_ba_grid) INDEPENDENT bundle
 * adjustments in ONE cooperative launch on the context's stream; never synchronises.  problems is a HOST array;
 * every problem uses the context's cameras and the one set of options opt (HOST, NULL = defaults).  Problem k runs
 * on its own G / K + (k < G % K) CTAs with its own barrier and workspace, and gives the same bits (poses and report,
 * phase_ms aside) as mocap_bundle_adjust_dev on a context whose budget is that number of CTAs; a problem without a
 * point that has two views reports status -3 and keeps its poses, the others are unaffected. */
MOCAP_API int  mocap_bundle_adjust_batch_dev(mocap_ctx* ctx, const mocap_ba_problem* problems, int n_problems,
                                   const mocap_ba_options* opt);
/* Matcher output of a batch -> the explicit correspondences S4 consumes (BASELINE config 3: S1-S3, then one
 * bundle adjustment per batch), on the device: track_xy int32 [n_frame_sets][max_roots][n_cam][2] as written by
 * mocap_pipeline_tracks_dev ((-1, -1) = no view), n_obj / err the matcher's outputs; tracks whose reprojection
 * error exceeds max_err are left out (max_err <= 0: keep all; err may then be NULL).  One row per kept track, in
 * frame order then root order: obs double [capacity][n_cam][2], mask uint8 [capacity][n_cam]; *n_points (device)
 * = number of rows written (<= capacity).  DEVICE pointers, stream-ordered. */
MOCAP_API int  mocap_tracks_to_observations_dev(mocap_ctx* ctx, const int32_t* track_xy, const int32_t* n_obj,
                                      const double* err, int n_frame_sets, double max_err, double* obs,
                                      uint8_t* mask, int32_t* n_points, int capacity);
/* Per-view screening of explicit correspondences against poses (rule in DESIGN section 5): for each track, the
 * 2-view DLT point of every pair of its views in mask_in, the pair whose point the most views reproject to within
 * threshold_px wins (ties to the earlier pair), its supporting views are re-triangulated and the views within
 * threshold_px of that point are kept if they are >= 2 and all pass against their own DLT point; otherwise the row is
 * emptied (the track leaves the adjustment).  Rows with fewer than two views are copied unchanged.  The arithmetic is
 * that of the bundle adjustment's residual.  Screen again from the caller's ORIGINAL mask after each adjustment, so
 * that a view dropped under poor poses can come back.  obs double [n_points_max][n_cam][2], mask_in / mask_out uint8
 * [n_points_max][n_cam] (rows past *n_points are left untouched), R [n_cam][9], t [n_cam][3] the CURRENT poses (e.g.
 * the buffers mocap_bundle_adjust_dev updates), stats int32 [4] = views in, views kept, views dropped, rows emptied.
 * DEVICE pointers, one launch, never synchronises; n_points may be NULL (= n_points_max); stats may be NULL.  A
 * threshold_px that is <= 0 or not finite, a NULL obs / mask / R / t / mask_out, or mask_out == mask_in returns
 * MOCAP_EINVAL before any launch. */
MOCAP_API int  mocap_screen_observations_dev(mocap_ctx* ctx, const double* obs, const uint8_t* mask_in, int n_points_max,
                                   const int32_t* n_points, const double* R, const double* t, double threshold_px,
                                   uint8_t* mask_out, int32_t* stats);
/* The same with HOST pointers (n_points a host int32, may be NULL); copies inside and synchronises. */
MOCAP_API int  mocap_screen_observations_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask_in, int n_points_max,
                                    const int32_t* n_points, const double* R, const double* t, double threshold_px,
                                    uint8_t* mask_out, int32_t* stats);
/* residual vector of S4 at explicit poses (helpers.py:264-276); r float [n_points],
 * valid uint8 [n_points]; returns the number of valid residuals in *n_valid. HOST pointers. */
MOCAP_API int  mocap_ba_residuals_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                             const double* R, const double* t, float* r, uint8_t* valid, int* n_valid);

/* page-locked host memory for the *_host entry points */
MOCAP_API int  mocap_host_alloc(void** out, uint64_t bytes);
MOCAP_API void mocap_host_free(void* p);

/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
MOCAP_API uint64_t mocap_launch_count(const mocap_ctx* ctx);
/* Average device time in ms of the blob-detection kernel over the launches since the
 * last call with reset != 0, measured with CUDA events on the context's stream when
 * enabled by mocap_enable_kernel_timing(ctx, 1).  Synchronises the stream. */
MOCAP_API int  mocap_enable_kernel_timing(mocap_ctx* ctx, int on);
MOCAP_API int  mocap_detect_kernel_ms(mocap_ctx* ctx, int reset, double* avg_ms, int* n_launches);

#ifdef __cplusplus
}
#endif
#endif /* MOCAP_B200_H */

// Test-only: the single-pass pipeline kernel k_pipeline_fused (csrc/fused_device.cuh: dynamic unit claiming,
// rolling-window stream loop, "last arriver does the follow-up" blob reduce and matcher, worklists, self-resetting
// counters) run UNCHANGED on the host through the SIMT emulation in simt_emu.h: one CTA of n_warps warps, every
// CUDA thread a std::thread, so the warps really do race for units and for the last-arriver roles.
// Parameter set-up mirrors launch_pipeline_fused (csrc/fused_kernel.cu).
// NOT part of libmocap_b200.so and never used by the product path.
#include "simt_emu.h"
#include "../../low-cost-mocap_b200/csrc/fused_device.cuh"
#include "../../low-cost-mocap_b200/csrc/camera_tables.h"

alignas(16) unsigned char smem_raw[64 * 1024 * 4];            // the kernel's `extern __shared__` array (one CTA)

// frames uint8 [n_sets][C][H][W] -> obj [n_sets][RMAX][3], err [n_sets][RMAX], n_obj, set_flags, blob_xy
// [n_img][MB][2], blob_n [n_img]; counters[0..1] = images / frame-sets left on the worklists, counters[2] = number of
// self-resetting scratch words found non-zero after the run (must be 0), counters[3] = units claimed.
extern "C" int hc_pipeline_fused(const uint8_t* frames, int n_sets, int C, int W, int H, int threshold, const double* K, const double* R,
                                 const double* t, int MB, int E, int RMAX, int KC, unsigned GMAX, int n_warps, int runs,
                                 double* obj, double* err, int32_t* n_obj, int32_t* set_flags, int32_t* blob_xy, int32_t* blob_n,
                                 uint32_t* img_worklist, uint32_t* set_worklist, long long* counters, int channels) {
    static CameraTables T;
    memset(&T, 0, sizeof(T));
    build_camera_tables(T, C, K, R, t);
    const int n_img = n_sets * C;
    FusedParams P;
    memset(&P, 0, sizeof(P));
    P.frames = reinterpret_cast<const uint4*>(frames);
    P.n_sets = n_sets; P.C = C; P.W = W; P.H = H;
    P.seg_per_image = W * H / MOCAP_SEG_PX;
    P.u4_per_image = P.seg_per_image * (channels == 3 ? 3 : 1);
    P.threshold = threshold;
    const int iters_total = (P.u4_per_image + FUSED_SEGS_PER_ITER - 1) / FUSED_SEGS_PER_ITER;
    P.units_per_image = (iters_total + 15) / 16;
    P.iters_per_unit = (iters_total + P.units_per_image - 1) / P.units_per_image;
    P.total_units = (long long)n_sets * C * P.units_per_image;
    P.tc = thresh_const(threshold);
    P.E = E;
    std::vector<uint32_t> seg_count(n_img, 0), seg_list((size_t)n_img * E, 0), img_done(n_img, 0), set_done(n_sets, 0), set_defer(n_sets, 0);
    std::vector<uint32_t> work_count(4, 0);
    std::vector<int32_t> img_flags(n_img, 0);
    unsigned long long unit_counter = 0;
    P.seg_count = seg_count.data(); P.seg_list = seg_list.data();
    P.img_done = img_done.data(); P.set_done = set_done.data(); P.set_defer = set_defer.data();
    P.unit_counter = &unit_counter;
    P.blob_xy = blob_xy; P.blob_n = blob_n; P.img_flags = img_flags.data();
    P.img_worklist = img_worklist; P.img_work_count = work_count.data();
    P.set_worklist = set_worklist; P.set_work_count = work_count.data() + 2;
    P.tb = &T;
    P.MB = MB; P.RMAX = RMAX; P.KC = KC; P.GMAX = GMAX;
    P.obj = obj; P.err = err; P.n_obj = n_obj; P.set_flags = set_flags;
    const size_t a = sizeof(WarpSlab), b = warp_state_bytes(RMAX, C, KC, MB);
    P.slab_bytes = ((a > b ? a : b) + 15) & ~(size_t)15;
    if (P.slab_bytes * n_warps > sizeof(smem_raw)) return -1;
    const long long mx = W > H ? W : H;
    const bool wide = 6ll * mx * W * H >= (1ll << 32);
    for (int run = 0; run < runs; ++run) {                   // a second run must find every counter re-armed
        unit_counter = 0;                                    // (the launcher resets this one with a memset)
        if (run > 0 && (work_count[0] || work_count[2])) break;       // worklists are consumed by the fallback kernels
        simt::launch(32 * n_warps, [&] {
            if (channels == 3) {
                if (wide) { if (P.tc.use_and) k_pipeline_fused<true, true, true>(P); else k_pipeline_fused<true, false, true>(P); }
                else      { if (P.tc.use_and) k_pipeline_fused<false, true, true>(P); else k_pipeline_fused<false, false, true>(P); }
            } else {
                if (wide) { if (P.tc.use_and) k_pipeline_fused<true, true>(P); else k_pipeline_fused<true, false>(P); }
                else      { if (P.tc.use_and) k_pipeline_fused<false, true>(P); else k_pipeline_fused<false, false>(P); }
            }
        });
    }
    long long dirty = 0;
    for (int i = 0; i < n_img; ++i) {
        dirty += img_done[i] != 0;
        bool listed = false;
        for (uint32_t w = 0; w < work_count[0]; ++w) listed = listed || img_worklist[w] == (uint32_t)i;
        if (!listed) dirty += seg_count[i] != 0;             // deferred images keep their list for the fallback kernel
    }
    for (int s = 0; s < n_sets; ++s) dirty += (set_done[s] != 0) + (set_defer[s] != 0);
    counters[0] = work_count[0]; counters[1] = work_count[2]; counters[2] = dirty; counters[3] = (long long)unit_counter;
    return 0;
}

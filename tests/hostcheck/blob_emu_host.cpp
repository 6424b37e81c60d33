// Test-only: the S1 device code of low-cost-mocap_b200/csrc/blob_device.cuh (packed threshold, segment masks,
// and the whole sparse per-image reduction: sort, runs, lock-free union-find, 2x2-cell moments, ranking) run
// UNCHANGED on the host through the SIMT emulation in simt_emu.h, one std::thread per CUDA thread, the way
// k_blob_reduce_warp (one warp per image) and k_blob_reduce (128-thread CTA per deferred image) drive it.
// NOT part of libmocap_b200.so and never used by the product path.
#include "simt_emu.h"
#include "../../low-cost-mocap_b200/csrc/blob_device.cuh"
#include <algorithm>
#include <random>

namespace {

// the stream kernel's per-segment work (k_threshold_segments_c1), in a shuffled order: the kernel's atomic
// append gives no order either
std::vector<uint32_t> segments_of(const uint8_t* img, int W, int H, int threshold, unsigned seed) {
    const ThreshConst tc = thresh_const(threshold);
    std::vector<uint32_t> list;
    const int n_seg = W * H / MOCAP_SEG_PX;
    for (int s = 0; s < n_seg; ++s) {
        uint4 v;
        memcpy(&v, img + (size_t)s * 16, 16);
        const bool any = tc.use_and ? any_above<true>(v, tc) : any_above<false>(v, tc);
        const uint32_t h0 = swar_gt(v.x, tc), h1 = swar_gt(v.y, tc), h2 = swar_gt(v.z, tc), h3 = swar_gt(v.w, tc);
        const uint32_t m = nibble_of(h0) | (nibble_of(h1) << 4) | (nibble_of(h2) << 8) | (nibble_of(h3) << 12);
        if (any != (m != 0)) return {0xDEADBEEFu};          // the fast test and the mask must agree
        if (m) list.push_back(((uint32_t)s << 16) | m);
    }
    std::mt19937 rng(seed);
    std::shuffle(list.begin(), list.end(), rng);
    return list;
}

template <bool WIDE>
int reduce_image(const std::vector<uint32_t>& list, int W, int H, int max_blobs, int E, int force_cta,
                 int32_t* xy, int32_t* n_out, int64_t* mom, int32_t* flags) {
    const int cnt = (int)list.size();
    if (cnt == 0) { *n_out = 0; *flags = 0; return 0; }
    bool ok = false;
    if (!force_cta && cnt <= BLOB_WE) {                      // k_blob_reduce_warp
        static WarpSlab slab;
        bool results[32];
        simt::launch(32, [&] {
            BlobSmem sm;
            sm.seg = slab.seg; sm.parent = slab.parent; sm.base = slab.base; sm.node_seg = slab.node_seg;
            sm.node_bits = slab.node_bits; sm.rank = slab.rank; sm.acc = slab.acc; sm.wsum = nullptr; sm.hs = nullptr;
            sm.rowfirst = BLOB_ROWFIRST(slab, WIDE); sm.row_cap = WIDE ? 0 : BLOB_ROWS;
            const int lane = threadIdx.x & 31;
            for (int i = lane; i < cnt; i += 32) sm.seg[i] = list[i];
            __syncwarp();
            results[lane] = blob_reduce<32, true, WIDE>(sm, cnt, BLOB_WE, BLOB_WACC, W, H, max_blobs, xy, n_out, mom, flags, 0);
        });
        ok = results[0];
        for (int l = 1; l < 32; ++l) if (results[l] != ok) return -2;     // the verdict must be warp-uniform
        if (ok) return 1;
    }
    // k_blob_reduce: 128-thread CTA, full-size capacities
    int fl = 0, n = cnt;
    if (cnt > E) { fl |= MOCAP_F_SEGMENTS; n = 0; }
    if (n == 0) { *n_out = 0; *flags = fl; return 2; }
    std::vector<unsigned long long> raw(blob_reduce_smem_bytes(E) / 8 + 2);
    simt::launch(128, [&] {
        BlobSmem sm = carve_blob_smem(reinterpret_cast<unsigned char*>(raw.data()), E);
        for (int i = threadIdx.x; i < n; i += 128) sm.seg[i] = list[i];
        __syncthreads();
        blob_reduce<128, false, WIDE>(sm, n, E, MOCAP_ACC_CAP, W, H, max_blobs, xy, n_out, mom, flags, fl);
    });
    return 2;
}

}  // namespace

// img uint8 [H][W] -> blobs as mocap_detect_dev reports them.  Returns 1 (warp path), 2 (CTA path), 0 (empty),
// < 0 on an internal inconsistency.  force_cta != 0 sends every image through the 128-thread variant.
extern "C" int hc_blob_detect(const uint8_t* img, int W, int H, int threshold, int max_blobs, int E, int force_cta, unsigned seed,
                              int32_t* xy, int32_t* n_out, int64_t* mom, int32_t* flags) {
    const std::vector<uint32_t> list = segments_of(img, W, H, threshold, seed);
    if (list.size() == 1 && list[0] == 0xDEADBEEFu) return -1;
    const long long mx = W > H ? W : H;
    const bool wide = 6ll * mx * W * H >= (1ll << 32);
    return wide ? reduce_image<true>(list, W, H, max_blobs, E, force_cta, xy, n_out, mom, flags)
                : reduce_image<false>(list, W, H, max_blobs, E, force_cta, xy, n_out, mom, flags);
}

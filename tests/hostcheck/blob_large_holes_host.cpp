// Test-only: the full-size S1 reduction (k_blob_reduce's 128-thread CTA) of csrc/blob_device.cuh run UNCHANGED on the
// host through simt_emu.h, with the whole-image window of the RETR_TREE slow path switched on (mocap_set_large_holes):
// the window lives in host memory here, as it lives in global memory on the device.  NOT part of libmocap_b200.so.
#include "blob_emu_host.cpp"

// img uint8 [H][W] -> what k_blob_reduce reports for it; large != 0: with the whole-image window.  Returns 2, or 0 for
// an image without a set pixel.
extern "C" int hc_blob_detect_large(const uint8_t* img, int W, int H, int threshold, int max_blobs, int E, int large, unsigned seed,
                                    int32_t* xy, int32_t* n_out, int64_t* mom, int32_t* flags) {
    const std::vector<uint32_t> list = segments_of(img, W, H, threshold, seed);
    if (list.size() == 1 && list[0] == 0xDEADBEEFu) return -1;
    const int cnt = (int)list.size();
    if (cnt == 0) { *n_out = 0; *flags = 0; return 0; }
    int fl = 0, n = cnt;
    if (cnt > E) { fl |= MOCAP_F_SEGMENTS; n = 0; }
    if (n == 0) { *n_out = 0; *flags = fl; return 2; }
    const long long mx = W > H ? W : H;
    const bool wide = 6ll * mx * W * H >= (1ll << 32);
    std::vector<unsigned long long> raw(blob_reduce_smem_bytes(E) / 8 + 2);
    std::vector<unsigned long long> win(large ? 4 * hole_wide_words(W, H) : 0);
    simt::launch(128, [&] {
        BlobSmem sm = carve_blob_smem(reinterpret_cast<unsigned char*>(raw.data()), E);
        if (large) sm.hole_win = win.data();
        for (int i = threadIdx.x; i < n; i += 128) sm.seg[i] = list[i];
        __syncthreads();
        if (wide) blob_reduce<128, false, true>(sm, n, E, MOCAP_ACC_CAP, W, H, max_blobs, xy, n_out, mom, flags, fl);
        else blob_reduce<128, false, false>(sm, n, E, MOCAP_ACC_CAP, W, H, max_blobs, xy, n_out, mom, flags, fl);
    });
    return 2;
}

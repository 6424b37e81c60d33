// Test-only host build of csrc/overlay.cuh (the detection overlay's drawing code), so that what the overlay kernels
// draw can be checked against cv2 on a machine without a GPU.  It walks images the way the kernels do: the contour
// layer from the grey plane of the undrawn frame, then every blob's label characters and plus.  NOT part of
// libmocap_b200.so and never used by the product path.
#include <stdint.h>
#include <vector>
#include "../../low-cost-mocap_b200/csrc/overlay.cuh"

extern "C" {
// frames [n][H][W][3] in place; blob_xy [n][MB][2], blob_n [n] (NULL: the contour layer only)
void hc_overlay(uint8_t* frames, int n, int W, int H, int MB, const int32_t* blob_xy, const int32_t* blob_n) {
    std::vector<uint8_t> g((size_t)W * H);
    for (int i = 0; i < n; ++i) {
        uint8_t* f = frames + (size_t)i * W * H * 3;
        for (size_t p = 0; p < g.size(); ++p) g[p] = (uint8_t)ov_gray(f + p * 3);
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x)
                if (ov_border(g.data(), W, H, x, y)) ov_put(f, W, H, x, y, OV_CONTOUR_0, OV_CONTOUR_1, OV_CONTOUR_2);
        if (!blob_xy) continue;
        const int nb = blob_n[i] < MB ? blob_n[i] : MB;
        for (int b = 0; b < nb; ++b) ov_marks(f, W, H, blob_xy[((size_t)i * MB + b) * 2], blob_xy[((size_t)i * MB + b) * 2 + 1]);
    }
}

// one label, or one plus, alone
void hc_label(uint8_t* frame, int W, int H, int x, int y) {
    for (int k = 0; ov_label_char(frame, W, H, x, y, k); ++k) {}
}
void hc_plus(uint8_t* frame, int W, int H, int x, int y) { ov_plus(frame, W, H, x, y); }

// one line of cv::line(img, p1, p2, colour, 1, LINE_8) with integer end points, or with 16.16 fixed-point ones (shift=16)
void hc_line(uint8_t* frame, int W, int H, int64_t x1, int64_t y1, int64_t x2, int64_t y2, int fixed) {
    if (fixed) ov_line_fx(frame, W, H, x1, y1, x2, y2);
    else ov_line(frame, W, H, x1, y1, x2, y2, OV_MARK_0, OV_MARK_1, OV_MARK_2);
}
}

extern "C" {
// drawlines' end points of a float32 line; 0 where the reference raises
int hc_epiline_ends(float a, float b, float c, int width, int64_t* y0, int64_t* y1) { return ov_epiline_ends(a, b, c, width, y0, y1); }
// np.random.RandomState(seed).randint(0, 255, (n, 3))
void hc_palette(uint32_t seed, int n, uint8_t* out) { ov_palette(seed, n, out); }
// one integer line drawn by `lanes` lanes one after another
void hc_line_lanes(uint8_t* frame, int W, int H, int64_t x1, int64_t y1, int64_t x2, int64_t y2, int lanes) {
    for (int l = 0; l < lanes; ++l) ov_line(frame, W, H, x1, y1, x2, y2, OV_MARK_0, OV_MARK_1, OV_MARK_2, l, lanes);
}
}

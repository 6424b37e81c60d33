// Test-only host build of csrc/live.cuh (the live loop's per-read step code), so that k_live_blobs's arithmetic can be
// checked on a machine without a GPU.  It walks a batch the way k_live_blobs does, one read after another.  NOT part of
// libmocap_b200.so and never used by the product path.
#include <stdint.h>
#include "../../low-cost-mocap_b200/csrc/live.cuh"

extern "C" {
// blob_xy [n][C][MB][2], blob_n / img_flags [n][C] -> cnt [n][C], first [n][C][2], gate / called [n], flags [n] (in/out
// when merge); frames [n][C][S][S][3] or NULL
void hc_live(const int32_t* blob_xy, const int32_t* blob_n, const int32_t* img_flags, int n, int C, int MB, int S, int have_blobs,
             int mode, int32_t* cnt, int32_t* first, uint8_t* gate, uint8_t* called, int32_t* flags, uint8_t* frames) {
    for (int r = 0; r < n; ++r) {
        const int32_t* xy = blob_xy + (size_t)r * C * MB * 2;
        live_read(C, MB, xy, blob_n + (size_t)r * C, img_flags + (size_t)r * C, have_blobs, mode & LIVE_LOCATE, mode & LIVE_TRIANGULATE,
                  cnt + (size_t)r * C, first + (size_t)r * C * 2, gate + r, called + r, flags + r);
        if (frames && have_blobs && (mode & LIVE_CAPTURE))
            for (int c = 0; c < C; ++c)
                live_dots(MB, xy + (size_t)c * MB * 2, blob_n[(size_t)r * C + c], S, frames + ((size_t)r * C + c) * S * S * 3);
    }
}
}

// Test-only host build of csrc/screen.cuh (the per-view screen of explicit correspondences), so that the rule can be
// checked against a numpy restatement on a machine without a GPU.  NOT part of libmocap_b200.so and never used by the
// product path.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../../low-cost-mocap_b200/csrc/screen.cuh"

extern "C" {
// obs [n][C][2], mask_in / mask_out [n][C], K [C][9], R [C][9], t [C][3] (row-major); stats [4] = views in, kept, dropped,
// rows emptied -- what k_screen_observations computes, row after row
void hc_screen(const double* obs, const uint8_t* mask_in, int n, int C, const double* K, const double* R, const double* t, double thr,
               uint8_t* mask_out, int32_t* stats) {
    ScreenCams* S = static_cast<ScreenCams*>(calloc(1, sizeof(ScreenCams)));
    for (int k = 0; k < C; ++k)
        for (int c = 0; c < C; ++c) screen_set_P(*S, k, c, K + 9 * k, R + 9 * c, t + 3 * c);
    for (int c = 0; c < C; ++c) screen_set_cam(*S, c, R + 9 * c, t + 3 * c, K[9 * c + 0], K[9 * c + 4], K[9 * c + 2], K[9 * c + 5]);
    memset(stats, 0, 4 * sizeof(int32_t));
    for (int f = 0; f < n; ++f) {
        unsigned Sm = 0u;
        for (int c = 0; c < C; ++c) Sm |= (mask_in[(size_t)f * C + c] ? 1u : 0u) << c;
        const unsigned out = screen_row(*S, obs + (size_t)f * C * 2, C, Sm, thr * thr);
        for (int c = 0; c < C; ++c) mask_out[(size_t)f * C + c] = (uint8_t)((out >> c) & 1u);
        const int nv = screen_popc(Sm), nk = screen_popc(out);
        stats[0] += nv; stats[1] += nk; stats[2] += nv - nk; stats[3] += (nv >= 2 && out == 0u) ? 1 : 0;
    }
    free(S);
}

// the two-bit mask of the p-th pair of the views S
unsigned hc_screen_pair(unsigned S, int p) { return screen_pair(S, p); }
}

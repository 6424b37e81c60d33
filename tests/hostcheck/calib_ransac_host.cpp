// Test-only host build of csrc/calib_ransac.cuh (sampler, 7-point solver, cv2's fundamental-matrix error, the
// per-pair selection rule), so that the RANSAC arithmetic can be checked against cv2 and numpy on a machine without
// a GPU.  NOT part of libmocap_b200.so and never used by the product path.
#include <stdint.h>
#include <string.h>
#include "../../low-cost-mocap_b200/csrc/calib_ransac.cuh"

struct HP4 { float x, y, z, w; };

extern "C" {
// q1, q2: 7 points (x, y interleaved) of view 1 / view 2; F [3][9]
int hc_seven_point(const double* q1, const double* q2, double* F) {
    double Fm[3][9];
    const int n = rs_seven_point(q1, q2, Fm);
    memcpy(F, Fm, sizeof(double) * 9 * n);
    return n;
}

// pts [n][4] = x1 y1 x2 y2
void hc_fm_error(const double* F, const double* pts, int n, double* err) {
    for (int i = 0; i < n; ++i) err[i] = rs_fm_error(F, pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3]);
}

void hc_inlier_mask(const double* F, const double* pts, int n, double thr, uint8_t* mask) {
    for (int i = 0; i < n; ++i) mask[i] = rs_is_inlier(F, pts[4 * i], pts[4 * i + 1], pts[4 * i + 2], pts[4 * i + 3], thr * thr);
}

// idx [count][7]: draw `attempt` of hypotheses h0 .. h0+count-1 of pair p
void hc_draw7(uint64_t seed, int p, int h0, int count, int attempt, int m, int* idx) {
    for (int k = 0; k < count; ++k) rs_draw7(seed, p, h0 + k, attempt, m, idx + 7 * k);
}

int hc_has_collinear(const double* q) { return rs_has_collinear(q) ? 1 : 0; }

// The per-pair RANSAC of k_ransac_hypotheses / k_ransac_score / k_ransac_mask stepped on the host: pts [m][4] float32,
// H hypotheses of pair p.  F_out [9] the winner, mask [m] its inliers, *count its inlier count; returns 0 if no
// hypothesis gave a model.
int hc_ransac_select(const float* pts, int m, int p, int H, uint64_t seed, double thr, double* F_out, uint8_t* mask, int* count) {
    const HP4* q = reinterpret_cast<const HP4*>(pts);
    const double thr2 = thr * thr;
    unsigned long long best = 0;
    for (int h = 0; h < H; ++h) {
        double F[3][9];
        const int n = rs_hypothesis(q, m, seed, p, h, F);
        for (int k = 0; k < n; ++k) {
            int c = 0;
            for (int i = 0; i < m; ++i) c += rs_is_inlier(F[k], q[i].x, q[i].y, q[i].z, q[i].w, thr2) ? 1 : 0;
            const unsigned long long key = rs_key(c, h, k);
            if (key > best) { best = key; memcpy(F_out, F[k], sizeof(F[k])); *count = c; }
        }
    }
    if (!best) return 0;
    for (int i = 0; i < m; ++i) mask[i] = rs_is_inlier(F_out, q[i].x, q[i].y, q[i].z, q[i].w, thr2) ? 1 : 0;
    return 1;
}

// Every model of hc_ransac_select's scan: n_models [H], counts [H][3] (-1 past a hypothesis' models), F [H][3][9]
void hc_ransac_models(const float* pts, int m, int p, int H, uint64_t seed, double thr, int* n_models, int* counts, double* F) {
    const HP4* q = reinterpret_cast<const HP4*>(pts);
    const double thr2 = thr * thr;
    for (int h = 0; h < H; ++h) {
        double Fh[3][9];
        const int n = rs_hypothesis(q, m, seed, p, h, Fh);
        n_models[h] = n;
        for (int k = 0; k < 3; ++k) {
            int c = -1;
            if (k < n) {
                c = 0;
                for (int i = 0; i < m; ++i) c += rs_is_inlier(Fh[k], q[i].x, q[i].y, q[i].z, q[i].w, thr2) ? 1 : 0;
                memcpy(F + 27 * (size_t)h + 9 * k, Fh[k], sizeof(Fh[k]));
            }
            counts[3 * h + k] = c;
        }
    }
}
}

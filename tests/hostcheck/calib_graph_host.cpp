// Test-only host build of csrc/calib_graph.cuh (the pose-graph cold start's arithmetic and host stages), so that it can
// be checked against numpy restatements on a machine without a GPU.  NOT part of libmocap_b200.so and never used by
// the product path.  hc_translations runs the device's translation stage with plain loops, track after track.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../low-cost-mocap_b200/csrc/calib_graph.cuh"

extern "C" {
// One track's contribution to the reduced translation system: obs [C][2], w [C] (0: view out), Kinv / R [C][9].
// H [3C][3C] (full, row-major) receives the block; returns 0 if the track does not enter (fewer than 2 views or a
// singular H_xx).
int hc_track_block(const double* obs, const double* w, const double* Kinv, const double* R, int C, double* H) {
    double N[CG_MAX_CAM][9], Q[CG_MAX_CAM][6], Hx[6] = {0, 0, 0, 0, 0, 0}, Hi[6];
    unsigned views = 0u;
    int nv = 0;
    for (int c = 0; c < C; ++c) {
        if (!(w[c] > 0.0)) continue;
        double x[3], RtQR[6];
        cg_bearing(Kinv + 9 * c, obs[2 * c], obs[2 * c + 1], x);
        cg_view_terms(x, w[c], R + 9 * c, Q[c], N[c], RtQR);
        for (int k = 0; k < 6; ++k) Hx[k] += RtQR[k];
        views |= 1u << c; ++nv;
    }
    const int n3 = 3 * C;
    memset(H, 0, sizeof(double) * n3 * n3);
    if (nv < 2 || !cg_inv_sym3(Hx, Hi)) return 0;
    for (int r = 0; r < n3; ++r)
        for (int col = 0; col < n3; ++col) {
            const int ca = r / 3, i = r % 3, cb = col / 3, j = col % 3;
            if (!((views >> ca) & 1u) || !((views >> cb) & 1u)) continue;
            double x = -cg_coupling(N[ca], Hi, N[cb], i, j);
            if (ca == cb) x += Q[ca][cg_s6(i, j)];
            H[r * n3 + col] = x;
        }
    return 1;
}

// Cheirality of one correspondence under the motion (R, t) with intrinsics Ka, Kb; front [1] out; returns the angle
double hc_cheirality(const double* Ka, const double* Kb, const double* R, const double* t, double xa, double ya, double xb, double yb,
                     int* front) {
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z3[3] = {0, 0, 0};
    double Pa[12], Pb[12];
    cg_make_P(Ka, I3, z3, Pa);
    cg_make_P(Kb, R, t, Pb);
    bool f;
    const double a = cg_cheirality_point(Pa, Pb, R, t, xa, ya, xb, yb, f);
    *front = f ? 1 : 0;
    return a;
}

void hc_motion_from_essential(const double* E, double* Rs /*[4][9]*/, double* ts /*[4][3]*/) {
    double R4[4][9], t4[4][3];
    calib_pose::motion_from_essential(E, R4, t4);
    memcpy(Rs, R4, sizeof(R4));
    memcpy(ts, t4, sizeof(t4));
}

// cg_rotation_average; returns 1 on success
int hc_rotation_average(int C, int P, const int* a, const int* b, const double* Rab, const double* w, double outlier_deg, uint8_t* use,
                        double* R, double* resid) {
    return cg_rotation_average(C, P, a, b, Rab, w, outlier_deg, use, R, resid) ? 1 : 0;
}

// The translation stage: obs [n][C][2], init [n][C] (views that enter), Kinv / R [C][9], f [C]; t [C][3] and the final
// weights w [n][C] out, in the gauge of mocap_calibrate_graph_host.  Returns 1 on success.
int hc_translations(const double* obs, const uint8_t* init, int n, int C, const double* Kinv, const double* R, const double* f, int rounds,
                    double scale_px, double* t, double* w_out) {
    const int n3 = 3 * C, E = n3 * (n3 + 1) / 2;
    std::vector<double> w((size_t)n * C), wn((size_t)n * C), Hu(E), H((size_t)n3 * n3);
    std::vector<uint8_t> front((size_t)n * C);
    for (size_t k = 0; k < w.size(); ++k) w[k] = init[k] ? 1.0 : 0.0;
    for (int round = 0; round < rounds; ++round) {
        std::fill(Hu.begin(), Hu.end(), 0.0);
        for (int p = 0; p < n; ++p) {
            if (!hc_track_block(obs + (size_t)p * C * 2, &w[(size_t)p * C], Kinv, R, C, H.data())) continue;
            for (int e = 0; e < E; ++e) { int r, c; cg_entry_rc(n3, e, r, c); Hu[e] += H[(size_t)r * n3 + c]; }
        }
        if (!cg_translation_solve(C, Hu.data(), t)) return 0;
        for (int p = 0; p < n; ++p) {
            double Hx[6] = {0, 0, 0, 0, 0, 0}, Hi[6], N[CG_MAX_CAM * 9];
            unsigned views = 0u;
            int nv = 0;
            for (int c = 0; c < C; ++c) {
                const double wv = w[(size_t)p * C + c];
                if (!(wv > 0.0)) continue;
                double x[3], Q[6], RtQR[6];
                cg_bearing(Kinv + 9 * c, obs[((size_t)p * C + c) * 2], obs[((size_t)p * C + c) * 2 + 1], x);
                cg_view_terms(x, wv, R + 9 * c, Q, N + 9 * c, RtQR);
                for (int k = 0; k < 6; ++k) Hx[k] += RtQR[k];
                views |= 1u << c; ++nv;
            }
            const bool ok = nv >= 2 && cg_inv_sym3(Hx, Hi);
            double X[3];
            if (ok) cg_track_point(Hi, N, t, views, C, X);
            for (int c = 0; c < C; ++c) {
                const size_t i = (size_t)p * C + c;
                wn[i] = 0.0; front[i] = 0;
                if (!init[i] || !ok) continue;
                double x[3];
                bool fb;
                cg_bearing(Kinv + 9 * c, obs[2 * i], obs[2 * i + 1], x);
                wn[i] = cg_cauchy(cg_view_residual_px(x, R + 9 * c, t + 3 * c, X, f[c], fb), scale_px);
                front[i] = fb ? 1 : 0;
            }
        }
        w.swap(wn);
    }
    long nf = 0, nb = 0;
    for (int p = 0; p < n; ++p) {
        int k = 0;
        for (int c = 0; c < C; ++c) k += w[(size_t)p * C + c] >= 0.5 ? 1 : 0;
        if (k < 2) continue;
        for (int c = 0; c < C; ++c) {
            const size_t i = (size_t)p * C + c;
            if (w[i] >= 0.5) { if (front[i]) ++nf; else ++nb; }
        }
    }
    cg_gauge(C, t, nf, nb);
    memcpy(w_out, w.data(), w.size() * sizeof(double));
    return 1;
}
}

// Arithmetic of the pose-graph cold start (calib_graph.cu), usable from device code and, for the host checks in
// tests/hostcheck, from g++.
//
// Per pair (a, b): the candidate motions of E = K_b^T F K_a are judged in the pair's own frame, P_a = K_a [I|0] and
// P_b = K_b [R_q|t_q]: a correspondence counts for q when its DLT point has positive depth in both cameras
// (cg_cheirality_point), and its triangulation angle -- between the rays from the two camera centres -- is returned so
// that near-opposed pairs, whose points are seen at a grazing angle, can be dropped.
//
// Translations with the rotations R_c known: view c of a track with bearing x = normalise(K_c^-1 [u v 1]) gives
// [x]_x (R_c X + t_c) = 0.  Weighted by w, its normal equations in (X, t_c) hold Q_c = w (I - x x^T) (= w [x]_x^T
// [x]_x for a unit x), H_xx += R_c^T Q_c R_c, H_xt_c = R_c^T Q_c = N_c^T with N_c = Q_c R_c, H_tt_cc = Q_c.  Eliminating
// X (Schur complement) leaves, per track, the 3C x 3C block (a, b) = delta_ab Q_a - N_a H_xx^-1 N_b^T, summed over the
// tracks into the reduced system of the translations; its smallest eigenvector with t_0 = 0 is the rig's translations
// up to scale.  The point is X = -H_xx^-1 sum_c N_c^T t_c.
#pragma once
#include <math.h>
#include <stdint.h>
#include "geom.cuh"

#define CG_MAX_CAM 16

// symmetric 3x3 as 6 entries: 00 01 02 11 12 22
GEOM_HD int cg_s6(int i, int j) { return i <= j ? (i == 0 ? j : (i == 1 ? 2 + j : 5)) : (j == 0 ? i : (j == 1 ? 2 + i : 5)); }

// x = normalise(Kinv [u v 1])
GEOM_HD void cg_bearing(const double* Kinv, double u, double v, double x[3]) {
    double r[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) r[i] = Kinv[3 * i] * u + Kinv[3 * i + 1] * v + Kinv[3 * i + 2];
    const double nr = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) x[i] = r[i] / nr;
}

// Q = w (I - x x^T) (6 entries), N = Q R (3x3 row-major), RtQR = R^T Q R (6 entries)
GEOM_HD void cg_view_terms(const double x[3], double w, const double* R, double Q[6], double N[9], double RtQR[6]) {
    Q[0] = w * (1.0 - x[0] * x[0]); Q[1] = -w * x[0] * x[1]; Q[2] = -w * x[0] * x[2];
    Q[3] = w * (1.0 - x[1] * x[1]); Q[4] = -w * x[1] * x[2]; Q[5] = w * (1.0 - x[2] * x[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            N[3 * i + j] = Q[cg_s6(i, 0)] * R[j] + Q[cg_s6(i, 1)] * R[3 + j] + Q[cg_s6(i, 2)] * R[6 + j];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = i; j < 3; ++j) RtQR[cg_s6(i, j)] = R[i] * N[j] + R[3 + i] * N[3 + j] + R[6 + i] * N[6 + j];
}

// inverse of a symmetric positive 3x3 by its adjugate; false when it is (numerically) singular -- a track whose
// weighted views do not fix its point
GEOM_HD bool cg_inv_sym3(const double H[6], double Hi[6]) {
    const double c00 = H[3] * H[5] - H[4] * H[4], c01 = H[2] * H[4] - H[1] * H[5], c02 = H[1] * H[4] - H[2] * H[3];
    const double c11 = H[0] * H[5] - H[2] * H[2], c12 = H[1] * H[2] - H[0] * H[4], c22 = H[0] * H[3] - H[1] * H[1];
    const double det = H[0] * c00 + H[1] * c01 + H[2] * c02;
    const double tr = H[0] + H[3] + H[5];
    if (!(tr > 0.0) || !(det > 1e-9 * tr * tr * tr)) return false;
    const double id = 1.0 / det;
    Hi[0] = c00 * id; Hi[1] = c01 * id; Hi[2] = c02 * id; Hi[3] = c11 * id; Hi[4] = c12 * id; Hi[5] = c22 * id;
    return true;
}

// (N_a Hi N_b^T)[i][j]
GEOM_HD double cg_coupling(const double* Na, const double Hi[6], const double* Nb, int i, int j) {
    double h[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) h[k] = Hi[cg_s6(k, 0)] * Nb[3 * j] + Hi[cg_s6(k, 1)] * Nb[3 * j + 1] + Hi[cg_s6(k, 2)] * Nb[3 * j + 2];
    return Na[3 * i] * h[0] + Na[3 * i + 1] * h[1] + Na[3 * i + 2] * h[2];
}

// The track's point X = -Hi sum_c N_c^T t_c over the views of `views` (bit c); N [C][9], t [C][3]
GEOM_HD void cg_track_point(const double Hi[6], const double* N, const double* t, unsigned views, int C, double X[3]) {
    double g[3] = {0.0, 0.0, 0.0};
    for (int c = 0; c < C; ++c) {
        if (!((views >> c) & 1u)) continue;
        const double* Nc = N + 9 * c;
#pragma unroll
        for (int k = 0; k < 3; ++k) g[k] += Nc[k] * t[3 * c] + Nc[3 + k] * t[3 * c + 1] + Nc[6 + k] * t[3 * c + 2];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) X[k] = -(Hi[cg_s6(k, 0)] * g[0] + Hi[cg_s6(k, 1)] * g[1] + Hi[cg_s6(k, 2)] * g[2]);
}

// Angular residual of a view against the point X, in pixels (sine of the angle between x and R X + t, times the focal
// length; the same for X and -X, so it does not depend on the sign of the translations), and whether the point lies
// in front of the camera.
GEOM_HD double cg_view_residual_px(const double x[3], const double* R, const double* t, const double X[3], double f, bool& front) {
    double p[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) p[i] = R[3 * i] * X[0] + R[3 * i + 1] * X[1] + R[3 * i + 2] * X[2] + t[i];
    const double cx = x[1] * p[2] - x[2] * p[1], cy = x[2] * p[0] - x[0] * p[2], cz = x[0] * p[1] - x[1] * p[0];
    const double np = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    front = p[2] > 0.0;
    return np > 0.0 ? f * sqrt(cx * cx + cy * cy + cz * cz) / np : 0.0;
}

// Cauchy weight of a residual at scale s px
GEOM_HD double cg_cauchy(double r, double s) { const double z = r / s; return 1.0 / (1.0 + z * z); }

// Cheirality of one correspondence under one candidate (R, t) of the pair's relative motion: DLT point X in camera
// a's frame from Pa = K_a [I|0] and Pb = K_b [R|t]; front when X_z > 0 and (R X + t)_z > 0.  Returns the triangulation
// angle in degrees, the angle at X between the rays to the camera centres 0 and -R^T t.
GEOM_HD double cg_cheirality_point(const double* Pa, const double* Pb, const double* R, const double* t, double xa, double ya,
                                   double xb, double yb, bool& front) {
    Sym4 B;
    sym4_zero(B);
    dlt_add_view(B, Pa, xa, ya);
    dlt_add_view(B, Pb, xb, yb);
    double X[3];
    dlt_solve(B, X);
    const double zb = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
    front = X[2] > 0.0 && zb > 0.0;
    double cb[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) cb[i] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
    const double u[3] = {X[0], X[1], X[2]}, v[3] = {X[0] - cb[0], X[1] - cb[1], X[2] - cb[2]};
    const double nu = sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    double c = (u[0] * v[0] + u[1] * v[1] + u[2] * v[2]) / (nu * nv);
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    return acos(c) * (180.0 / 3.14159265358979323846);
}

// Upper-triangle index e of the reduced system (row-major over r <= c of a 3C x 3C matrix) -> (r, c)
GEOM_HD void cg_entry_rc(int n, int e, int& r, int& c) {
    r = 0;
    while (e >= n - r) { e -= n - r; ++r; }
    c = r + e;
}

// P = K [R|t]
GEOM_HD void cg_make_P(const double* K, const double* R, const double* t, double P[12]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 4; ++j) {
            double a = 0.0;
            for (int k = 0; k < 3; ++k) a += K[3 * i + k] * (j < 3 ? R[3 * k + j] : t[k]);
            P[4 * i + j] = a;
        }
}

// ---------------------------------------------------------------------------------------------------------------------
// Host stages (at most 16 cameras, 120 pairs)
#include <vector>
#include "calib_pose.h"
#include "trf_core.h"

// Cholesky solve of the SPD system M X = B (n x n, B n x k, both row-major, overwritten); false if M is not SPD
inline bool cg_cholesky_solve(int n, std::vector<double>& M, std::vector<double>& B, int k) {
    for (int j = 0; j < n; ++j) {
        double d = M[(size_t)j * n + j];
        for (int p = 0; p < j; ++p) d -= M[(size_t)j * n + p] * M[(size_t)j * n + p];
        if (!(d > 0.0)) return false;
        d = sqrt(d);
        M[(size_t)j * n + j] = d;
        for (int i = j + 1; i < n; ++i) {
            double s = M[(size_t)i * n + j];
            for (int p = 0; p < j; ++p) s -= M[(size_t)i * n + p] * M[(size_t)j * n + p];
            M[(size_t)i * n + j] = s / d;
        }
    }
    for (int c = 0; c < k; ++c) {
        for (int i = 0; i < n; ++i) {
            double s = B[(size_t)i * k + c];
            for (int p = 0; p < i; ++p) s -= M[(size_t)i * n + p] * B[(size_t)p * k + c];
            B[(size_t)i * k + c] = s / M[(size_t)i * n + i];
        }
        for (int i = n - 1; i >= 0; --i) {
            double s = B[(size_t)i * k + c];
            for (int p = i + 1; p < n; ++p) s -= M[(size_t)p * n + i] * B[(size_t)p * k + c];
            B[(size_t)i * k + c] = s / M[(size_t)i * n + i];
        }
    }
    return true;
}

// angle of R_b R_a^T against R_ab, degrees
inline double cg_rot_residual_deg(const double* Ra, const double* Rb, const double* Rab) {
    double tr = 0.0;          // trace(R_ab^T R_b R_a^T)
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double m = 0.0;   // (R_b R_a^T)[i][j]
            for (int k = 0; k < 3; ++k) m += Rb[3 * i + k] * Ra[3 * j + k];
            tr += Rab[3 * i + j] * m;
        }
    double c = 0.5 * (tr - 1.0);
    c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
    return acos(c) * (180.0 / 3.14159265358979323846);
}

// Cameras not connected to camera 0 by the pairs with use[p] set: bit c of the result
inline unsigned cg_disconnected(int C, int P, const int* a, const int* b, const uint8_t* use) {
    unsigned reach = 1u;
    for (bool grew = true; grew;) {
        grew = false;
        for (int p = 0; p < P; ++p) {
            if (!use[p]) continue;
            const unsigned ma = 1u << a[p], mb = 1u << b[p];
            if ((reach & ma) && !(reach & mb)) { reach |= mb; grew = true; }
            if ((reach & mb) && !(reach & ma)) { reach |= ma; grew = true; }
        }
    }
    return ((C >= 32 ? 0u : (1u << C)) - 1u) & ~reach;
}

// One weighted chordal least-squares solve of R_b = R_ab R_a over the pairs with w[p] > 0, R_0 = I, each result
// projected onto SO(3).  R [C][9] out.  false if the normal equations are singular (pairs do not connect the rig).
inline bool cg_chordal_solve(int C, int P, const int* a, const int* b, const double* Rab, const double* w, double* R) {
    const int n = 3 * (C - 1);
    std::vector<double> M((size_t)n * n, 0.0), B((size_t)n * 3, 0.0);
    for (int p = 0; p < P; ++p) {
        if (!(w[p] > 0.0)) continue;
        // for each row i: r_{b,i} - sum_k Rab[i][k] r_{a,k} = 0, unknown rows r_{c,i} of R_c (c >= 1)
        for (int i = 0; i < 3; ++i) {
            int idx[4]; double g[4]; double known[3] = {0.0, 0.0, 0.0}; int m = 0;
            if (b[p] > 0) { idx[m] = 3 * (b[p] - 1) + i; g[m++] = 1.0; } else known[i] += 1.0;
            for (int k = 0; k < 3; ++k) {
                const double coef = -Rab[9 * p + 3 * i + k];
                if (a[p] > 0) { idx[m] = 3 * (a[p] - 1) + k; g[m++] = coef; } else known[k] += coef;
            }
            for (int u = 0; u < m; ++u) {
                for (int v = 0; v < m; ++v) M[(size_t)idx[u] * n + idx[v]] += w[p] * g[u] * g[v];
                for (int col = 0; col < 3; ++col) B[(size_t)idx[u] * 3 + col] -= w[p] * g[u] * known[col];
            }
        }
    }
    if (!cg_cholesky_solve(n, M, B, 3)) return false;
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    for (int c = 1; c < C; ++c) {
        double A[9], U[9], s[3], V[9];
        for (int i = 0; i < 9; ++i) A[i] = B[(size_t)(3 * (c - 1)) * 3 + i];       // rows r_{c,0..2}
        calib_pose::svd3(A, U, s, V);
        double Rc[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) Rc[3 * i + j] = U[3 * i] * V[3 * j] + U[3 * i + 1] * V[3 * j + 1] + U[3 * i + 2] * V[3 * j + 2];
        if (calib_pose::det3m(Rc) < 0.0)
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) Rc[3 * i + j] -= 2.0 * U[3 * i + 2] * V[3 * j + 2];
        for (int i = 0; i < 9; ++i) R[9 * c + i] = Rc[i];
    }
    return true;
}

#define CG_ROT_IRLS_ROUNDS 5

// Rotation averaging: weighted chordal least squares (weight w0[p], the pair's inliers), then CG_ROT_IRLS_ROUNDS rounds
// of Cauchy weights w0 / (1 + (residual / outlier_deg)^2) on the angular residual; pairs with a final residual above
// outlier_deg are marked unused (use[p] = 0) and the rotations re-solved on the others.  use[p] in: 1 for the pairs
// that enter.  resid_deg [P] out: every pair's residual against the final rotations.  Returns false if the pairs left
// do not connect every camera (use[] then says which pairs were left).
inline bool cg_rotation_average(int C, int P, const int* a, const int* b, const double* Rab, const double* w0, double outlier_deg,
                                uint8_t* use, double* R, double* resid_deg) {
    std::vector<double> w(P);
    for (int p = 0; p < P; ++p) w[p] = use[p] ? w0[p] : 0.0;
    if (cg_disconnected(C, P, a, b, use) || !cg_chordal_solve(C, P, a, b, Rab, w.data(), R)) return false;
    for (int round = 0; round < CG_ROT_IRLS_ROUNDS; ++round) {
        for (int p = 0; p < P; ++p)
            if (use[p]) w[p] = w0[p] * cg_cauchy(cg_rot_residual_deg(R + 9 * a[p], R + 9 * b[p], Rab + 9 * p), outlier_deg);
        if (!cg_chordal_solve(C, P, a, b, Rab, w.data(), R)) return false;
    }
    for (int p = 0; p < P; ++p)
        if (use[p] && cg_rot_residual_deg(R + 9 * a[p], R + 9 * b[p], Rab + 9 * p) > outlier_deg) use[p] = 0;
    for (int p = 0; p < P; ++p) w[p] = use[p] ? w0[p] : 0.0;
    if (cg_disconnected(C, P, a, b, use) || !cg_chordal_solve(C, P, a, b, Rab, w.data(), R)) return false;
    for (int p = 0; p < P; ++p) resid_deg[p] = cg_rot_residual_deg(R + 9 * a[p], R + 9 * b[p], Rab + 9 * p);
    return true;
}

// Translations from the reduced system: Hu holds its upper triangle (3C(3C+1)/2 entries).  t [C][3] out: t_0 = 0 and
// the smallest eigenvector of the 3(C-1) block of the other cameras, unit norm, sign unspecified.  false if the eigen
// problem fails.
inline bool cg_translation_solve(int C, const double* Hu, double* t) {
    const int n3 = 3 * C, n = n3 - 3;
    std::vector<double> A((size_t)n * n), lam;
    for (int e = 0, E = n3 * (n3 + 1) / 2; e < E; ++e) {
        int r, c;
        cg_entry_rc(n3, e, r, c);
        if (r < 3 || c < 3) continue;
        A[(size_t)(r - 3) * n + (c - 3)] = Hu[e];
        A[(size_t)(c - 3) * n + (r - 3)] = Hu[e];
    }
    if (!trf::sym_eig(n, A, lam)) return false;
    int best = 0;
    for (int i = 1; i < n; ++i) if (lam[i] < lam[best]) best = i;
    t[0] = t[1] = t[2] = 0.0;
    for (int i = 0; i < n; ++i) t[3 + i] = A[(size_t)i * n + best];
    return true;
}

// The chain's gauge: flip the sign when fewer views see their point in front than behind, then scale to |t_1| = 1
inline void cg_gauge(int C, double* t, long n_front, long n_back) {
    const double sgn = n_back > n_front ? -1.0 : 1.0;
    const double n1 = sqrt(t[3] * t[3] + t[4] * t[4] + t[5] * t[5]);
    const double s = n1 > 0.0 ? sgn / n1 : sgn;
    for (int i = 0; i < 3 * C; ++i) t[i] *= s;
}

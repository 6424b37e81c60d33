// Host algebra of the cold-start calibration (calib_init.cu, calib_graph.cu and the g++ host checks): symmetric 3x3
// eigen-decomposition, SVD, libmv's MotionFromEssential, and the normalised 8-point fit's Hartley transform and solve.
// Plain C++, no CUDA.
#pragma once
#include <math.h>
#include <stdint.h>
#include <vector>
#include "trf_core.h"

namespace calib_pose {

// symmetric 3x3 eigen-decomposition (cyclic Jacobi); eigenvalues descending, eigenvectors as columns of V
inline void eig3(const double A[9], double w[3], double V[9]) {
    double a[3][3] = {{A[0], A[1], A[2]}, {A[3], A[4], A[5]}, {A[6], A[7], A[8]}};
    double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 60; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
        if (off == 0.0) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (a[p][q] == 0.0) continue;
                const double theta = 0.5 * (a[q][q] - a[p][p]) / a[p][q];
                double t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));
                if (theta < 0) t = -t;
                const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
                for (int k = 0; k < 3; ++k) { const double x = a[k][p], y = a[k][q]; a[k][p] = c * x - s * y; a[k][q] = s * x + c * y; }
                for (int k = 0; k < 3; ++k) { const double x = a[p][k], y = a[q][k]; a[p][k] = c * x - s * y; a[q][k] = s * x + c * y; }
                for (int k = 0; k < 3; ++k) { const double x = v[k][p], y = v[k][q]; v[k][p] = c * x - s * y; v[k][q] = s * x + c * y; }
            }
    }
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 2; ++i) for (int j = i + 1; j < 3; ++j) if (a[o[j]][o[j]] > a[o[i]][o[i]]) { const int tmp = o[i]; o[i] = o[j]; o[j] = tmp; }
    for (int k = 0; k < 3; ++k) { w[k] = a[o[k]][o[k]]; for (int r = 0; r < 3; ++r) V[3 * r + k] = v[r][o[k]]; }
}

// M = U diag(s) V^T for a 3x3 matrix (row-major), s descending, via the eigen-decomposition of M^T M
inline void svd3(const double M[9], double U[9], double s[3], double V[9]) {
    double MtM[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double x = 0; for (int k = 0; k < 3; ++k) x += M[3 * k + i] * M[3 * k + j]; MtM[3 * i + j] = x; }
    double w[3];
    eig3(MtM, w, V);
    for (int k = 0; k < 3; ++k) s[k] = sqrt(fmax(w[k], 0.0));
    double u[3][3];
    for (int k = 0; k < 2; ++k) {
        for (int r = 0; r < 3; ++r) { double x = 0; for (int c = 0; c < 3; ++c) x += M[3 * r + c] * V[3 * c + k]; u[k][r] = x; }
        double nrm = sqrt(u[k][0] * u[k][0] + u[k][1] * u[k][1] + u[k][2] * u[k][2]);
        if (nrm == 0.0) nrm = 1.0;
        for (int r = 0; r < 3; ++r) u[k][r] /= nrm;
    }
    // second column re-orthogonalised against the first, third = u1 x u2 (covers the rank-2 case)
    const double d = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2];
    for (int r = 0; r < 3; ++r) u[1][r] -= d * u[0][r];
    double n2 = sqrt(u[1][0] * u[1][0] + u[1][1] * u[1][1] + u[1][2] * u[1][2]);
    if (n2 == 0.0) n2 = 1.0;
    for (int r = 0; r < 3; ++r) u[1][r] /= n2;
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    // sign of the third pair: make it consistent with M v3 when s3 is not negligible
    double mv[3];
    for (int r = 0; r < 3; ++r) { mv[r] = 0; for (int c = 0; c < 3; ++c) mv[r] += M[3 * r + c] * V[3 * c + 2]; }
    if (mv[0] * u[2][0] + mv[1] * u[2][1] + mv[2] * u[2][2] < 0) for (int r = 0; r < 3; ++r) V[3 * r + 2] = -V[3 * r + 2];
    for (int k = 0; k < 3; ++k) for (int r = 0; r < 3; ++r) U[3 * r + k] = u[k][r];
}

inline double det3m(const double A[9]) {
    return A[0] * (A[4] * A[8] - A[5] * A[7]) - A[1] * (A[3] * A[8] - A[5] * A[6]) + A[2] * (A[3] * A[7] - A[4] * A[6]);
}

inline void mat3mul(const double A[9], const double B[9], double C[9]) {
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double x = 0; for (int k = 0; k < 3; ++k) x += A[3 * i + k] * B[3 * k + j]; C[3 * i + j] = x; }
}

// Sign of a fitted F (9 entries): the entry of largest magnitude made positive (the first of equal magnitudes).  The
// smallest eigenvector's sign is otherwise whatever the eigen solver's rounding makes it: two summation orders of the
// same normal matrix (the device's and a host model's, or two runs under floating-point atomics) can give opposite
// signs, and with them the four motions of E in another order.
inline void fix_sign(double F[9]) {
    int k = 0;
    for (int i = 1; i < 9; ++i) if (fabs(F[i]) > fabs(F[k])) k = i;
    if (F[k] < 0) for (int i = 0; i < 9; ++i) F[i] = -F[i];
}

// libmv MotionFromEssential (cv.sfm.motionFromEssential, index.py:248): Rs = [UWV^T, UWV^T, UW^TV^T, UW^TV^T],
// ts = [u3, -u3, u3, -u3], after flipping the last column of U / last row of V^T when their determinant is negative
inline void motion_from_essential(const double E[9], double Rs[4][9], double ts[4][3]) {
    double U[9], s[3], V[9], Vt[9];
    svd3(E, U, s, V);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Vt[3 * i + j] = V[3 * j + i];
    if (det3m(U) < 0) for (int r = 0; r < 3; ++r) U[3 * r + 2] = -U[3 * r + 2];
    if (det3m(Vt) < 0) for (int c = 0; c < 3; ++c) Vt[6 + c] = -Vt[6 + c];
    const double W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1}, Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
    double UW[9], UWt[9], A[9], Bm[9];
    mat3mul(U, W, UW); mat3mul(UW, Vt, A);
    mat3mul(U, Wt, UWt); mat3mul(UWt, Vt, Bm);
    for (int k = 0; k < 9; ++k) { Rs[0][k] = A[k]; Rs[1][k] = A[k]; Rs[2][k] = Bm[k]; Rs[3][k] = Bm[k]; }
    for (int r = 0; r < 3; ++r) { ts[0][r] = U[3 * r + 2]; ts[1][r] = -U[3 * r + 2]; ts[2][r] = U[3 * r + 2]; ts[3][r] = -U[3 * r + 2]; }
}

// Hartley normalisation of a pair's fit set: pts [m][4] {x_a, y_a, x_b, y_b}, inl [m] the set (not empty).  T = {s_a,
// tx_a, ty_a, s_b, tx_b, ty_b}: per view x' = s x + tx, y' = s y + ty moves the set's centroid to 0 and its mean
// distance from it to sqrt(2).
inline void hartley(const float* pts, int m, const uint8_t* inl, double T[6]) {
    for (int side = 0; side < 2; ++side) {
        double cx = 0, cy = 0; int k = 0;
        for (int i = 0; i < m; ++i)
            if (inl[i]) { cx += pts[4 * i + 2 * side]; cy += pts[4 * i + 2 * side + 1]; ++k; }
        cx /= k; cy /= k;
        double md = 0;
        for (int i = 0; i < m; ++i)
            if (inl[i]) {
                const double x = pts[4 * i + 2 * side], y = pts[4 * i + 2 * side + 1];
                md += sqrt((x - cx) * (x - cx) + (y - cy) * (y - cy));
            }
        md /= k;
        const double sc = md > 0 ? sqrt(2.0) / md : 1.0;
        T[3 * side] = sc; T[3 * side + 1] = -sc * cx; T[3 * side + 2] = -sc * cy;
    }
}

// F (x_b^T F x_a = 0) from the 45-entry upper triangle of the 8-point normal matrix in the coordinates of hartley()'s T:
// smallest eigenvector, rank 2, de-normalised, unit norm, fix_sign.  False (F untouched) if the eigen problem fails.
inline bool fit_from_normal(const double* up, const double T[6], double F[9]) {
    std::vector<double> A(81), lam;
    int k = 0;
    for (int r = 0; r < 9; ++r) for (int c = r; c < 9; ++c) { A[9 * r + c] = up[k]; A[9 * c + r] = up[k]; ++k; }
    if (!trf::sym_eig(9, A, lam)) return false;
    int best = 0;
    for (int i = 1; i < 9; ++i) if (lam[i] < lam[best]) best = i;
    double Fn[9], U[9], sv[3], V[9], Fr[9], tmp[9];
    for (int i = 0; i < 9; ++i) Fn[i] = A[9 * i + best];
    svd3(Fn, U, sv, V);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Fr[3 * i + j] = U[3 * i] * sv[0] * V[3 * j] + U[3 * i + 1] * sv[1] * V[3 * j + 1];
    // F = T_b^T Fr T_a with T = [[s,0,tx],[0,s,ty],[0,0,1]]
    const double M1[9] = {T[0], 0, T[1], 0, T[0], T[2], 0, 0, 1}, M2t[9] = {T[3], 0, 0, 0, T[3], 0, T[4], T[5], 1};
    mat3mul(M2t, Fr, tmp); mat3mul(tmp, M1, F);
    double nf = 0; for (int i = 0; i < 9; ++i) nf += F[i] * F[i];
    nf = sqrt(nf); if (nf > 0) for (int i = 0; i < 9; ++i) F[i] /= nf;
    fix_sign(F);
    return true;
}

}  // namespace calib_pose

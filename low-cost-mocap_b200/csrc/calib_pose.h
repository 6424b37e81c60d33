// Host 3x3 algebra of the cold-start calibration (calib_init.cu, calib_graph.cu and the g++ host checks): symmetric
// eigen-decomposition, SVD, and libmv's MotionFromEssential.  Plain C++, no CUDA.
#pragma once
#include <math.h>

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

}  // namespace calib_pose

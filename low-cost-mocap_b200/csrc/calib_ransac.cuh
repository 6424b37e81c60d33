// Robust fundamental matrix (RANSAC) for the cold-start calibration: the pieces one hypothesis needs, usable from
// device code (csrc/calib_ransac.cu) and, for the host-side checks in tests/hostcheck, from plain C++.
//
// The reference estimates each adjacent pair's F with cv.findFundamentalMat(FM_RANSAC, 1 px, 0.99999)
// (computer_code/api/index.py:246).  cv2 seeds its RANSAC generator with a fixed state, so that call is repeatable,
// but its sample sequence is not replayed here; what is kept is the estimator:
//   * a sample is 7 distinct correspondences, drawn from a counter-based hash of (seed, pair, hypothesis, attempt)
//     -- no generator state is carried from one hypothesis to the next, so the draws do not depend on the launch
//     geometry -- and redrawn while three of its points are collinear in either view (cv2's checkSubset);
//   * the 7-point minimal solver: the 2-D null space of the 7x9 epipolar system on Hartley-normalised points, and
//     the real roots of det(l F1 + (1 - l) F2) = 0, giving 1 to 3 models;
//   * cv2's fundamental-matrix error: the larger of the squared distances of x2 to the line F x1 and of x1 to the
//     line F^T x2; a point is an inlier when that is <= thr^2.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define RS_HD __host__ __device__ __forceinline__
#else
#define RS_HD static inline
#endif

#define RS_MAX_ATTEMPTS 100     // draws per hypothesis before it gives up (cv2's getSubset allows 1000 for its loop)
#define RS_PIVOT_EPS    1e-10   // relative pivot below which a 7-point sample is degenerate

// ------------------------------------------------------------------------------------------------ sampler
RS_HD uint64_t rs_mix64(uint64_t z) {          // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    return z ^ (z >> 31);
}

RS_HD uint64_t rs_mulhi(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// 7 distinct indices in [0, m) (m >= 7) for draw `attempt` of hypothesis h of pair p: a splitmix64 stream started
// from a hash of the key; index = floor(m * u) with u the 64-bit output read as a fraction
RS_HD void rs_draw7(uint64_t seed, int p, int h, int attempt, int m, int idx[7]) {
    uint64_t s = rs_mix64(seed ^ rs_mix64(((uint64_t)(uint32_t)p << 32) ^ (uint32_t)h) ^ ((uint64_t)(uint32_t)attempt << 17));
    for (int k = 0; k < 7; ++k) {
        int v;
        bool dup;
        do {
            s += 0x9e3779b97f4a7c15ULL;
            v = (int)rs_mulhi(rs_mix64(s), (uint64_t)m);
            dup = false;
            for (int j = 0; j < k; ++j) dup |= idx[j] == v;
        } while (dup);
        idx[k] = v;
    }
}

// cv2's haveCollinearPoints over every triple of the 7 points (x, y interleaved): also true for repeated points
RS_HD bool rs_has_collinear(const double q[14]) {
    for (int i = 2; i < 7; ++i)
        for (int j = 0; j < i; ++j) {
            const double dx1 = q[2 * j] - q[2 * i], dy1 = q[2 * j + 1] - q[2 * i + 1];
            for (int k = 0; k < j; ++k) {
                const double dx2 = q[2 * k] - q[2 * i], dy2 = q[2 * k + 1] - q[2 * i + 1];
                if (fabs(dx2 * dy1 - dy2 * dx1) <= 1.1920928955078125e-07 * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2)))
                    return true;
            }
        }
    return false;
}

// ------------------------------------------------------------------------------------------------ 7-point solver
RS_HD double rs_det3(const double a[9]) {
    return a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) + a[2] * (a[3] * a[7] - a[4] * a[6]);
}

// determinant of the matrix whose columns are taken from A (bit k of `from_b` clear) or B (set)
RS_HD double rs_det3_mixed(const double A[9], const double B[9], int from_b) {
    double M[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) M[3 * r + c] = ((from_b >> c) & 1) ? B[3 * r + c] : A[3 * r + c];
    return rs_det3(M);
}

RS_HD double rs_poly3(const double c[4], double x) { return ((c[3] * x + c[2]) * x + c[1]) * x + c[0]; }

// real roots of c[3] x^3 + c[2] x^2 + c[1] x + c[0]; a leading coefficient that vanishes relative to the others
// drops the degree.  Returns the number of roots (0..3), each polished by Newton steps that lower |p(x)|.
RS_HD int rs_real_roots(const double c[4], double x[3]) {
    const double cmax = fmax(fmax(fabs(c[0]), fabs(c[1])), fmax(fabs(c[2]), fabs(c[3])));
    if (cmax == 0.0) return 0;
    const double tiny = 1e-12 * cmax;
    int n = 0;
    if (fabs(c[3]) > tiny) {
        // x^3 + a1 x^2 + a2 x + a3 (the trigonometric / Cardano split of cv2's solveCubic)
        const double a1 = c[2] / c[3], a2 = c[1] / c[3], a3 = c[0] / c[3];
        const double Q = (a1 * a1 - 3 * a2) * (1.0 / 9), R = (2 * a1 * a1 * a1 - 9 * a1 * a2 + 27 * a3) * (1.0 / 54);
        const double Qc = Q * Q * Q, d = Qc - R * R;
        if (d > 0) {
            const double theta = acos(fmin(fmax(R / sqrt(Qc), -1.0), 1.0)), t0 = -2 * sqrt(Q), t2 = a1 * (1.0 / 3);
            x[0] = t0 * cos(theta * (1.0 / 3)) - t2;
            x[1] = t0 * cos((theta + 2 * 3.14159265358979323846) * (1.0 / 3)) - t2;
            x[2] = t0 * cos((theta + 4 * 3.14159265358979323846) * (1.0 / 3)) - t2;
            n = 3;
        } else {
            double e = cbrt(sqrt(-d) + fabs(R));
            if (R > 0) e = -e;
            x[0] = (e == 0.0 ? 0.0 : e + Q / e) - a1 * (1.0 / 3);
            n = 1;
        }
    } else if (fabs(c[2]) > tiny) {
        const double disc = c[1] * c[1] - 4 * c[2] * c[0];
        if (disc < 0) return 0;
        const double q = -0.5 * (c[1] + (c[1] >= 0 ? sqrt(disc) : -sqrt(disc)));
        x[0] = q / c[2];
        n = 1;
        if (q != 0.0) x[n++] = c[0] / q;
    } else if (fabs(c[1]) > tiny) {
        x[0] = -c[0] / c[1];
        n = 1;
    }
    for (int k = 0; k < n; ++k)
        for (int it = 0; it < 2; ++it) {
            const double p = rs_poly3(c, x[k]), dp = (3 * c[3] * x[k] + 2 * c[2]) * x[k] + c[1];
            if (dp == 0.0) break;
            const double y = x[k] - p / dp;
            if (!(fabs(rs_poly3(c, y)) < fabs(p))) break;
            x[k] = y;
        }
    return n;
}

// Hartley normalisation of 7 points: T = [s 0 tx; 0 s ty; 0 0 1] stored as {s, tx, ty}; false if all coincide
RS_HD bool rs_normalise7(const double q[14], double T[3]) {
    double cx = 0, cy = 0;
    for (int i = 0; i < 7; ++i) { cx += q[2 * i]; cy += q[2 * i + 1]; }
    cx /= 7; cy /= 7;
    double md = 0;
    for (int i = 0; i < 7; ++i) md += sqrt((q[2 * i] - cx) * (q[2 * i] - cx) + (q[2 * i + 1] - cy) * (q[2 * i + 1] - cy));
    md /= 7;
    if (!(md > 0)) return false;
    const double s = sqrt(2.0) / md;
    T[0] = s; T[1] = -s * cx; T[2] = -s * cy;
    return true;
}

// 7-point fundamental matrices from q1 (view 1) / q2 (view 2), x, y interleaved: x2^T F x1 = 0, row-major,
// unit Frobenius norm.  Returns the number of models (0 for a degenerate sample).
RS_HD int rs_seven_point(const double q1[14], const double q2[14], double F[3][9]) {
    double T1[3], T2[3];
    if (!rs_normalise7(q1, T1) || !rs_normalise7(q2, T2)) return 0;
    double A[7][9];
    double amax = 0;
    for (int i = 0; i < 7; ++i) {
        const double x1 = T1[0] * q1[2 * i] + T1[1], y1 = T1[0] * q1[2 * i + 1] + T1[2];
        const double x2 = T2[0] * q2[2 * i] + T2[1], y2 = T2[0] * q2[2 * i + 1] + T2[2];
        const double a[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
        for (int j = 0; j < 9; ++j) { A[i][j] = a[j]; amax = fmax(amax, fabs(a[j])); }
    }
    // Gauss-Jordan with partial pivoting on columns 0..6: A -> [I | B], null space spanned by (-B e_k, e_k)
    for (int j = 0; j < 7; ++j) {
        int piv = j;
        for (int i = j + 1; i < 7; ++i) if (fabs(A[i][j]) > fabs(A[piv][j])) piv = i;
        if (!(fabs(A[piv][j]) > RS_PIVOT_EPS * amax)) return 0;
        if (piv != j)
            for (int c = 0; c < 9; ++c) { const double tmp = A[j][c]; A[j][c] = A[piv][c]; A[piv][c] = tmp; }
        const double inv = 1.0 / A[j][j];
        for (int c = j; c < 9; ++c) A[j][c] *= inv;
        for (int i = 0; i < 7; ++i) {
            if (i == j) continue;
            const double f = A[i][j];
            if (f == 0.0) continue;
            for (int c = j; c < 9; ++c) A[i][c] -= f * A[j][c];
        }
    }
    double F1[9], F2[9], D[9];
    for (int i = 0; i < 7; ++i) { F1[i] = -A[i][7]; F2[i] = -A[i][8]; }
    F1[7] = 1; F1[8] = 0; F2[7] = 0; F2[8] = 1;
    for (int i = 0; i < 9; ++i) D[i] = F1[i] - F2[i];
    // det(F2 + l D) = c3 l^3 + c2 l^2 + c1 l + c0, by multilinearity in the columns
    double c[4];
    c[0] = rs_det3(F2);
    c[1] = rs_det3_mixed(F2, D, 1) + rs_det3_mixed(F2, D, 2) + rs_det3_mixed(F2, D, 4);
    c[2] = rs_det3_mixed(F2, D, 6) + rs_det3_mixed(F2, D, 5) + rs_det3_mixed(F2, D, 3);
    c[3] = rs_det3(D);
    double lam[3];
    const int nr = rs_real_roots(c, lam);
    int n = 0;
    for (int k = 0; k < nr; ++k) {
        double Fn[9];
        for (int i = 0; i < 9; ++i) Fn[i] = F2[i] + lam[k] * D[i];
        // de-normalise: F = T2^T Fn T1
        double G[9];
        for (int r = 0; r < 3; ++r) {
            const double f0 = Fn[3 * r], f1 = Fn[3 * r + 1], f2 = Fn[3 * r + 2];
            G[3 * r] = f0 * T1[0];
            G[3 * r + 1] = f1 * T1[0];
            G[3 * r + 2] = f0 * T1[1] + f1 * T1[2] + f2;
        }
        double* out = F[n];
        for (int col = 0; col < 3; ++col) {
            out[col] = T2[0] * G[col];
            out[3 + col] = T2[0] * G[3 + col];
            out[6 + col] = T2[1] * G[col] + T2[2] * G[3 + col] + G[6 + col];
        }
        double nf = 0;
        for (int i = 0; i < 9; ++i) nf += out[i] * out[i];
        if (!(nf > 0)) continue;
        nf = 1.0 / sqrt(nf);
        for (int i = 0; i < 9; ++i) out[i] *= nf;
        ++n;
    }
    return n;
}

// ------------------------------------------------------------------------------------------------ scoring
// cv2's fundamental-matrix error (fundam.cpp computeError): max(d^2 / |F^T x2|_xy^2, d^2 / |F x1|_xy^2) with
// d = x2^T F x1, i.e. the larger squared point-to-epipolar-line distance of the two views
RS_HD double rs_fm_error(const double F[9], double x1, double y1, double x2, double y2) {
    const double a = F[0] * x1 + F[1] * y1 + F[2], b = F[3] * x1 + F[4] * y1 + F[5], c = F[6] * x1 + F[7] * y1 + F[8];
    const double d2 = x2 * a + y2 * b + c;
    const double a1 = F[0] * x2 + F[3] * y2 + F[6], b1 = F[1] * x2 + F[4] * y2 + F[7], c1 = F[2] * x2 + F[5] * y2 + F[8];
    const double d1 = x1 * a1 + y1 * b1 + c1;
    return fmax(d1 * d1 / (a1 * a1 + b1 * b1), d2 * d2 / (a * a + b * b));
}

// rs_fm_error(...) <= thr2 without the divisions: both views' lines share d = x2^T F x1, so the test is
// d^2 <= thr2 * min(|F x1|_xy^2, |F^T x2|_xy^2)
RS_HD bool rs_is_inlier(const double F[9], double x1, double y1, double x2, double y2, double thr2) {
    const double a = F[0] * x1 + F[1] * y1 + F[2], b = F[3] * x1 + F[4] * y1 + F[5], c = F[6] * x1 + F[7] * y1 + F[8];
    const double d = x2 * a + y2 * b + c;
    const double a1 = F[0] * x2 + F[3] * y2 + F[6], b1 = F[1] * x2 + F[4] * y2 + F[7];
    return d * d <= thr2 * fmin(a * a + b * b, a1 * a1 + b1 * b1);
}

// ------------------------------------------------------------------------------------------------ one hypothesis
// Sample (with redraws) and solve hypothesis h of a pair of m correspondences pts[i] = {x1, y1, x2, y2}.  Returns
// the number of models written to F (0 when every attempt was collinear or degenerate).
template <typename P4>
RS_HD int rs_hypothesis(const P4* pts, int m, uint64_t seed, int p, int h, double F[3][9]) {
    for (int attempt = 0; attempt < RS_MAX_ATTEMPTS; ++attempt) {
        int idx[7];
        rs_draw7(seed, p, h, attempt, m, idx);
        double q1[14], q2[14];
        for (int k = 0; k < 7; ++k) {
            const P4 v = pts[idx[k]];
            q1[2 * k] = v.x; q1[2 * k + 1] = v.y; q2[2 * k] = v.z; q2[2 * k + 1] = v.w;
        }
        if (rs_has_collinear(q1) || rs_has_collinear(q2)) continue;
        return rs_seven_point(q1, q2, F);
    }
    return 0;
}

// packed selection key: more inliers first, then the lower (hypothesis, root) index; 0 means "no model"
RS_HD unsigned long long rs_key(int count, int h, int r) {
    return ((unsigned long long)(uint32_t)count << 32) | (uint32_t)~(uint32_t)(3 * h + r);
}

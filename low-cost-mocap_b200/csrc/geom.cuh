// Per-point geometry of S3 / reprojection error, usable from device and (for the
// host-side unit checks in tests/hostcheck) from host code.
//
// Reference semantics restated here (computer_code/api/helpers.py):
//   triangulate_point  :293-327  rows y*P[2]-P[1], P[0]-x*P[2]; B = A^T A; SVD(B); X = Vh[3,:3]/Vh[3,3]
//   calculate_reprojection_error :214-241  X -> float32, cv.projectPoints (double math,
//        float32 result), mean of squared pixel residuals in float64
#pragma once
#include <math.h>

#if defined(__CUDA_ARCH__)
#define GEOM_HD __host__ __device__ __forceinline__
// exact (non-fused) double ops where the reference's rounding sequence must be kept
#define DMUL(a, b) __dmul_rn((a), (b))
#define DADD(a, b) __dadd_rn((a), (b))
#define DSUB(a, b) __dsub_rn((a), (b))
#define DFMA(a, b, c) fma((a), (b), (c))
#elif defined(__CUDACC__)
#define GEOM_HD __host__ __device__ __forceinline__
#define DMUL(a, b) ((a) * (b))
#define DADD(a, b) ((a) + (b))
#define DSUB(a, b) ((a) - (b))
#define DFMA(a, b, c) fma((a), (b), (c))
#else
#define GEOM_HD static inline
#define DMUL(a, b) ((a) * (b))
#define DADD(a, b) ((a) + (b))
#define DSUB(a, b) ((a) - (b))
#define DFMA(a, b, c) fma((a), (b), (c))
#endif

// Upper triangle of the 4x4 normal matrix, order 00 01 02 03 11 12 13 22 23 33.
struct Sym4 { double v[10]; };

GEOM_HD void sym4_zero(Sym4& B) {
#pragma unroll
    for (int i = 0; i < 10; ++i) B.v[i] = 0.0;
}

GEOM_HD void sym4_add_row(Sym4& B, double r0, double r1, double r2, double r3) {
    B.v[0] = DFMA(r0, r0, B.v[0]); B.v[1] = DFMA(r0, r1, B.v[1]); B.v[2] = DFMA(r0, r2, B.v[2]); B.v[3] = DFMA(r0, r3, B.v[3]);
    B.v[4] = DFMA(r1, r1, B.v[4]); B.v[5] = DFMA(r1, r2, B.v[5]); B.v[6] = DFMA(r1, r3, B.v[6]);
    B.v[7] = DFMA(r2, r2, B.v[7]); B.v[8] = DFMA(r2, r3, B.v[8]);
    B.v[9] = DFMA(r3, r3, B.v[9]);
}

// One view of the DLT system (helpers.py:314-316).  P: 3x4 row-major.  The A entries are
// formed with separately rounded multiply and subtract, exactly as numpy forms them.
GEOM_HD void dlt_add_view(Sym4& B, const double* __restrict__ P, double x, double y) {
    const double a0 = DSUB(DMUL(y, P[8]), P[4]), a1 = DSUB(DMUL(y, P[9]), P[5]);
    const double a2 = DSUB(DMUL(y, P[10]), P[6]), a3 = DSUB(DMUL(y, P[11]), P[7]);
    sym4_add_row(B, a0, a1, a2, a3);
    const double b0 = DSUB(P[0], DMUL(x, P[8])), b1 = DSUB(P[1], DMUL(x, P[9]));
    const double b2 = DSUB(P[2], DMUL(x, P[10])), b3 = DSUB(P[3], DMUL(x, P[11]));
    sym4_add_row(B, b0, b1, b2, b3);
}

// K_k [R|t] (Kk 3x3, Rt 3x4, both row-major) summed like the BLAS micro-kernel the reference's numpy call runs:
// fused multiply-adds over the inner index (see ba.cu make_P)
GEOM_HD void make_P_like_blas(const double* Kk, const double* Rt, double P[12]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 4; ++j) {
            double acc = DMUL(Kk[3 * i + 0], Rt[j]);
            acc = DFMA(Kk[3 * i + 1], Rt[4 + j], acc);
            acc = DFMA(Kk[3 * i + 2], Rt[8 + j], acc);
            P[4 * i + j] = acc;
        }
}

#define JROT(p, q)                                                                       \
    {                                                                                     \
        const double apq = a[p][q];                                                       \
        if (apq != 0.0) {                                                                 \
            const double g100 = 100.0 * fabs(apq);                                        \
            if (sweep > 3 && fabs(a[p][p]) + g100 == fabs(a[p][p]) &&                     \
                fabs(a[q][q]) + g100 == fabs(a[q][q])) {                                  \
                a[p][q] = 0.0;                                                            \
            } else {                                                                      \
                const double hdiff = a[q][q] - a[p][p];                                   \
                double tt;                                                                \
                if (fabs(hdiff) + g100 == fabs(hdiff)) {                                  \
                    tt = apq / hdiff;                                                     \
                } else {                                                                  \
                    const double theta = 0.5 * hdiff / apq;                               \
                    tt = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));                 \
                    if (theta < 0.0) tt = -tt;                                            \
                }                                                                         \
                const double cc = 1.0 / sqrt(1.0 + tt * tt);                              \
                const double ss = tt * cc;                                                \
                const double tau = ss / (1.0 + cc);                                       \
                const double hh = tt * apq;                                               \
                a[p][p] -= hh;                                                            \
                a[q][q] += hh;                                                            \
                a[p][q] = 0.0;                                                            \
                _Pragma("unroll") for (int r = 0; r < 4; ++r) {                           \
                    if (r != p && r != q) {                                               \
                        const double gg = (r < p) ? a[r][p] : a[p][r];                    \
                        const double h2 = (r < q) ? a[r][q] : a[q][r];                    \
                        const double ng = gg - ss * (h2 + gg * tau);                      \
                        const double nh = h2 + ss * (gg - h2 * tau);                      \
                        if (r < p) a[r][p] = ng; else a[p][r] = ng;                       \
                        if (r < q) a[r][q] = nh; else a[q][r] = nh;                       \
                    }                                                                     \
                }                                                                         \
                _Pragma("unroll") for (int r = 0; r < 4; ++r) {                           \
                    const double gg = v[r][p], h2 = v[r][q];                              \
                    v[r][p] = gg - ss * (h2 + gg * tau);                                  \
                    v[r][q] = h2 + ss * (gg - h2 * tau);                                  \
                }                                                                         \
            }                                                                             \
        }                                                                                 \
    }

// Null-space direction of the symmetric 4x4 normal matrix: the eigenvector of the
// eigenvalue of smallest magnitude (== last right singular vector, Vh[3] of
// scipy.linalg.svd(B), helpers.py:320-321, up to sign -- the sign cancels in X).
// Cyclic Jacobi in registers: small eigenvalues of a positive matrix come out with
// high relative accuracy, which the squared conditioning of A^T A needs.
GEOM_HD void sym4_null_vector(const Sym4& B, double out[4]) {
    double a[4][4], v[4][4];
    a[0][0] = B.v[0]; a[0][1] = B.v[1]; a[0][2] = B.v[2]; a[0][3] = B.v[3];
    a[1][1] = B.v[4]; a[1][2] = B.v[5]; a[1][3] = B.v[6];
    a[2][2] = B.v[7]; a[2][3] = B.v[8];
    a[3][3] = B.v[9];
    a[1][0] = a[2][0] = a[2][1] = a[3][0] = a[3][1] = a[3][2] = 0.0;   // only the upper triangle is used
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) v[r][c] = (r == c) ? 1.0 : 0.0;
    // Tournament order: rounds {(0,1),(2,3)}, {(0,2),(1,3)}, {(0,3),(1,2)}.  Only the first round is
    // written out; the other two are the same code after relabelling the indices by the cycle
    // 1 -> 2 -> 3 -> 1 (register moves), which returns to the identity after three rounds.  Keeps the
    // instruction footprint at two rotation bodies instead of six (the kernels are I-cache bound).
#pragma unroll 1
    for (int sweep = 0; sweep < 30; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[0][3]) + fabs(a[1][2]) + fabs(a[1][3]) + fabs(a[2][3]);
        if (off == 0.0) break;
#pragma unroll 1
        for (int round = 0; round < 3; ++round) {
            JROT(0, 1) JROT(2, 3)
            // relabel: new[i][j] = old[rho(i)][rho(j)], rho = (0, 2, 3, 1)
            const double n01 = a[0][2], n02 = a[0][3], n03 = a[0][1];
            const double n11 = a[2][2], n12 = a[2][3], n13 = a[1][2];
            const double n22 = a[3][3], n23 = a[1][3], n33 = a[1][1];
            a[0][1] = n01; a[0][2] = n02; a[0][3] = n03;
            a[1][1] = n11; a[1][2] = n12; a[1][3] = n13;
            a[2][2] = n22; a[2][3] = n23; a[3][3] = n33;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const double c1 = v[r][2], c2 = v[r][3], c3 = v[r][1];
                v[r][1] = c1; v[r][2] = c2; v[r][3] = c3;
            }
        }
    }
    int best = 0;
    double bv = fabs(a[0][0]);
    if (fabs(a[1][1]) < bv) { bv = fabs(a[1][1]); best = 1; }
    if (fabs(a[2][2]) < bv) { bv = fabs(a[2][2]); best = 2; }
    if (fabs(a[3][3]) < bv) { bv = fabs(a[3][3]); best = 3; }
#pragma unroll
    for (int r = 0; r < 4; ++r)
        out[r] = best == 0 ? v[r][0] : best == 1 ? v[r][1] : best == 2 ? v[r][2] : v[r][3];
}

// Fast path for the same null vector: two plain inverse-iteration steps on the LDL^T factors of B (they pull the
// start vector towards the eigenvector of the smallest eigenvalue at the rate lambda4/lambda3 per step), then
// Rayleigh-quotient iteration -- every step re-factors B - rho I with rho = y^T B y / y^T y and converges cubically,
// so that candidate groups whose views do NOT agree on a point (lambda4/lambda3 near 1: most groups of a busy
// frame-set) settle in the same handful of steps as the good ones and a warp's lanes stay together.  The iteration
// stops when two successive iterates agree to 2e-14.  Because a Rayleigh quotient can be drawn to lambda3 when
// the two smallest eigenvalues are close, the result is accepted only if B - (rho - delta) I is positive definite
// (no eigenvalue below rho: pivot signs of one more LDL^T, delta = 1e-9 trace(B)); otherwise -- and whenever a
// pivot breaks down or nothing settles -- this returns false and the caller runs the Jacobi solver above.
// The two agree to ~1e-13 relative.
struct Ldl4 { double l10, l20, l30, l21, l31, l32, i0, i1, i2, i3; };

// 1 / d for the pivots of the ITERATIVE solver below: the hardware's approximate reciprocal refined by two Newton steps
// (full double precision to an ulp or two, a handful of instructions) instead of the correctly rounded division
// (~40 instructions) -- the iteration converges to the same vector either way and its result is checked.  Everything
// whose rounding the reference fixes (A entries, projections, the final dehomogenisation) keeps exact division.
GEOM_HD double geom_rcp(double d) {
#if defined(__CUDA_ARCH__)
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    return r;
#else
    return 1.0 / d;
#endif
}

// LDL^T of B - shift I without pivoting; false on a zero / non-finite pivot.  n_neg = number of negative pivots.
GEOM_HD bool sym4_ldl(const Sym4& B, double shift, Ldl4& f, int& n_neg) {
    const double b00 = B.v[0] - shift, b01 = B.v[1], b02 = B.v[2], b03 = B.v[3], b11 = B.v[4] - shift, b12 = B.v[5], b13 = B.v[6];
    const double b22 = B.v[7] - shift, b23 = B.v[8], b33 = B.v[9] - shift;
    if (!(b00 != 0.0)) return false;
    f.i0 = geom_rcp(b00);
    f.l10 = b01 * f.i0; f.l20 = b02 * f.i0; f.l30 = b03 * f.i0;
    const double d1 = b11 - f.l10 * b01;
    if (!(d1 != 0.0)) return false;
    f.i1 = geom_rcp(d1);
    f.l21 = (b12 - f.l20 * b01) * f.i1; f.l31 = (b13 - f.l30 * b01) * f.i1;
    const double d2 = b22 - f.l20 * b02 - f.l21 * (f.l21 * d1);
    if (!(d2 != 0.0)) return false;
    f.i2 = geom_rcp(d2);
    f.l32 = (b23 - f.l30 * b02 - f.l31 * (f.l21 * d1)) * f.i2;
    double d3 = b33 - f.l30 * b03 - f.l31 * (f.l31 * d1) - f.l32 * (f.l32 * d2);
    if (!(d3 == d3)) return false;
    if (fabs(d3) < 1e-290) d3 = 1e-290;                 // exactly singular: any huge amplification along the null vector will do
    f.i3 = geom_rcp(d3);
    n_neg = (b00 < 0.0) + (d1 < 0.0) + (d2 < 0.0) + (d3 < 0.0);
    return true;
}

// y <- normalised (B - shift I)^-1 y through the factors; ym = max |y_i| afterwards (in [0.5, 1)); false if it overflowed
GEOM_HD bool sym4_invit_step(const Ldl4& f, double y[4], double& ym) {
    const double z0 = y[0], z1 = y[1] - f.l10 * z0, z2 = y[2] - f.l20 * z0 - f.l21 * z1, z3 = y[3] - f.l30 * z0 - f.l31 * z1 - f.l32 * z2;
    const double w3 = z3 * f.i3;
    const double w2 = z2 * f.i2 - f.l32 * w3;
    const double w1 = z1 * f.i1 - f.l21 * w2 - f.l31 * w3;
    const double w0 = z0 * f.i0 - f.l10 * w1 - f.l20 * w2 - f.l30 * w3;
    // renormalise by an exact power of two (keeps the iterates in range without rounding)
    const double m = fmax(fmax(fabs(w0), fabs(w1)), fmax(fabs(w2), fabs(w3)));
    if (!(m > 0.0) || !(m < 1e300)) return false;
#if defined(__CUDA_ARCH__)
    // 2^-e with e = frexp's exponent, straight from the exponent field: one multiply per component
    const int ebits = (__double2hiint(m) >> 20) & 0x7ff;
    const double sc2 = __hiloint2double((2045 - ebits) << 20, 0);
    y[0] = w0 * sc2; y[1] = w1 * sc2; y[2] = w2 * sc2; y[3] = w3 * sc2;
    ym = m * sc2;
#else
    int e;
    (void)frexp(m, &e);
    y[0] = ldexp(w0, -e); y[1] = ldexp(w1, -e); y[2] = ldexp(w2, -e); y[3] = ldexp(w3, -e);
    ym = ldexp(m, -e);
#endif
    return true;
}

GEOM_HD bool sym4_null_vector_invit(const Sym4& B, double out[4]) {
    Ldl4 f;
    int n_neg = 0;
    if (!(B.v[0] > 0.0)) return false;
    if (!sym4_ldl(B, 0.0, f, n_neg) || n_neg != 0) return false;          // B = A^T A must be (numerically) positive definite
    double y[4] = {0.0, 0.0, 0.0, 1.0}, ym = 1.0;
    if (!sym4_invit_step(f, y, ym)) return false;
    if (!sym4_invit_step(f, y, ym)) return false;
    double p0 = y[0], p1 = y[1], p2 = y[2], p3 = y[3], pm = ym, rho = 0.0;
    bool settled = false;
#pragma unroll 1
    for (int it = 0; it < 12; ++it) {
        // Rayleigh quotient of the current iterate
        const double q0 = B.v[0] * y[0] + B.v[1] * y[1] + B.v[2] * y[2] + B.v[3] * y[3];
        const double q1 = B.v[1] * y[0] + B.v[4] * y[1] + B.v[5] * y[2] + B.v[6] * y[3];
        const double q2 = B.v[2] * y[0] + B.v[5] * y[1] + B.v[7] * y[2] + B.v[8] * y[3];
        const double q3 = B.v[3] * y[0] + B.v[6] * y[1] + B.v[8] * y[2] + B.v[9] * y[3];
        rho = (y[0] * q0 + y[1] * q1 + y[2] * q2 + y[3] * q3) / (y[0] * y[0] + y[1] * y[1] + y[2] * y[2] + y[3] * y[3]);
        if (!sym4_ldl(B, rho, f, n_neg)) return false;
        if (!sym4_invit_step(f, y, ym)) return false;
        // direction change since the previous iterate, sign-insensitive and division-free:
        // y ~ sg (ym / pm) p when settled  <=>  |y pm - sg ym p| small against ym pm   (ym, pm in [0.5, 1))
        const double dot = y[0] * p0 + y[1] * p1 + y[2] * p2 + y[3] * p3;
        const double sy = dot < 0.0 ? -ym : ym;
        const double dev = fmax(fmax(fabs(y[0] * pm - sy * p0), fabs(y[1] * pm - sy * p1)),
                                fmax(fabs(y[2] * pm - sy * p2), fabs(y[3] * pm - sy * p3)));
        p0 = y[0]; p1 = y[1]; p2 = y[2]; p3 = y[3]; pm = ym;
        if (dev <= 2e-14 * (ym * pm)) { settled = true; break; }
    }
    if (!settled) return false;
    // the smallest eigenvalue?  (rho is the shift the last step was taken with: within O(dev) of the eigenvalue)
    const double delta = 1e-9 * (B.v[0] + B.v[4] + B.v[7] + B.v[9]);
    if (!sym4_ldl(B, rho - delta, f, n_neg) || n_neg != 0) return false;
    out[0] = y[0]; out[1] = y[1]; out[2] = y[2]; out[3] = y[3];
    return true;
}

GEOM_HD void dlt_solve(const Sym4& B, double X[3]) {
    double n[4];
    if (!sym4_null_vector_invit(B, n)) sym4_null_vector(B, n);
    X[0] = n[0] / n[3]; X[1] = n[1] / n[3]; X[2] = n[2] / n[3];     // helpers.py:321
}

// cv.projectPoints with zero distortion on a float32 point (helpers.py:231-238): the
// float32-rounded point is widened, x = R X + t summed left to right, z -> 1/z (1 if
// z == 0), u = x*fx + cx, result stored as float32.  Verified bit-exact against cv2 4.13.
GEOM_HD void project_like_cv(const double* __restrict__ R, const double* __restrict__ t,
                             double fx, double fy, double cx, double cy,
                             const double X[3], float& u, float& v) {
    const double Xs = (double)(float)X[0], Ys = (double)(float)X[1], Zs = (double)(float)X[2];
    double x = DADD(DADD(DADD(DMUL(R[0], Xs), DMUL(R[1], Ys)), DMUL(R[2], Zs)), t[0]);
    double y = DADD(DADD(DADD(DMUL(R[3], Xs), DMUL(R[4], Ys)), DMUL(R[5], Zs)), t[1]);
    double z = DADD(DADD(DADD(DMUL(R[6], Xs), DMUL(R[7], Ys)), DMUL(R[8], Zs)), t[2]);
    z = (z != 0.0) ? 1.0 / z : 1.0;
    x = DMUL(x, z);
    y = DMUL(y, z);
    u = (float)DADD(DMUL(x, fx), cx);
    v = (float)DADD(DMUL(y, fy), cy);
}

// numpy's reduction of n squared residuals (n = 2 * views <= 32) followed by / n.
//  pairwise == false: left fold (object-dtype arrays: any group that contains a None view)
//  pairwise == true : np.add.reduce on float64, blocked 8-accumulator form for 8 <= n < 128
GEOM_HD double mean_like_numpy(const double* sq, int n, bool pairwise) {
    double res;
    if (!pairwise || n < 8) {
        res = 0.0;
        if (pairwise) { res = sq[0]; for (int i = 1; i < n; ++i) res = DADD(res, sq[i]); }
        else { for (int i = 0; i < n; ++i) res = DADD(res, sq[i]); }
    } else {
        double r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = sq[j];
        int i = 8;
#pragma unroll 1
        for (; i < n - (n % 8); i += 8) {
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = DADD(r[j], sq[i + j]);
        }
        res = DADD(DADD(DADD(r[0], r[1]), DADD(r[2], r[3])), DADD(DADD(r[4], r[5]), DADD(r[6], r[7])));
        for (; i < n; ++i) res = DADD(res, sq[i]);
    }
    return res / (double)n;
}

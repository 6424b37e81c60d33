// Per-view screening of explicit correspondences against camera poses: which views of each track enter the bundle
// adjustment.  Written against geom.cuh only (no CUDA headers), so that tests/hostcheck/screen_host.cpp runs this very
// rule with g++ and the kernel (screen.cu) runs it with its lanes split over view pairs and views.
//
// The rule, for one track whose caller's mask holds the views S:
//   1. |S| < 2: the row is unchanged.
//   2. Every pair (a, b) of S, a < b, in lexicographic order: X_ab is the DLT point of the pair, its support the views
//      c of S with e_c(X_ab)^2 <= thr^2.  The pair with the largest support wins, ties to the earlier pair.
//   3. A support of >= 2 views is re-triangulated, X, and S' = {c in S : e_c(X)^2 <= thr^2}.  S' is kept if it has
//      >= 2 views and every view of S' passes against the DLT point of S' itself.  Otherwise -- and for a winning
//      support of < 2 views -- the row is emptied: the track leaves the adjustment.
// Arithmetic is the bundle adjustment's residual (ba_residual): a DLT over a view set T builds the view of rank k in T
// with K_k [R_c | t_c] (the reference's "K of the k-th present view", helpers.py:305-307), summed in ascending camera
// order; e_c is the pixel distance to project_like_cv of the point, with the intrinsics of the rank c holds in T + {c}.
// So the final check of step 3 is exactly the residual arithmetic of the objective the row then enters.
#pragma once
#include "geom.cuh"

#define SCREEN_MAX_CAM 16

// the cameras as the screen reads them: built from the CURRENT poses (not the context's camera tables)
struct ScreenCams {
    double P[SCREEN_MAX_CAM][SCREEN_MAX_CAM][12];      // P[k][c] = K_k [R_c | t_c]
    double R[SCREEN_MAX_CAM][9], t[SCREEN_MAX_CAM][3];
    double fx[SCREEN_MAX_CAM], fy[SCREEN_MAX_CAM], cx[SCREEN_MAX_CAM], cy[SCREEN_MAX_CAM];   // of K_k, by rank k
};

GEOM_HD int screen_popc(unsigned v) {
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}

// entry (k, c) of the table: K_k [R_c | t_c], R row-major 3x3, t 3
GEOM_HD void screen_set_P(ScreenCams& S, int k, int c, const double* Kk, const double* Rc, const double* tc) {
    const double Rt[12] = {Rc[0], Rc[1], Rc[2], tc[0], Rc[3], Rc[4], Rc[5], tc[1], Rc[6], Rc[7], Rc[8], tc[2]};
    make_P_like_blas(Kk, Rt, S.P[k][c]);
}

// camera c's pose and the four intrinsics cv.projectPoints reads of K_c
GEOM_HD void screen_set_cam(ScreenCams& S, int c, const double* Rc, const double* tc, double fx, double fy, double cx, double cy) {
    for (int i = 0; i < 9; ++i) S.R[c][i] = Rc[i];
    for (int i = 0; i < 3; ++i) S.t[c][i] = tc[i];
    S.fx[c] = fx; S.fy[c] = fy; S.cx[c] = cx; S.cy[c] = cy;
}

// DLT point of the views T (bit c = camera c) of one row o = obs [C][2]
GEOM_HD void screen_point(const ScreenCams& S, const double* o, unsigned T, int C, double X[3]) {
    Sym4 B;
    sym4_zero(B);
    int k = 0;
    for (int c = 0; c < C; ++c)
        if ((T >> c) & 1u) { dlt_add_view(B, S.P[k][c], o[2 * c], o[2 * c + 1]); ++k; }
    dlt_solve(B, X);
}

// squared pixel distance of view c to the point X triangulated from T
GEOM_HD double screen_err2(const ScreenCams& S, const double* o, unsigned T, int c, const double X[3]) {
    const int k = screen_popc(T & ((1u << c) - 1u));
    float u, v;
    project_like_cv(S.R[c], S.t[c], S.fx[k], S.fy[k], S.cx[k], S.cy[k], X, u, v);
    const double dx = DSUB(o[2 * c], (double)u), dy = DSUB(o[2 * c + 1], (double)v);
    return DADD(DMUL(dx, dx), DMUL(dy, dy));
}

// the p-th pair of the views S in lexicographic order, as a two-bit mask
GEOM_HD unsigned screen_pair(unsigned S, int p) {
    for (unsigned rest = S; rest; rest &= rest - 1) {
        const unsigned a = rest & (0u - rest);
        unsigned above = rest & ~a;                              // the views after a
        const int cnt = screen_popc(above);
        if (p < cnt) {
            for (int i = 0; i < p; ++i) above &= above - 1;
            return a | (above & (0u - above));
        }
        p -= cnt;
    }
    return 0u;
}

// ordering key of a pair's support: more views first, then the earlier pair (p < 120 at 16 cameras)
GEOM_HD unsigned screen_key(int support, int p) { return ((unsigned)support << 16) | (0xffffu - (unsigned)p); }

// views of Q that pass against the DLT point of T, one view at a time
GEOM_HD unsigned screen_support(const ScreenCams& S, const double* o, int C, unsigned T, unsigned Q, double thr2) {
    double X[3];
    screen_point(S, o, T, C, X);
    unsigned out = 0u;
    for (int c = 0; c < C; ++c)
        if (((Q >> c) & 1u) && screen_err2(S, o, T, c, X) <= thr2) out |= 1u << c;
    return out;
}

// step 3 from the winning pair's support W.  support_of(T, Q): the views of Q that pass against the DLT point of T
// (screen_support on the host, split over a warp's lanes by view on the device)
template <class SupportOf>
GEOM_HD unsigned screen_refit(unsigned S, unsigned W, SupportOf support_of) {
    if (screen_popc(W) < 2) return 0u;
    const unsigned Sp = support_of(W, S);
    if (screen_popc(Sp) < 2) return 0u;
    return support_of(Sp, Sp) == Sp ? Sp : 0u;
}

// the whole rule for one row, sequentially: the views kept (bit c = camera c)
GEOM_HD unsigned screen_row(const ScreenCams& S, const double* o, int C, unsigned Sm, double thr2) {
    const int n = screen_popc(Sm);
    if (n < 2) return Sm;
    unsigned best = 0u, W = 0u;
    for (int p = 0; p < n * (n - 1) / 2; ++p) {
        const unsigned sup = screen_support(S, o, C, screen_pair(Sm, p), Sm, thr2);
        const unsigned key = screen_key(screen_popc(sup), p);
        if (key > best) { best = key; W = sup; }
    }
    return screen_refit(Sm, W, [&](unsigned T, unsigned Q) { return screen_support(S, o, C, T, Q, thr2); });
}

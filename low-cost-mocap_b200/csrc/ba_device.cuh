// S4 wholly on the device: the bundle adjustment of the camera poses as ONE persistent, grid-synchronous kernel.
//
// Replaces bundle_adjustment (reference computer_code/api/helpers.py:244-290) -- the same algorithm as the
// host-stepped path of ba.cu (classic Levenberg-Marquardt over poses + points with the point blocks eliminated by a
// Schur complement, then scipy's trust-region iteration on the reference objective: float32-cast per-point mean squared
// reprojection error after DLT re-triangulation, Cauchy loss, 2-point finite differences), but without a single host
// round trip: residuals, Jacobians, the reduction to normal equations, the <= 90 x 90 dense solves and the
// accept / reject logic all run inside k_ba_solve.
//
// Organisation
//   * points are cut into tiles; tile T belongs to CTA T mod ncta for the whole solve, so a point's 3D
//     estimate never leaves its CTA;
//   * a CTA turns a tile into rows of a small dense system in SHARED memory (prefit: the three rows
//     Z = W L^-T of every point's eliminated 3x3 block plus its per-camera 2x6 Jacobians; polish: the robust-scaled
//     finite-difference Jacobian rows) and every thread then owns a fixed set of (i, j) entries of the normal
//     matrix, which it updates from the tile: no atomics anywhere, so the sums have a fixed order and the result is
//     reproducible;
//   * per-CTA partial systems go to global memory, a grid barrier, every CTA adds a slice of the entries over all
//     CTAs, a grid barrier, and then EVERY CTA solves the small dense system redundantly in shared memory
//     (Cholesky; the trust-region sub-problem of scipy's solve_lsq_trust_region is iterated on Cholesky factors of
//     A + alpha I instead of scipy's SVD -- the same phi(alpha), phi'(alpha)), so that the step, the trial poses and
//     every accept / reject decision are bit-identical on all CTAs and need no broadcast;
//   * trial points cost one residual pass and one grid barrier.
// "The grid" above is the problem's SUB-grid: one launch can run several independent problems (BABatch), each on
// its own contiguous range of CTAs with its own barrier words and workspace.  The body never uses blockIdx / gridDim
// directly but the CTA's index and count within its problem (BACtrl::cta / ncta), so that a problem gives the same
// bits on a sub-grid of g CTAs as alone on a grid of g CTAs.
// The code is written against threadIdx / blockIdx / blockDim / gridDim and ba_grid_sync() only, so that
// tests/hostcheck runs it unchanged on the host (several CTAs of real threads) against the host-stepped model.
#pragma once
#include "common.cuh"
#include "geom.cuh"

// the prefit stops when an accepted step lowers the squared pixel error by less than this fraction (shared with the
// host-stepped solve in ba.cu): the polish that follows works on a float32-quantised objective whose resolution is
// coarser than that
#define BA_PREFIT_REL_STOP 1e-7
// trust radius the polish starts with after a prefit that took a step (rad / pose units; scipy would start at ||x0|| ~ the focal length and
// spend its evaluations shrinking).  The prefit ends within ~1e-5 of the reference objective's own minimiser, and scipy's
// radius doubles whenever a step at the boundary is good, so a small start costs nothing when more room is needed;
// measured on the three S4 goldens: 1e-2 -> 7 evaluations, 1e-4 -> 4, final costs equal to 1e-4 relative (the float32
// resolution of the objective).  -DBA_POLISH_RADIUS=... overrides it (host-run experiments).
#ifndef BA_POLISH_RADIUS
#define BA_POLISH_RADIUS 1e-4
#endif
#define BA_TILE 32                 // points per tile (one warp = one column of a tile in the finite-difference pass)
#define BA_MAX_N (6 * (MOCAP_MAX_CAM - 1))

struct BAParams {
    const CameraTables* tb;
    const double* obs;             // [m][C][2]
    const uint8_t* mask;           // [m][C]
    const int32_t* m_dev;          // number of points (device), or nullptr: m_max
    int m_max, C;
    double* R; double* t;          // [C][9], [C][3]  in / out
    double ftol, xtol, gtol;
    int max_nfev, jac_mode, prefit, prefit_max_iter;
    // workspace
    double* X; double* Xnew;       // [m_max][3]
    uint8_t* valid;                // [m_max]
    double* part; int pstride;     // [grid][pstride] per-CTA partial systems
    double* fin;                   // [pstride] reduced system
    double* cpart;                 // [2][grid][4] trial-point partials (cost, non-finite, count)
    unsigned* bar;                 // [2] grid barrier: arrivals, generation
    mocap_ba_report* report;       // device, may be nullptr
    int cta0, ncta;                // this problem's CTAs of the launch: [cta0, cta0 + ncta); ncta == 0: the whole grid
};

// the problems of one launch: problem k owns CTAs [p[k].cta0, p[k].cta0 + p[k].ncta), in increasing k
struct BABatch {
    int n;
    BAParams p[MOCAP_BA_MAX_BATCH];
};

#if defined(__CUDA_ARCH__)
#define BA_DEV __device__ __forceinline__
// barrier of the n CTAs that share the words bar (arrivals, generation)
__device__ __forceinline__ void ba_grid_sync(unsigned* bar, unsigned n) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned gen = *reinterpret_cast<volatile unsigned*>(bar + 1);
        if (atomicAdd(bar, 1u) == n - 1) {
            bar[0] = 0;
            __threadfence();
            atomicAdd(bar + 1, 1u);
        } else {
            while (*reinterpret_cast<volatile unsigned*>(bar + 1) == gen) {}
        }
        __threadfence();
    }
    __syncthreads();
}
#elif defined(__CUDACC__)
#define BA_DEV __device__ __forceinline__
__device__ __forceinline__ void ba_grid_sync(unsigned*, unsigned) {}
#else
#define BA_DEV static inline
// host emulation (tests/hostcheck/simt_emu.h): the device's counter-and-generation scheme, waiting with a yield, so
// that sub-grids which iterate different numbers of times do not wait for each other
static inline void ba_grid_sync(unsigned* bar, unsigned n) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned gen = __atomic_load_n(bar + 1, __ATOMIC_SEQ_CST);
        if (__atomic_fetch_add(bar, 1u, __ATOMIC_SEQ_CST) == n - 1) {
            __atomic_store_n(bar, 0u, __ATOMIC_SEQ_CST);
            __atomic_fetch_add(bar + 1, 1u, __ATOMIC_SEQ_CST);
        } else {
            while (__atomic_load_n(bar + 1, __ATOMIC_SEQ_CST) == gen) std::this_thread::yield();
        }
    }
    __syncthreads();
}
#endif

// index of this CTA's problem in the launch
BA_DEV int ba_problem_of(const BABatch& B) {
    int k = 0;
#pragma unroll
    for (int q = 1; q < MOCAP_BA_MAX_BATCH; ++q) k += (q < B.n && (int)blockIdx.x >= B.p[q].cta0) ? 1 : 0;
    return k;
}

// ---- parameterisation (scipy.spatial.transform.Rotation as the reference uses it, helpers.py:247-262, 278-285;
//      same arithmetic as trf_core.h) --------------------------------------------------------------------------
BA_DEV void ba_rotvec_to_matrix(const double rv[3], double R[9]) {
    const double angle = sqrt(rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2]);
    double scale;
    if (angle <= 1e-3) {
        const double a2 = angle * angle;
        scale = 0.5 - a2 / 48.0 + a2 * a2 / 3840.0;
    } else scale = sin(angle / 2.0) / angle;
    double x = scale * rv[0], y = scale * rv[1], z = scale * rv[2], w = cos(angle / 2.0);
    const double nq = sqrt(x * x + y * y + z * z + w * w);
    x /= nq; y /= nq; z /= nq; w /= nq;
    const double x2 = x * x, y2 = y * y, z2 = z * z, w2 = w * w;
    const double xy = x * y, zw = z * w, xz = x * z, yw = y * w, yz = y * z, xw = x * w;
    R[0] = x2 - y2 - z2 + w2; R[3] = 2 * (xy + zw);       R[6] = 2 * (xz - yw);
    R[1] = 2 * (xy - zw);     R[4] = -x2 + y2 - z2 + w2;  R[7] = 2 * (yz + xw);
    R[2] = 2 * (xz + yw);     R[5] = 2 * (yz - xw);       R[8] = -x2 - y2 + z2 + w2;
}

BA_DEV void ba_matrix_to_rotvec(const double R[9], double rv[3]) {
    const double m00 = R[0], m11 = R[4], m22 = R[8], tr = m00 + m11 + m22;
    const double dec[4] = {m00, m11, m22, tr};
    int choice = 0;
    for (int i = 1; i < 4; ++i) if (dec[i] > dec[choice]) choice = i;
    double q[4];   // x y z w
    if (choice != 3) {
        const int i = choice, j = (i + 1) % 3, k = (j + 1) % 3;
        q[i] = 1 - dec[3] + 2 * R[i * 3 + i];
        q[j] = R[j * 3 + i] + R[i * 3 + j];
        q[k] = R[k * 3 + i] + R[i * 3 + k];
        q[3] = R[k * 3 + j] - R[j * 3 + k];
    } else {
        q[0] = R[2 * 3 + 1] - R[1 * 3 + 2];
        q[1] = R[0 * 3 + 2] - R[2 * 3 + 0];
        q[2] = R[1 * 3 + 0] - R[0 * 3 + 1];
        q[3] = 1 + dec[3];
    }
    const double nq = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int i = 0; i < 4; ++i) q[i] /= nq;
    if (q[3] < 0) for (int i = 0; i < 4; ++i) q[i] = -q[i];
    const double sn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    const double angle = 2.0 * atan2(sn, q[3]);
    double scale;
    if (angle <= 1e-3) {
        const double a2 = angle * angle;
        scale = 2.0 + a2 / 12.0 + 7.0 * a2 * a2 / 2880.0;
    } else scale = angle / sin(angle / 2.0);
    rv[0] = scale * q[0]; rv[1] = scale * q[1]; rv[2] = scale * q[2];
}

// [R|t] (3x4 row-major) of camera c from the parameter vector x = [f0, (f_c, rotvec_c, t_c) c = 1..C-1]
BA_DEV void ba_pose_from_x(const double* x, int c, double Rt[12]) {
    if (c == 0) {                                              // helpers.py:250-253
        for (int i = 0; i < 12; ++i) Rt[i] = 0.0;
        Rt[0] = Rt[5] = Rt[10] = 1.0;
        return;
    }
    const double* q = x + 1 + 7 * (c - 1);
    double R[9];
    ba_rotvec_to_matrix(q + 1, R);
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rt[4 * i + j] = R[3 * i + j];
        Rt[4 * i + 3] = q[4 + i];
    }
}

// K_k [R|t] summed like the BLAS micro-kernel the reference's numpy call runs (geom.cuh; the screen of screen.cuh
// builds its projection matrices with the same function)
BA_DEV void ba_make_P(const double* Kk, const double* Rt, double P[12]) { make_P_like_blas(Kk, Rt, P); }

// residual_function of the reference for one point (helpers.py:264-276): DLT with the trial poses, reprojection
// error like cv.projectPoints, mean in numpy's order.  Camera `cam` (if >= 0) takes the pose colRt instead of its
// base pose.  Same arithmetic as ba_point_residual in ba.cu.
BA_DEV double ba_residual(const CameraTables* tb, const double* baseRt, int cam, const double* colRt,
                          const double* o, const uint8_t* mk, int C, double X[3]) {
    Sym4 B;
    sym4_zero(B);
    int k = 0;
    for (int c = 0; c < C; ++c)
        if (mk[c]) {
            const double* Rt = (c == cam) ? colRt : baseRt + 12 * c;
            double P[12];
            ba_make_P(tb->Kmat[k], Rt, P);                   // K of the k-th PRESENT view (helpers.py:305-307)
            dlt_add_view(B, P, o[2 * c], o[2 * c + 1]);
            ++k;
        }
    dlt_solve(B, X);
    double sq[2 * MOCAP_MAX_CAM];
    k = 0;
    for (int c = 0; c < C; ++c)
        if (mk[c]) {
            const double* Rt = (c == cam) ? colRt : baseRt + 12 * c;
            const double R[9] = {Rt[0], Rt[1], Rt[2], Rt[4], Rt[5], Rt[6], Rt[8], Rt[9], Rt[10]};
            const double t[3] = {Rt[3], Rt[7], Rt[11]};
            float u, v;
            project_like_cv(R, t, tb->fx[k], tb->fy[k], tb->cx[k], tb->cy[k], X, u, v);
            const double dx = DSUB(o[2 * c], (double)u), dy = DSUB(o[2 * c + 1], (double)v);
            sq[2 * k] = DMUL(dx, dx); sq[2 * k + 1] = DMUL(dy, dy);
            ++k;
        }
    return mean_like_numpy(sq, 2 * k, false);
}

// one view of the classic bundle adjustment: pixel residual e, its derivative wrt the camera's 6 local
// parameters (Exp(w) R, t + dt) and wrt the point
struct BAViewJac { double e[2]; double Jc[2][6]; double Jp[2][3]; };
BA_DEV void ba_view_jacobian(const double* Rt, double fx, double fy, double cx, double cy,
                             const double X[3], double uo, double vo, BAViewJac& J) {
    const double rx = Rt[0] * X[0] + Rt[1] * X[1] + Rt[2] * X[2];
    const double ry = Rt[4] * X[0] + Rt[5] * X[1] + Rt[6] * X[2];
    const double rz = Rt[8] * X[0] + Rt[9] * X[1] + Rt[10] * X[2];
    const double x = rx + Rt[3], y = ry + Rt[7], z = rz + Rt[11];
    const double iz = 1.0 / z;
    J.e[0] = fx * x * iz + cx - uo;
    J.e[1] = fy * y * iz + cy - vo;
    const double du[3] = {fx * iz, 0.0, -fx * x * iz * iz};
    const double dv[3] = {0.0, fy * iz, -fy * y * iz * iz};
    J.Jc[0][0] = du[1] * (-rz) + du[2] * ry;  J.Jc[0][1] = du[0] * rz + du[2] * (-rx);  J.Jc[0][2] = du[0] * (-ry) + du[1] * rx;
    J.Jc[1][0] = dv[1] * (-rz) + dv[2] * ry;  J.Jc[1][1] = dv[0] * rz + dv[2] * (-rx);  J.Jc[1][2] = dv[0] * (-ry) + dv[1] * rx;
    for (int q = 0; q < 3; ++q) { J.Jc[0][3 + q] = du[q]; J.Jc[1][3 + q] = dv[q]; }
    for (int q = 0; q < 3; ++q) {
        J.Jp[0][q] = du[0] * Rt[q] + du[1] * Rt[4 + q] + du[2] * Rt[8 + q];
        J.Jp[1][q] = dv[0] * Rt[q] + dv[1] * Rt[4 + q] + dv[2] * Rt[8 + q];
    }
}

BA_DEV void ba_exp_so3(const double w[3], double E[9]) {
    const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    double a, b;
    if (th < 1e-8) { a = 1.0 - th * th / 6.0; b = 0.5 - th * th / 24.0; }
    else { a = sin(th) / th; b = (1.0 - cos(th)) / (th * th); }
    const double K[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
    double K2[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += K[3 * i + k] * K[3 * k + j]; K2[3 * i + j] = s; }
    for (int i = 0; i < 9; ++i) E[i] = (i % 4 == 0 ? 1.0 : 0.0) + a * K[i] + b * K2[i];
}

// ---- CTA-wide dense linear algebra on a full n x n row-major matrix in shared memory ------------------------
// In place Cholesky of the lower triangle.  *flag (shared) is 1 on entry; 0 on exit if not positive definite.
BA_DEV bool ba_chol_factor(double* L, int n, int* flag) {
    const int tid = threadIdx.x, nt = blockDim.x;
    (void)flag;
    for (int j = 0; j < n; ++j) {
        __syncthreads();                                           // column j has all its updates
        const double d = L[j * n + j];                             // every thread reads the same pivot: a uniform decision
        if (!(d > 0.0)) return false;
        const double dj = sqrt(d);
        for (int i = j + 1 + tid; i < n; i += nt) L[i * n + j] /= dj;
        __syncthreads();                                           // everybody has read the pivot; column j is scaled
        if (tid == 0) L[j * n + j] = dj;
        const int cnt = n - j - 1;
        for (int idx = tid; idx < cnt * cnt; idx += nt) {
            const int ii = idx / cnt, kk = idx - ii * cnt;
            if (kk <= ii) L[(j + 1 + ii) * n + j + 1 + kk] -= L[(j + 1 + ii) * n + j] * L[(j + 1 + kk) * n + j];
        }
    }
    __syncthreads();
    return true;
}
// The two triangular solves run in ONE warp (the other warps wait at a single barrier): a step is a handful of
// multiply-adds per lane, and 2n CTA-wide barriers per solve cost ten times the arithmetic.
BA_DEV void ba_solve_lower(const double* L, int n, double* v) {          // L y = v, in place
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        for (int j = 0; j < n; ++j) {
            const double vj = v[j] / L[j * n + j];                 // every lane the same value
            __syncwarp();
            if (lane == 0) v[j] = vj;
            for (int i = j + 1 + lane; i < n; i += 32) v[i] -= L[i * n + j] * vj;
            __syncwarp();
        }
    }
    __syncthreads();
}
BA_DEV void ba_solve_upper(const double* L, int n, double* v) {          // L^T x = v, in place
    __syncthreads();
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        for (int j = n - 1; j >= 0; --j) {
            const double vj = v[j] / L[j * n + j];
            __syncwarp();
            if (lane == 0) v[j] = vj;
            for (int i = lane; i < j; i += 32) v[i] -= L[j * n + i] * vj;
            __syncwarp();
        }
    }
    __syncthreads();
}
// sum of squares of v[0..n) by one thread in index order (n <= 106): every CTA gets the same bits
BA_DEV double ba_norm2_serial(const double* v, int n) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += v[i] * v[i];
    return sqrt(s);
}

// wall clock of the solve's phases (device: %globaltimer in ns; host-run checks: 0)
BA_DEV unsigned long long ba_clock() {
#if defined(__CUDA_ARCH__)
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
#else
    return 0ull;
#endif
}
// phases reported in mocap_ba_report.phase_ms
#define BA_PH_SETUP 0
#define BA_PH_PF_SYSTEM 1
#define BA_PH_PF_SOLVE 2
#define BA_PH_PF_TRIAL 3
#define BA_PH_LINEARIZE 4
#define BA_PH_TRIDIAG 5
#define BA_PH_TR_SOLVE 6
#define BA_PH_TRIAL 7
#define BA_TICK(k) do { if (threadIdx.x == 0) { const unsigned long long t__ = ba_clock(); S.ctl->prof[k] += t__ - S.ctl->t_last; S.ctl->t_last = t__; } } while (0)

// scalar state of the solve, in shared memory, written by thread 0 between barriers
struct BACtrl {
    unsigned long long prof[8], t_last;
    double cost, cost_new, cost_initial, Delta, alpha, lambda, g_norm, pred, step_norm, actual, pcost, pcost_new;
    double pf_cost0, pf_cost1;
    double tr_alpha, tr_lower, tr_upper, tr_conv, a_diag, hh_beta, hh_alpha, hh_K;
    int m, ntiles, n_valid, nfev, njev, iteration, termination, finite, flag, go, pf_it, pf_taken, accepted, tr_its, tr_calls;
    int cta, ncta;                     // this CTA's index in its problem's sub-grid, and the sub-grid's size
};

struct BAShared {
    BACtrl* ctl;
    double* x; double* x_new;          // [nf]
    double* Rt; double* Rt_new;        // [C][12]
    double* colRt; int* colcam; double* dx;   // [n][12], [n], [n]
    double* g; double* p; double* q; double* w;   // [n]
    double* td; double* te; double* ghat; double* yhat; double* zhat; double* hv; double* hp; double* hu;   // [n] tridiagonal form of A
    double* pcr;                       // [10][n] cyclic-reduction work arrays (two generations of a, b, 1/b, c, d)
    uint8_t* pi; uint8_t* pj;          // [npair] pair -> (i, j), i <= j
    double* acc;                       // [pstride] this CTA's partial system
    double* scratch;                   // [threads] block sums
    unsigned char* uni;                // union: tile buffers | A, L
    double* A; double* L;              // [n*n] each, inside uni
};

static __host__ __device__ inline size_t ba_align16(size_t b) { return (b + 15) & ~(size_t)15; }
// points per prefit tile piece: the largest power of two <= min(BA_TILE, threads / cameras)
static __host__ __device__ inline int ba_prefit_points(int C, int nt) {
    int lim = nt / C < BA_TILE ? nt / C : BA_TILE, p = 1;
    while (2 * p <= lim) p *= 2;
    return p;
}

// bytes of the tile buffers of the two accumulation passes
static __host__ __device__ inline size_t ba_tile_bytes(int C, int n, int nt) {
    const int Pp = ba_prefit_points(C, nt);
    const size_t prefit = (size_t)(3 * Pp) * n * 8 + (size_t)Pp * C * (12 + 6 + 2) * 8 + (size_t)Pp * (6 + 3 + 3 + 1) * 8 + (size_t)Pp * C;
    const size_t polish = (size_t)BA_TILE * (n + 1) * 8 + (size_t)BA_TILE * 2 * 8;
    return ba_align16(prefit > polish ? prefit : polish);
}
static __host__ __device__ inline size_t ba_smem_bytes(int C, int nt) {
    const int n = 6 * (C - 1), nf = 1 + 7 * (C - 1), npair = n * (n + 1) / 2;
    const int pstride = npair + 2 * n + 8;
    size_t b = 0;
    b += ba_align16(sizeof(BACtrl));
    b += ba_align16((size_t)2 * nf * 8);
    b += ba_align16((size_t)2 * C * 12 * 8);
    b += ba_align16((size_t)n * 12 * 8) + ba_align16((size_t)n * 4) + ba_align16((size_t)n * 8);
    b += 12 * ba_align16((size_t)n * 8);
    b += ba_align16((size_t)10 * n * 8);
    b += 2 * ba_align16((size_t)npair);
    b += ba_align16((size_t)pstride * 8);
    b += ba_align16((size_t)nt * 8);
    const size_t tile = ba_tile_bytes(C, n, nt), mats = ba_align16((size_t)2 * n * n * 8);
    b += tile > mats ? tile : mats;
    return b;
}

BA_DEV BAShared ba_carve(unsigned char* raw, int C, int nt) {
    const int n = 6 * (C - 1), nf = 1 + 7 * (C - 1), npair = n * (n + 1) / 2;
    const int pstride = npair + 2 * n + 8;
    BAShared s;
    s.ctl = reinterpret_cast<BACtrl*>(raw); raw += ba_align16(sizeof(BACtrl));
    s.x = reinterpret_cast<double*>(raw); s.x_new = s.x + nf; raw += ba_align16((size_t)2 * nf * 8);
    s.Rt = reinterpret_cast<double*>(raw); s.Rt_new = s.Rt + C * 12; raw += ba_align16((size_t)2 * C * 12 * 8);
    s.colRt = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 12 * 8);
    s.colcam = reinterpret_cast<int*>(raw); raw += ba_align16((size_t)n * 4);
    s.dx = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.g = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.p = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.q = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.w = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.td = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.te = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.ghat = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.yhat = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.zhat = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.hv = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.hp = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.hu = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)n * 8);
    s.pcr = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)10 * n * 8);
    s.pi = raw; raw += ba_align16((size_t)npair);
    s.pj = raw; raw += ba_align16((size_t)npair);
    s.acc = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)pstride * 8);
    s.scratch = reinterpret_cast<double*>(raw); raw += ba_align16((size_t)nt * 8);
    s.uni = raw;
    s.A = reinterpret_cast<double*>(raw); s.L = s.A + (size_t)n * n;
    return s;
}

// a value of this CTA's problem (or of BACtrl) read afresh at every use.  k_ba_solve stages the CTA's problem in shared
// memory; a pointer that is reloaded (one shared load) where it is used holds no register across the hot loops, which
// keeps the kernel's spills at or below those of the kernel that read a single problem from its parameter
template <typename T> BA_DEV T ba_fresh(const T& v) { return *const_cast<const volatile T*>(&v); }

// this CTA's points: local index i -> global point (tile T = cta + (i / BA_TILE) * ncta)
BA_DEV int ba_local_tiles(const BACtrl* ctl) {
    const int b = ba_fresh(ctl->cta), G = ba_fresh(ctl->ncta), ntiles = ctl->ntiles;
    return ntiles > b ? (ntiles - b + G - 1) / G : 0;
}
BA_DEV int ba_point_of(const BACtrl* ctl, int local_index) {
    const int lt = local_index / BA_TILE;
    return (ba_fresh(ctl->cta) + lt * ba_fresh(ctl->ncta)) * BA_TILE + (local_index - lt * BA_TILE);
}

// CTA-wide sum of per-thread values, fixed order (thread 0 adds the warps' partial sums held in `scratch`)
BA_DEV double ba_block_sum(double v, double* scratch) {
    const int tid = threadIdx.x, nt = blockDim.x;
    __syncthreads();
    scratch[tid] = v;
    __syncthreads();
    for (int s = 1; s < nt; s <<= 1) {                         // pairwise tree: the same bits for a given nt
        const int i = tid * 2 * s;
        if (i + s < nt) scratch[i] += scratch[i + s];
        __syncthreads();
    }
    const double r = scratch[0];
    __syncthreads();
    return r;
}

// ---- passes over this CTA's points ---------------------------------------------------------------------------
// reference objective at the poses Rt: 0.5 * sum log1p(f^2) over the CTA's valid points (+ non-finite flag);
// optionally marks valid points and stores the DLT points (start of the prefit)
BA_DEV void ba_cost_pass(const BAParams& P, const BAParams& Q, const BAShared& S, const double* Rt, bool first, double* scratch, double out[3]) {
    const int tid = threadIdx.x, nt = blockDim.x, C = Q.C;
    const int lt = ba_local_tiles(S.ctl);
    double c = 0.0, bad = 0.0, cnt = 0.0;
    const uint8_t* mask = ba_fresh(P.mask);
    const double* obs = ba_fresh(P.obs);
    uint8_t* valid = ba_fresh(P.valid);
    for (int i = tid; i < lt * BA_TILE; i += nt) {
        const int p = ba_point_of(S.ctl, i);
        if (p >= ba_fresh(S.ctl->m)) continue;
        const uint8_t* mk = mask + (size_t)p * C;
        if (first) {
            int nv = 0;
            for (int k = 0; k < C; ++k) nv += mk[k] ? 1 : 0;
            valid[p] = nv > 1 ? 1 : 0;             // helpers.py:207-208,222-223: <= 1 view is skipped
        }
        if (!valid[p]) continue;
        double X[3];
        const double r = ba_residual(Q.tb, Rt, -1, nullptr, obs + (size_t)p * C * 2, mk, C, X);
        if (first) { ba_fresh(P.X)[3 * p] = X[0]; ba_fresh(P.X)[3 * p + 1] = X[1]; ba_fresh(P.X)[3 * p + 2] = X[2]; }
        const float fv = (float)r;                             // helpers.py:273
        if (!isfinite(fv)) bad = 1.0;
        c += (double)log1pf(fv * fv);
        cnt += 1.0;
    }
    out[0] = 0.5 * ba_block_sum(c, scratch);
    out[1] = ba_block_sum(bad, scratch);
    out[2] = ba_block_sum(cnt, scratch);
}

// publish 3 numbers of this CTA, grid barrier, read the grid totals (every CTA sums in CTA order)
BA_DEV void ba_grid_sum3(const BAParams& P, const BAShared& S, int slot, const double v[3], double tot[3]) {
    const int G = S.ctl->ncta, b = S.ctl->cta;
    double* cp = ba_fresh(P.cpart) + (size_t)slot * G * 4;
    if (threadIdx.x == 0) { cp[4 * b] = v[0]; cp[4 * b + 1] = v[1]; cp[4 * b + 2] = v[2]; }
    ba_grid_sync(ba_fresh(P.bar), G);
    if (threadIdx.x < 3) {                                         // one thread per component, in CTA order; the CTA shares the result
        double a = 0.0;
        for (int g = 0; g < G; ++g) a += __ldcg(cp + 4 * g + threadIdx.x);
        S.scratch[threadIdx.x] = a;
    }
    __syncthreads();
    tot[0] = S.scratch[0]; tot[1] = S.scratch[1]; tot[2] = S.scratch[2];
    __syncthreads();
}

// write this CTA's partial system, grid barrier, add a slice of the entries over all CTAs, grid barrier
BA_DEV void ba_reduce_system(const BAParams& P, const BAParams& Q, const BAShared& S, int n_entries) {
    const int tid = threadIdx.x, nt = blockDim.x, G = S.ctl->ncta, b = S.ctl->cta;
    for (int e = tid; e < n_entries; e += nt) ba_fresh(P.part)[(size_t)b * Q.pstride + e] = S.acc[e];
    ba_grid_sync(ba_fresh(P.bar), G);
    // every CTA adds its slice of the entries over all CTAs: W threads per entry fetch the partials side by side
    // (the few loads of one thread are independent), then one thread adds the W sub-sums in a fixed order
    const int per = (n_entries + G - 1) / G;
    const int e0 = b * per, e1 = (e0 + per < n_entries) ? e0 + per : n_entries;
    const int Wd = nt >= 64 * per ? 64 : 16;
    for (int base = e0; base < e1; base += nt / Wd) {
        const int e = base + tid / Wd, j = tid % Wd;
        double s = 0.0;
        if (e < e1 && tid / Wd < nt / Wd)
            for (int g = j; g < G; g += Wd) s += ba_fresh(P.part)[(size_t)g * Q.pstride + e];
        __syncthreads();
        S.scratch[tid] = s;
        __syncthreads();
        if (j == 0 && e < e1 && tid / Wd < nt / Wd) {
            double t = 0.0;
            for (int q = 0; q < Wd; ++q) t += S.scratch[tid + q];
            ba_fresh(P.fin)[e] = t;
        }
    }
    ba_grid_sync(ba_fresh(P.bar), G);
}

// ---- prefit: Levenberg-Marquardt over poses and points --------------------------------------------------------
// accumulate the reduced camera system of this CTA's points at (S.Rt, P.X) with damping lambda into S.acc:
// [0, npair) S (upper pairs), [npair, npair+n) r, [npair+n, npair+2n) D, [npair+2n] cost
BA_DEV void ba_prefit_accumulate(const BAParams& P, const BAParams& Q, const BAShared& S, double lambda) {
    const int tid = threadIdx.x, nt = blockDim.x, C = Q.C, n = 6 * (C - 1), npair = n * (n + 1) / 2;
    const int Pp = ba_prefit_points(C, nt);
    const int lt = ba_local_tiles(S.ctl);
    // tile buffers
    double* Z = reinterpret_cast<double*>(S.uni);                 // [3*Pp][n]
    double* Jc = Z + (size_t)3 * Pp * n;                           // [Pp][C][12]
    double* Jp = Jc + (size_t)Pp * C * 12;                         // [Pp][C][6]
    double* ev = Jp + (size_t)Pp * C * 6;                          // [Pp][C][2]
    double* Li = ev + (size_t)Pp * C * 2;                          // [Pp][6]  inverse of the Cholesky factor of the damped point block
    double* yv = Li + (size_t)Pp * 6;                              // [Pp][3]  L^-1 gp
    double* gp = yv + (size_t)Pp * 3;                              // [Pp][3]
    double* pc = gp + (size_t)Pp * 3;                              // [Pp]     0.5 * squared pixel residuals of the point
    uint8_t* pres = reinterpret_cast<uint8_t*>(pc + Pp);           // [Pp][C]
    for (int e = tid; e < npair + 2 * n + 1; e += nt) S.acc[e] = 0.0;
    const int sub = BA_TILE / Pp;                                  // a BA_TILE tile is walked in `sub` pieces of Pp points
    for (int l = 0; l < lt * sub; ++l) {
        const int base = ba_point_of(S.ctl, (l / sub) * BA_TILE) + (l % sub) * Pp;
        __syncthreads();
        for (int e = tid; e < 3 * Pp * n; e += nt) Z[e] = 0.0;
        // (point, view): Jacobians
        for (int it = tid; it < Pp * C; it += nt) {
            const int c = it / Pp, pt = it - c * Pp, p = base + pt;
            bool pr = false;
            if (p < ba_fresh(S.ctl->m) && ba_fresh(P.valid)[p] && ba_fresh(P.mask)[(size_t)p * C + c]) {
                int k = 0;
                for (int cc = 0; cc < c; ++cc) k += ba_fresh(P.mask)[(size_t)p * C + cc] ? 1 : 0;
                const double Xp[3] = {ba_fresh(P.X)[3 * p], ba_fresh(P.X)[3 * p + 1], ba_fresh(P.X)[3 * p + 2]};
                BAViewJac J;
                ba_view_jacobian(S.Rt + 12 * c, Q.tb->fx[k], Q.tb->fy[k], Q.tb->cx[k], Q.tb->cy[k], Xp,
                                 ba_fresh(P.obs)[((size_t)p * C + c) * 2], ba_fresh(P.obs)[((size_t)p * C + c) * 2 + 1], J);
                double* jc = Jc + ((size_t)pt * C + c) * 12;
                double* jp = Jp + ((size_t)pt * C + c) * 6;
                for (int a = 0; a < 6; ++a) { jc[a] = J.Jc[0][a]; jc[6 + a] = J.Jc[1][a]; }
                for (int a = 0; a < 3; ++a) { jp[a] = J.Jp[0][a]; jp[3 + a] = J.Jp[1][a]; }
                ev[((size_t)pt * C + c) * 2] = J.e[0]; ev[((size_t)pt * C + c) * 2 + 1] = J.e[1];
                pr = true;
            }
            pres[pt * C + c] = pr ? 1 : 0;
        }
        __syncthreads();
        // point: Hpp, gp, Cholesky of the damped block, its inverse factor, y = L^-1 gp
        for (int pt = tid; pt < Pp; pt += nt) {
            double H[6] = {0, 0, 0, 0, 0, 0}, g3[3] = {0, 0, 0}, cst = 0.0;
            for (int c = 0; c < C; ++c) {
                if (!pres[pt * C + c]) continue;
                const double* jp = Jp + ((size_t)pt * C + c) * 6;
                const double e0 = ev[((size_t)pt * C + c) * 2], e1 = ev[((size_t)pt * C + c) * 2 + 1];
                cst += e0 * e0 + e1 * e1;
                H[0] += jp[0] * jp[0] + jp[3] * jp[3]; H[1] += jp[0] * jp[1] + jp[3] * jp[4]; H[2] += jp[0] * jp[2] + jp[3] * jp[5];
                H[3] += jp[1] * jp[1] + jp[4] * jp[4]; H[4] += jp[1] * jp[2] + jp[4] * jp[5]; H[5] += jp[2] * jp[2] + jp[5] * jp[5];
                for (int q = 0; q < 3; ++q) g3[q] += jp[q] * e0 + jp[3 + q] * e1;
            }
            pc[pt] = 0.5 * cst;
            gp[pt * 3] = g3[0]; gp[pt * 3 + 1] = g3[1]; gp[pt * 3 + 2] = g3[2];
            // damped block  [h00 h01 h02; . h11 h12; . . h22]
            const double h00 = H[0] * (1.0 + lambda), h11 = H[3] * (1.0 + lambda), h22 = H[5] * (1.0 + lambda);
            double* li = Li + (size_t)pt * 6;
            bool ok = h00 > 0.0;
            double l00 = 0, l10 = 0, l20 = 0, l11 = 0, l21 = 0, l22 = 0;
            if (ok) {
                l00 = sqrt(h00); l10 = H[1] / l00; l20 = H[2] / l00;
                const double d1 = h11 - l10 * l10;
                ok = d1 > 0.0;
                if (ok) {
                    l11 = sqrt(d1); l21 = (H[4] - l20 * l10) / l11;
                    const double d2 = h22 - l20 * l20 - l21 * l21;
                    ok = d2 > 0.0;
                    if (ok) l22 = sqrt(d2);
                }
            }
            if (ok) {
                // M = L^-1 (lower): m00 m10 m11 m20 m21 m22
                const double m00 = 1.0 / l00, m11 = 1.0 / l11, m22 = 1.0 / l22;
                const double m10 = -l10 * m00 * m11;
                const double m21 = -l21 * m11 * m22;
                const double m20 = -(l20 * m00 + l21 * m10) * m22;
                li[0] = m00; li[1] = m10; li[2] = m11; li[3] = m20; li[4] = m21; li[5] = m22;
            } else {
                for (int q = 0; q < 6; ++q) li[q] = 0.0;          // degenerate point: contributes nothing to the Schur part
            }
            yv[pt * 3] = li[0] * g3[0];
            yv[pt * 3 + 1] = li[1] * g3[0] + li[2] * g3[1];
            yv[pt * 3 + 2] = li[3] * g3[0] + li[4] * g3[1] + li[5] * g3[2];
        }
        __syncthreads();
        // (point, view != 0): Z rows = W L^-T, W = Jc^T Jp (6x3);  (W L^-T)[a][q] = sum_s W[a][s] M[q][s]
        for (int it = tid; it < Pp * C; it += nt) {
            const int c = it / Pp, pt = it - c * Pp;
            if (c == 0 || !pres[pt * C + c]) continue;            // camera 0 is pinned (helpers.py:250-253)
            const double* jc = Jc + ((size_t)pt * C + c) * 12;
            const double* jp = Jp + ((size_t)pt * C + c) * 6;
            const double* li = Li + (size_t)pt * 6;
            for (int a = 0; a < 6; ++a) {
                const double w0 = jc[a] * jp[0] + jc[6 + a] * jp[3];
                const double w1 = jc[a] * jp[1] + jc[6 + a] * jp[4];
                const double w2 = jc[a] * jp[2] + jc[6 + a] * jp[5];
                const int col = 6 * (c - 1) + a;
                Z[(size_t)(3 * pt + 0) * n + col] = w0 * li[0];
                Z[(size_t)(3 * pt + 1) * n + col] = w0 * li[1] + w1 * li[2];
                Z[(size_t)(3 * pt + 2) * n + col] = w0 * li[3] + w1 * li[4] + w2 * li[5];
            }
        }
        __syncthreads();
        // every thread updates the entries it owns: 2x2 blocks of (i, j) (n is even), so that a step over one row of Z
        // costs two 16-byte shared-memory loads per four multiply-adds
        {
            const int nb2 = n / 2, nblk = nb2 * (nb2 + 1) / 2;
            for (int blk = tid; blk < nblk; blk += nt) {
                int bi = 0, rem = blk;
                while (rem >= nb2 - bi) { rem -= nb2 - bi; ++bi; }
                const int bj = bi + rem, i0 = 2 * bi, j0 = 2 * bj;
                double a00 = 0.0, a01 = 0.0, a10 = 0.0, a11 = 0.0;
                for (int r = 0; r < 3 * Pp; ++r) {
                    const double2 zi = *reinterpret_cast<const double2*>(Z + (size_t)r * n + i0);
                    const double2 zj = *reinterpret_cast<const double2*>(Z + (size_t)r * n + j0);
                    a00 -= zi.x * zj.x; a01 -= zi.x * zj.y; a10 -= zi.y * zj.x; a11 -= zi.y * zj.y;
                }
                if (bi / 3 == bj / 3) {                           // same camera block: + Jc^T Jc
                    const int c = bi / 3 + 1, a = i0 % 6, b2 = j0 % 6;
                    for (int pt = 0; pt < Pp; ++pt)
                        if (pres[pt * C + c]) {
                            const double* jc = Jc + ((size_t)pt * C + c) * 12;
                            a00 += jc[a] * jc[b2] + jc[6 + a] * jc[6 + b2];
                            a01 += jc[a] * jc[b2 + 1] + jc[6 + a] * jc[6 + b2 + 1];
                            a10 += jc[a + 1] * jc[b2] + jc[6 + a + 1] * jc[6 + b2];
                            a11 += jc[a + 1] * jc[b2 + 1] + jc[6 + a + 1] * jc[6 + b2 + 1];
                        }
                }
                const int k0 = i0 * n - i0 * (i0 - 1) / 2 + (j0 - i0);            // (i0, j0), (i0, j0 + 1) are neighbours in row i0
                const int k1 = (i0 + 1) * n - (i0 + 1) * i0 / 2 + (j0 - i0 - 1);  // (i0 + 1, j0)
                S.acc[k0] += a00; S.acc[k0 + 1] += a01;
                S.acc[k1 + 1] += a11;
                if (bi < bj) S.acc[k1] += a10;                    // below the diagonal inside a diagonal block
            }
        }
        for (int i = tid; i < n; i += nt) {
            const int c = i / 6 + 1, a = i % 6;
            double r = 0.0, d = 0.0;
            for (int pt = 0; pt < Pp; ++pt)
                if (pres[pt * C + c]) {
                    const double* jc = Jc + ((size_t)pt * C + c) * 12;
                    r += jc[a] * ev[((size_t)pt * C + c) * 2] + jc[6 + a] * ev[((size_t)pt * C + c) * 2 + 1];
                    d += jc[a] * jc[a] + jc[6 + a] * jc[6 + a];
                }
            for (int rr = 0; rr < 3 * Pp; ++rr) r -= Z[(size_t)rr * n + i] * yv[rr];
            S.acc[npair + i] += r;
            S.acc[npair + n + i] += d;
        }
        if (tid == 0) {
            double cst = 0.0;
            for (int pt = 0; pt < Pp; ++pt) if (base + pt < ba_fresh(S.ctl->m) && ba_fresh(P.valid)[base + pt]) cst += pc[pt];
            S.acc[npair + 2 * n] += cst;
        }
    }
    __syncthreads();
}

// back-substitution of this CTA's points for the camera step dc (S.p) at (S.Rt, P.X) -> P.Xnew, and
// 0.5 * squared pixel residuals at (S.Rt_new, P.Xnew)
BA_DEV double ba_prefit_backsub(const BAParams& P, const BAParams& Q, const BAShared& S, double lambda, double* scratch) {
    const int tid = threadIdx.x, nt = blockDim.x, C = Q.C;
    const int lt = ba_local_tiles(S.ctl);
    double cst = 0.0;
    const uint8_t* const mask = ba_fresh(P.mask);
    const double* const obs = ba_fresh(P.obs);
    for (int i = tid; i < lt * BA_TILE; i += nt) {
        const int p = ba_point_of(S.ctl, i);
        if (p >= ba_fresh(S.ctl->m) || !ba_fresh(P.valid)[p]) continue;
        const double Xp[3] = {ba_fresh(P.X)[3 * p], ba_fresh(P.X)[3 * p + 1], ba_fresh(P.X)[3 * p + 2]};
        double H[6] = {0, 0, 0, 0, 0, 0}, rhs[3] = {0, 0, 0};
        int k = 0;
        for (int c = 0; c < C; ++c) {
            if (!mask[(size_t)p * C + c]) continue;
            BAViewJac J;
            ba_view_jacobian(S.Rt + 12 * c, Q.tb->fx[k], Q.tb->fy[k], Q.tb->cx[k], Q.tb->cy[k], Xp,
                             obs[((size_t)p * C + c) * 2], obs[((size_t)p * C + c) * 2 + 1], J);
            ++k;
            H[0] += J.Jp[0][0] * J.Jp[0][0] + J.Jp[1][0] * J.Jp[1][0]; H[1] += J.Jp[0][0] * J.Jp[0][1] + J.Jp[1][0] * J.Jp[1][1];
            H[2] += J.Jp[0][0] * J.Jp[0][2] + J.Jp[1][0] * J.Jp[1][2]; H[3] += J.Jp[0][1] * J.Jp[0][1] + J.Jp[1][1] * J.Jp[1][1];
            H[4] += J.Jp[0][1] * J.Jp[0][2] + J.Jp[1][1] * J.Jp[1][2]; H[5] += J.Jp[0][2] * J.Jp[0][2] + J.Jp[1][2] * J.Jp[1][2];
            double s0 = J.e[0], s1 = J.e[1];                        // e + Jc dc
            if (c > 0) {
                const double* d = S.p + 6 * (c - 1);
                for (int a = 0; a < 6; ++a) { s0 += J.Jc[0][a] * d[a]; s1 += J.Jc[1][a] * d[a]; }
            }
            for (int q = 0; q < 3; ++q) rhs[q] += J.Jp[0][q] * s0 + J.Jp[1][q] * s1;   // gp + W^T dc
        }
        const double h00 = H[0] * (1.0 + lambda), h11 = H[3] * (1.0 + lambda), h22 = H[5] * (1.0 + lambda);
        double dp[3] = {0, 0, 0};
        if (h00 > 0.0) {
            const double l00 = sqrt(h00), l10 = H[1] / l00, l20 = H[2] / l00;
            const double d1 = h11 - l10 * l10;
            if (d1 > 0.0) {
                const double l11 = sqrt(d1), l21 = (H[4] - l20 * l10) / l11;
                const double d2 = h22 - l20 * l20 - l21 * l21;
                if (d2 > 0.0) {
                    const double l22 = sqrt(d2);
                    const double y0 = rhs[0] / l00, y1 = (rhs[1] - l10 * y0) / l11, y2 = (rhs[2] - l20 * y0 - l21 * y1) / l22;
                    dp[2] = y2 / l22; dp[1] = (y1 - l21 * dp[2]) / l11; dp[0] = (y0 - l10 * dp[1] - l20 * dp[2]) / l00;
                }
            }
        }
        const double Xn[3] = {Xp[0] - dp[0], Xp[1] - dp[1], Xp[2] - dp[2]};
        ba_fresh(P.Xnew)[3 * p] = Xn[0]; ba_fresh(P.Xnew)[3 * p + 1] = Xn[1]; ba_fresh(P.Xnew)[3 * p + 2] = Xn[2];
        k = 0;
        for (int c = 0; c < C; ++c)
            if (mask[(size_t)p * C + c]) {
                const double* Rt = S.Rt_new + 12 * c;
                const double x = Rt[0] * Xn[0] + Rt[1] * Xn[1] + Rt[2] * Xn[2] + Rt[3];
                const double y = Rt[4] * Xn[0] + Rt[5] * Xn[1] + Rt[6] * Xn[2] + Rt[7];
                const double z = Rt[8] * Xn[0] + Rt[9] * Xn[1] + Rt[10] * Xn[2] + Rt[11];
                const double eu = Q.tb->fx[k] * x / z + Q.tb->cx[k] - obs[((size_t)p * C + c) * 2];
                const double ev = Q.tb->fy[k] * y / z + Q.tb->cy[k] - obs[((size_t)p * C + c) * 2 + 1];
                cst += eu * eu + ev * ev;
                ++k;
            }
    }
    return 0.5 * ba_block_sum(cst, scratch);
}

// ---- polish: scipy's trust-region iteration on the reference objective ------------------------------------------
// finite-difference columns at S.x (scipy _compute_absolute_step / 2-point): colRt, colcam, dx
BA_DEV void ba_make_columns(const BAParams& P, const BAParams& Q, const BAShared& S) {
    const int tid = threadIdx.x, nt = blockDim.x, C = Q.C, n = 6 * (C - 1);
    for (int j = tid; j < n; j += nt) {
        const int cam = 1 + j / 6, idx = 1 + 7 * (cam - 1) + 1 + j % 6;
        double xq[7];
        for (int q = 0; q < 7; ++q) xq[q] = S.x[1 + 7 * (cam - 1) + q];
        const double x0 = S.x[idx];
        const double h = 1.4901161193847656e-08 * (x0 >= 0 ? 1.0 : -1.0) * fmax(1.0, fabs(x0));
        const double xp = x0 + h;
        xq[1 + j % 6] = xp;
        S.dx[j] = xp - x0;
        S.colcam[j] = cam;
        double R[9];
        ba_rotvec_to_matrix(xq + 1, R);
        double* Rt = S.colRt + 12 * j;
        for (int i = 0; i < 3; ++i) { for (int jj = 0; jj < 3; ++jj) Rt[4 * i + jj] = R[3 * i + jj]; Rt[4 * i + 3] = xq[4 + i]; }
    }
    __syncthreads();
}

// robust-scaled normal equations of this CTA's points at S.x (S.Rt holds its poses) into S.acc:
// [0, npair) J^T J (upper pairs), [npair, npair+n) J^T f, [npair+n] cost, [npair+n+1] non-finite
BA_DEV void ba_polish_accumulate(const BAParams& P, const BAParams& Q, const BAShared& S) {
    const int tid = threadIdx.x, nt = blockDim.x, C = Q.C, n = 6 * (C - 1), npair = n * (n + 1) / 2, ncol = n + 1;
    const int lt = ba_local_tiles(S.ctl);
    double* F = reinterpret_cast<double*>(S.uni);                  // [BA_TILE][ncol] residuals, then the scaled Jacobian rows
    double* fs = F + (size_t)BA_TILE * ncol;                        // [BA_TILE] scaled residual
    double* ct = fs + BA_TILE;                                      // [BA_TILE] log1p(f^2)
    for (int e = tid; e < npair + n + 2; e += nt) S.acc[e] = 0.0;
    for (int l = 0; l < lt; ++l) {
        const int base = ba_point_of(S.ctl, l * BA_TILE);
        const uint8_t* const mask = ba_fresh(P.mask);
        const double* const obs = ba_fresh(P.obs);
        const uint8_t* const valid = ba_fresh(P.valid);
        const int m = ba_fresh(S.ctl->m);
        __syncthreads();
        // (column, point): one warp = one column of the tile
        for (int it = tid; it < BA_TILE * ncol; it += nt) {
            const int col = it / BA_TILE, pt = it - col * BA_TILE, p = base + pt;
            double r = 0.0;
            if (p < m && valid[p]) {
                const uint8_t* mk = mask + (size_t)p * C;
                const int cam = col == 0 ? -1 : S.colcam[col - 1];
                if (cam < 0 || mk[cam]) {                          // a column that touches no view of the point: difference 0
                    double X[3];
                    r = ba_residual(Q.tb, S.Rt, cam, cam < 0 ? nullptr : S.colRt + 12 * (col - 1), obs + (size_t)p * C * 2, mk, C, X);
                }
            }
            F[(size_t)pt * ncol + col] = r;
        }
        __syncthreads();
        // point: Cauchy pieces in the precisions scipy uses for a float32 residual vector (as k_ba_rows)
        for (int pt = tid; pt < BA_TILE; pt += nt) {
            const int p = base + pt;
            double* row = F + (size_t)pt * ncol;
            if (!(p < m && valid[p])) {
                fs[pt] = 0.0; ct[pt] = 0.0;
                for (int j = 0; j < n; ++j) row[j] = 0.0;
                continue;
            }
            const uint8_t* mk = mask + (size_t)p * C;
            const double f0d = row[0];
            const float fv = (float)f0d;
            if (!isfinite(fv)) S.acc[npair + n + 1] = 1.0;          // any writer stores the same value
            const float z = fv * fv, t1 = 1.0f + z;
            const float rho1 = 1.0f / t1, rho2 = -(1.0f / (t1 * t1));
            ct[pt] = (double)log1pf(z);
            double js = (double)rho1 + 2.0 * (double)rho2 * (double)z;
            if (js < 2.220446049250313e-16) js = 2.220446049250313e-16;
            js = sqrt(js);
            fs[pt] = (double)(float)((double)fv * ((double)rho1 / js));
            for (int j = 0; j < n; ++j) {                          // in place: entry j is written after entry j + 1 was read
                double Jv = 0.0;
                if (mk[S.colcam[j]]) {
                    if (Q.jac_mode == 0) Jv = (double)((float)row[j + 1] - fv) / S.dx[j];
                    else Jv = (row[j + 1] - f0d) / S.dx[j];
                }
                row[j] = Jv * js;
            }
        }
        __syncthreads();
        for (int k = tid; k < npair; k += nt) {
            const int i = S.pi[k], j = S.pj[k];
            double s = 0.0;
            for (int pt = 0; pt < BA_TILE; ++pt) s += F[(size_t)pt * ncol + i] * F[(size_t)pt * ncol + j];
            S.acc[k] += s;
        }
        for (int i = tid; i < n; i += nt) {
            double s = 0.0;
            for (int pt = 0; pt < BA_TILE; ++pt) s += F[(size_t)pt * ncol + i] * fs[pt];
            S.acc[npair + i] += s;
        }
        if (tid == 0) {
            double s = 0.0;
            for (int pt = 0; pt < BA_TILE; ++pt) s += ct[pt];
            S.acc[npair + n] += 0.5 * s;
        }
    }
    __syncthreads();
}

// sum over the warp of per-lane partial sums, fixed tree: every CTA gets the same bits
BA_DEV double ba_warp_sum(double v) {
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// load the reduced system P.fin -> S.A (full symmetric), S.g
BA_DEV void ba_load_system(const BAParams& P, const BAShared& S, int n) {
    const int tid = threadIdx.x, nt = blockDim.x, npair = n * (n + 1) / 2;
    __syncthreads();
    for (int k = tid; k < npair; k += nt) {
        const int i = S.pi[k], j = S.pj[k];
        const double v = ba_fresh(P.fin)[k];
        S.A[(size_t)i * n + j] = v; S.A[(size_t)j * n + i] = v;
    }
    for (int i = tid; i < n; i += nt) S.g[i] = ba_fresh(P.fin)[npair + i];
    __syncthreads();
    if (tid == 0) {
        double d = 0.0;
        for (int i = 0; i < n; ++i) d = fmax(d, fabs(S.A[(size_t)i * n + i]));
        S.ctl->a_diag = d;
    }
    __syncthreads();
}

// Householder tridiagonalisation of the symmetric S.A (destroyed): A = Q T Q^T with T = tridiag(S.td, S.te) and
// Q^T left in S.L (row j = j-th basis vector), then ghat = Q^T g.  Once per linearisation; it plays the part of the
// SVD scipy takes of J (trf.py: "U, s, V = svd(J_h)"): afterwards every trust-region sub-problem at this point costs
// O(n) per trial alpha.  The symmetric access A[j][i] / Qt[j][r] keeps consecutive threads on consecutive words.
BA_DEV void ba_tridiagonalise(const BAShared& S, int n) {
    const int tid = threadIdx.x, nt = blockDim.x;
    BACtrl* ctl = S.ctl;
    double* A = S.A;
    double* Qt = S.L;
    __syncthreads();
    for (int e = tid; e < n * n; e += nt) Qt[e] = (e / n == e % n) ? 1.0 : 0.0;
    __syncthreads();
    for (int k = 0; k + 2 < n; ++k) {
        if (tid < 32) {
            double part = 0.0;
            for (int i = k + 1 + tid; i < n; i += 32) part += A[(size_t)i * n + k] * A[(size_t)i * n + k];
            const double sigma = ba_warp_sum(part);
            if (tid == 0) {
            const double x0 = A[(size_t)(k + 1) * n + k];
            double tail = sigma - x0 * x0;                          // what the reflection has to remove
            if (!(tail > 0.0)) { ctl->hh_beta = 0.0; ctl->hh_alpha = x0; }
            else {
                const double nrm = sqrt(sigma);
                const double alpha = x0 >= 0.0 ? -nrm : nrm;
                const double v0 = x0 - alpha;
                ctl->hh_beta = 2.0 / (tail + v0 * v0);
                ctl->hh_alpha = alpha;
                S.hv[k + 1] = v0;
            }
            }
        }
        __syncthreads();
        const double beta = ctl->hh_beta;
        if (beta == 0.0) { if (tid == 0) S.te[k] = ctl->hh_alpha; __syncthreads(); continue; }     // column already tridiagonal
        for (int i = k + 2 + tid; i < n; i += nt) S.hv[i] = A[(size_t)i * n + k];
        __syncthreads();
        // p = beta * A v on the trailing block (threads 0..m-1), u = Q v (threads after them)
        const int m = n - k - 1;
        for (int it = tid; it < m + n; it += nt) {
            if (it < m) {
                const int i = k + 1 + it;
                double acc = 0.0;
                for (int j = k + 1; j < n; ++j) acc += A[(size_t)j * n + i] * S.hv[j];
                S.hp[i] = beta * acc;
            } else {
                const int r = it - m;
                double acc = 0.0;
                for (int j = k + 1; j < n; ++j) acc += Qt[(size_t)j * n + r] * S.hv[j];
                S.hu[r] = beta * acc;
            }
        }
        __syncthreads();
        if (tid < 32) {
            double part = 0.0;
            for (int i = k + 1 + tid; i < n; i += 32) part += S.hp[i] * S.hv[i];
            const double dot = ba_warp_sum(part);
            if (tid == 0) ctl->hh_K = 0.5 * beta * dot;
        }
        __syncthreads();
        const double K = ctl->hh_K;
        for (int i = k + 1 + tid; i < n; i += nt) S.hp[i] -= K * S.hv[i];      // w
        __syncthreads();
        for (int idx = tid; idx < m * m + m * n; idx += nt) {
            if (idx < m * m) {
                const int ii = idx / m, jj = idx - ii * m, i = k + 1 + ii, j = k + 1 + jj;
                A[(size_t)i * n + j] -= S.hv[i] * S.hp[j] + S.hp[i] * S.hv[j];
            } else {
                const int e2 = idx - m * m, jj = e2 / n, r = e2 - jj * n, j = k + 1 + jj;
                Qt[(size_t)j * n + r] -= S.hv[j] * S.hu[r];
            }
        }
        if (tid == 0) S.te[k] = ctl->hh_alpha;
        __syncthreads();
    }
    if (tid == 0) { if (n >= 2) S.te[n - 2] = A[(size_t)(n - 1) * n + n - 2]; S.te[n - 1] = 0.0; }
    for (int i = tid; i < n; i += nt) S.td[i] = A[(size_t)i * n + i];
    for (int j = tid; j < n; j += nt) {
        double acc = 0.0;
        for (int r = 0; r < n; ++r) acc += Qt[(size_t)j * n + r] * S.g[r];
        S.ghat[j] = acc;
    }
    __syncthreads();
}

// one WARP: (T + alpha I) x = rhs for the symmetric tridiagonal T = tridiag(S.td, S.te) by parallel cyclic reduction:
// ceil(log2 n) steps, in each of which every equation i eliminates its neighbours i - s and i + s (two independent
// divisions per equation), instead of a chain of n dependent pivots -- the trust-region sub-problem evaluates this
// twice per Newton step on alpha and used to spend most of its time in that chain.  For a positive definite matrix
// every diagonal entry stays positive (they are Schur complements); returns false (warp-uniform) if one does not.
BA_DEV bool ba_pcr_solve(const BAShared& S, int n, double alpha, const double* rhs, double* x, int lane) {
    // two generations of (a, b, 1/b, c, d): an equation stores the reciprocal of its diagonal entry next to it, so that
    // a step costs ONE division per equation (its own new diagonal) and its neighbours only multiply
    double* buf = S.pcr;
    int cur = 0;
    bool ok = true;
    for (int i = lane; i < n; i += 32) {
        const double b = S.td[i] + alpha;
        if (!(b > 0.0)) ok = false;
        buf[0 * n + i] = i > 0 ? S.te[i - 1] : 0.0;               // a: sub-diagonal
        buf[1 * n + i] = b;                                        // diagonal
        buf[2 * n + i] = 1.0 / b;
        buf[3 * n + i] = i + 1 < n ? S.te[i] : 0.0;                // c: super-diagonal
        buf[4 * n + i] = rhs[i];
    }
    __syncwarp();
    for (int st = 1; st < n; st <<= 1) {
        const double* A0 = buf + (size_t)(5 * cur + 0) * n; const double* B0 = buf + (size_t)(5 * cur + 1) * n;
        const double* R0 = buf + (size_t)(5 * cur + 2) * n; const double* C0 = buf + (size_t)(5 * cur + 3) * n;
        const double* D0 = buf + (size_t)(5 * cur + 4) * n;
        double* A1 = buf + (size_t)(5 * (cur ^ 1) + 0) * n; double* B1 = buf + (size_t)(5 * (cur ^ 1) + 1) * n;
        double* R1 = buf + (size_t)(5 * (cur ^ 1) + 2) * n; double* C1 = buf + (size_t)(5 * (cur ^ 1) + 3) * n;
        double* D1 = buf + (size_t)(5 * (cur ^ 1) + 4) * n;
        for (int i = lane; i < n; i += 32) {
            const int im = i - st, ip = i + st;
            double bb = B0[i], dd = D0[i], aa = 0.0, cc = 0.0;
            if (im >= 0) { const double k1 = A0[i] * R0[im]; bb -= C0[im] * k1; dd -= D0[im] * k1; aa = -A0[im] * k1; }
            if (ip < n) { const double k2 = C0[i] * R0[ip]; bb -= A0[ip] * k2; dd -= D0[ip] * k2; cc = -C0[ip] * k2; }
            if (!(bb > 0.0)) ok = false;
            A1[i] = aa; B1[i] = bb; R1[i] = 1.0 / bb; C1[i] = cc; D1[i] = dd;
        }
        __syncwarp();
        cur ^= 1;
    }
    const double* Rf = buf + (size_t)(5 * cur + 2) * n; const double* Df = buf + (size_t)(5 * cur + 4) * n;
    for (int i = lane; i < n; i += 32) x[i] = Df[i] * Rf[i];
    ok = __ballot_sync(0xffffffffu, ok ? 0 : 1) == 0u;
    __syncwarp();
    return ok;
}

// scipy common.py solve_lsq_trust_region (rank-deficient branch, as the reference's dead focal parameters force):
// step p of norm Delta minimising the quadratic model, iterated in the tridiagonal basis of ba_tridiagonalise:
// phi(alpha) = |(T + alpha I)^-1 ghat| - Delta and phi'(alpha) = -y^T (T + alpha I)^-1 y / |y| are what scipy
// evaluates from the singular values.  One warp runs the Newton iteration on alpha (every lane carries the same
// scalars).  In: ctl->Delta, ctl->alpha.  Out: S.p, ctl->alpha, ctl->pred (the predicted reduction
// -(0.5 p^T A p + g^T p)), ctl->step_norm.
BA_DEV void ba_solve_tr(const BAShared& S, int n) {
    const int tid = threadIdx.x, nt = blockDim.x;
    BACtrl* ctl = S.ctl;
    __syncthreads();
    if (tid < 32) {
        const int lane = tid;
        const double Delta = ctl->Delta;
        double part = 0.0;
        for (int i = lane; i < n; i += 32) { part += S.ghat[i] * S.ghat[i]; S.q[i] = -S.ghat[i]; }
        double upper = sqrt(ba_warp_sum(part)) / Delta, lower = 0.0;
        double alpha = ctl->alpha;
        if (alpha == 0.0) alpha = fmax(0.001 * upper, sqrt(lower * upper));
        __syncwarp();
        int newton = 0;
        for (int it = 0; it < 10; ++it) {
            ++newton;
            if (alpha < lower || alpha > upper) alpha = fmax(0.001 * upper, sqrt(lower * upper));
            int tries = 0;
            while (!ba_pcr_solve(S, n, alpha, S.q, S.yhat, lane) && tries < 64) {        // rounding: T + alpha I not positive
                const double floor_a = 2.220446049250313e-16 * ctl->a_diag * (double)(1 << (tries < 30 ? tries : 30));
                lower = fmax(lower, alpha);
                alpha = fmax(2.0 * alpha, floor_a);
                if (alpha > upper) upper = alpha;
                ++tries;
            }
            ba_pcr_solve(S, n, alpha, S.yhat, S.zhat, lane);
            double p2 = 0.0, yz = 0.0;
            for (int i = lane; i < n; i += 32) { p2 += S.yhat[i] * S.yhat[i]; yz += S.yhat[i] * S.zhat[i]; }
            const double pn = sqrt(ba_warp_sum(p2));
            yz = ba_warp_sum(yz);
            const double phi = pn - Delta, phi_prime = -yz / pn;
            if (phi < 0) upper = alpha;
            const double ratio = phi / phi_prime;
            lower = fmax(lower, alpha - ratio);
            alpha -= (phi + Delta) * ratio / Delta;
            if (fabs(phi) < 0.01 * Delta) break;
        }
        int tries = 0;
        while (!ba_pcr_solve(S, n, alpha, S.q, S.yhat, lane) && tries < 64) {
            alpha = fmax(2.0 * alpha, 2.220446049250313e-16 * ctl->a_diag * (double)(1 << (tries < 30 ? tries : 30)));
            ++tries;
        }
        double p2 = 0.0;
        for (int i = lane; i < n; i += 32) p2 += S.yhat[i] * S.yhat[i];
        const double pn = sqrt(ba_warp_sum(p2));
        const double sc = pn > 0.0 ? Delta / pn : 0.0;
        for (int i = lane; i < n; i += 32) S.yhat[i] *= sc;
        __syncwarp();
        double l = 0.0, qd = 0.0;                                   // g^T p = ghat^T phat, p^T A p = phat^T T phat
        for (int i = lane; i < n; i += 32) {
            l += S.yhat[i] * S.ghat[i];
            double r = S.td[i] * S.yhat[i];
            if (i > 0) r += S.te[i - 1] * S.yhat[i - 1];
            if (i + 1 < n) r += S.te[i] * S.yhat[i + 1];
            qd += S.yhat[i] * r;
        }
        l = ba_warp_sum(l); qd = ba_warp_sum(qd);
        if (lane == 0) {
            ctl->pred = -(0.5 * qd + l);
            ctl->alpha = alpha;
            ctl->tr_calls += 1; ctl->tr_its += newton;
        }
    }
    __syncthreads();
    for (int r = tid; r < n; r += nt) {                            // p = Q phat
        double acc = 0.0;
        for (int j = 0; j < n; ++j) acc += S.L[(size_t)j * n + r] * S.yhat[j];
        S.p[r] = acc;
    }
    __syncthreads();
    if (tid == 0) ctl->step_norm = ba_norm2_serial(S.p, n);
    __syncthreads();
}

// the whole solve; every CTA runs the same control flow on the same numbers.
// P: this CTA's problem.  Q: any problem of the launch, read ONLY for what all of them share (cameras, options,
// pstride): in a batched launch Q is problem 0, whose fields sit at fixed offsets of the kernel parameter, so that
// the hot loops read them as constants instead of through the per-CTA problem index
BA_DEV void ba_solve_body(const BAParams& P, const BAParams& Q, unsigned char* smem) {
    const int tid = threadIdx.x, nt = blockDim.x, C = Q.C;
    const int n = 6 * (C - 1), nf = 1 + 7 * (C - 1), npair = n * (n + 1) / 2;
    const BAShared S = ba_carve(smem, C, nt);
    BACtrl* ctl = S.ctl;
    double* scratch = S.scratch;
    int slot = 0;

    if (tid == 0) {
        int m = P.m_dev ? *P.m_dev : P.m_max;
        if (m > P.m_max) m = P.m_max;
        if (m < 0) m = 0;
        ctl->m = m; ctl->ntiles = (m + BA_TILE - 1) / BA_TILE;
        ctl->cta = (int)blockIdx.x - P.cta0; ctl->ncta = P.ncta > 0 ? P.ncta : (int)gridDim.x;
        S.x[0] = Q.tb->Kmat[0][0];
    }
    for (int k = tid; k < npair; k += nt) {                        // pair table: k -> (i, j), i <= j, row by row
        int i = 0, rem = k;
        while (rem >= n - i) { rem -= n - i; ++i; }
        S.pi[k] = (uint8_t)i; S.pj[k] = (uint8_t)(i + rem);
    }
    for (int c = 1 + tid; c < C; c += nt) {                        // helpers.py:278-285
        double* q = S.x + 1 + 7 * (c - 1);
        q[0] = Q.tb->Kmat[c - 1][0];
        ba_matrix_to_rotvec(P.R + 9 * c, q + 1);
        q[4] = P.t[3 * c]; q[5] = P.t[3 * c + 1]; q[6] = P.t[3 * c + 2];
    }
    __syncthreads();
    for (int c = tid; c < C; c += nt) ba_pose_from_x(S.x, c, S.Rt + 12 * c);
    __syncthreads();

    if (tid == 0) { for (int k = 0; k < 8; ++k) ctl->prof[k] = 0; ctl->t_last = ba_clock(); }
    // reference objective and DLT points at the start
    double v3[3], tot[3];
    ba_cost_pass(P, Q, S, S.Rt, true, scratch, v3);
    ba_grid_sum3(P, S, slot, v3, tot); slot ^= 1;
    if (tid == 0) {
        ctl->cost_initial = tot[0]; ctl->cost = tot[0]; ctl->finite = tot[1] == 0.0; ctl->n_valid = (int)tot[2];
        ctl->pf_cost0 = 0.0; ctl->pf_cost1 = 0.0; ctl->pf_it = 0; ctl->pf_taken = 0;
        ctl->nfev = 0; ctl->njev = 0; ctl->iteration = 0; ctl->termination = -99; ctl->g_norm = 0.0; ctl->tr_its = 0; ctl->tr_calls = 0;
    }
    __syncthreads();
    if (ctl->n_valid == 0) {
        if (ctl->cta == 0 && tid == 0 && P.report) {
            mocap_ba_report r;
            r.cost_initial = 0; r.cost_final = 0; r.optimality = 0; r.n_iterations = 0; r.n_fev = 0; r.status = -3; r.n_residuals = 0;
            r.prefit_cost_initial = 0; r.prefit_cost_final = 0; r.prefit_iterations = 0; r.n_launches = 1;
            r.n_tr_solves = 0; r.n_tr_newton = 0;
            for (int k = 0; k < 8; ++k) r.phase_ms[k] = 0.0f;
            *P.report = r;
        }
        return;
    }

    // ---- prefit ------------------------------------------------------------------------------------------------
    if (Q.prefit) {
        const int max_iter = Q.prefit_max_iter > 0 ? Q.prefit_max_iter : 50;
        if (tid == 0) { ctl->lambda = 1e-3; ctl->go = 1; ctl->pcost = -1.0; }
        __syncthreads();
        int it = 0;
        while (it < max_iter && ctl->go) {
            const double lambda = ctl->lambda;
            __syncthreads();                                       // everybody has read go / lambda
            BA_TICK(BA_PH_SETUP);
            ba_prefit_accumulate(P, Q, S, lambda);
            ba_reduce_system(P, Q, S, npair + 2 * n + 1);
            ba_load_system(P, S, n);                               // S.A = S, S.g = r
            BA_TICK(BA_PH_PF_SYSTEM);
            if (tid == 0) {
                const double c0 = ba_fresh(P.fin)[npair + 2 * n];
                if (ctl->pcost < 0.0) { ctl->pf_cost0 = c0; ctl->pf_cost1 = c0; }
                ctl->pcost = c0;
                ctl->flag = 1;
            }
            // a parameter with a zero diagonal belongs to a camera that sees no point: its rows of the reduced system are
            // zero at every lambda, so it is pinned (unit diagonal, zero right-hand side) and its step is 0
            for (int e = tid; e < n * n; e += nt) {
                const int i = e / n, j = e - i * n;
                const double Di = ba_fresh(P.fin)[npair + n + i], Dj = ba_fresh(P.fin)[npair + n + j];
                S.L[e] = (Di == 0.0 || Dj == 0.0) ? (i == j ? 1.0 : 0.0) : S.A[e] + (i == j ? lambda * Di : 0.0);
            }
            __syncthreads();
            const bool pd = ba_chol_factor(S.L, n, &ctl->flag);
            if (!pd) {
                __syncthreads();
                if (tid == 0) { ctl->lambda *= 10.0; if (ctl->lambda > 1e12) ctl->go = 0; }
                ++it;
                __syncthreads();
                continue;
            }
            for (int i = tid; i < n; i += nt) S.p[i] = ba_fresh(P.fin)[npair + n + i] == 0.0 ? 0.0 : -S.g[i];
            __syncthreads();
            ba_solve_lower(S.L, n, S.p);
            ba_solve_upper(S.L, n, S.p);                           // dc
            for (int c = tid; c < C; c += nt) {                    // candidate poses: R' = Exp(dw) R, t' = t + dt
                double* o = S.Rt_new + 12 * c;
                const double* r0 = S.Rt + 12 * c;
                if (c == 0) { for (int i = 0; i < 12; ++i) o[i] = r0[i]; continue; }
                const double* d = S.p + 6 * (c - 1);
                double E[9];
                ba_exp_so3(d, E);
                for (int i = 0; i < 3; ++i) {
                    for (int j = 0; j < 3; ++j) {
                        double v = 0;
                        for (int k = 0; k < 3; ++k) v += E[3 * i + k] * r0[4 * k + j];
                        o[4 * i + j] = v;
                    }
                    o[4 * i + 3] = r0[4 * i + 3] + d[3 + i];
                }
            }
            __syncthreads();
            BA_TICK(BA_PH_PF_SOLVE);
            v3[0] = ba_prefit_backsub(P, Q, S, lambda, scratch); v3[1] = 0.0; v3[2] = 0.0;
            ba_grid_sum3(P, S, slot, v3, tot); slot ^= 1;
            BA_TICK(BA_PH_PF_TRIAL);
            const double cost = ctl->pcost, cost_new = tot[0];
            const bool accept = cost_new < cost && isfinite(cost_new);
            __syncthreads();
            if (accept) {
                for (int e = tid; e < C * 12; e += nt) S.Rt[e] = S.Rt_new[e];
                const int lt = ba_local_tiles(ctl);
                for (int i = tid; i < lt * BA_TILE; i += nt) {
                    const int p = ba_point_of(S.ctl, i);
                    if (p < ctl->m && ba_fresh(P.valid)[p]) {
                        double* X = ba_fresh(P.X);
                        const double* Xn = ba_fresh(P.Xnew);
                        X[3 * p] = Xn[3 * p]; X[3 * p + 1] = Xn[3 * p + 1]; X[3 * p + 2] = Xn[3 * p + 2];
                    }
                }
                if (tid == 0) {
                    const double rel = (cost - cost_new) / fmax(cost, 1e-300);
                    ctl->pf_cost1 = cost_new;
                    ctl->pf_taken = 1;
                    ctl->lambda = fmax(lambda * 0.3, 1e-12);
                    if (rel < BA_PREFIT_REL_STOP) ctl->go = 0;
                }
            } else if (tid == 0) {
                ctl->pf_cost1 = cost;
                ctl->lambda = lambda * 10.0;
                if (ctl->lambda > 1e12) ctl->go = 0;
            }
            ++it;
            __syncthreads();
        }
        if (tid == 0) ctl->pf_it = it;
        // poses -> parameter vector (rotation vector round trip, as ba.cu)
        for (int c = 1 + tid; c < C; c += nt) {
            const double* r0 = S.Rt + 12 * c;
            const double Rc[9] = {r0[0], r0[1], r0[2], r0[4], r0[5], r0[6], r0[8], r0[9], r0[10]};
            double* q = S.x + 1 + 7 * (c - 1);
            ba_matrix_to_rotvec(Rc, q + 1);
            q[4] = r0[3]; q[5] = r0[7]; q[6] = r0[11];
        }
        __syncthreads();
        for (int c = tid; c < C; c += nt) ba_pose_from_x(S.x, c, S.Rt + 12 * c);
        __syncthreads();
    }

    // ---- polish: trf_no_bounds -----------------------------------------------------------------------------------
    // linearize at x
    BA_TICK(BA_PH_SETUP);
    ba_make_columns(P, Q, S);
    ba_polish_accumulate(P, Q, S);
    ba_reduce_system(P, Q, S, npair + n + 2);
    ba_load_system(P, S, n);
    BA_TICK(BA_PH_LINEARIZE);
    ba_tridiagonalise(S, n);
    BA_TICK(BA_PH_TRIDIAG);
    if (tid == 0) {
        ctl->cost = ba_fresh(P.fin)[npair + n]; ctl->finite = ba_fresh(P.fin)[npair + n + 1] == 0.0;
        if (!Q.prefit) ctl->cost_initial = ctl->cost;
        ctl->nfev = 1; ctl->njev = 1;
        // after a prefit that took a step the start is already close (ba.cu); otherwise the polish starts as scipy does
        double D = (Q.prefit && ctl->pf_taken) ? BA_POLISH_RADIUS : ba_norm2_serial(S.x, nf);
        if (D == 0.0) D = 1.0;
        ctl->Delta = D; ctl->alpha = 0.0; ctl->iteration = 0; ctl->termination = -99;
        if (!ctl->finite) ctl->termination = -1;
    }
    __syncthreads();
    const int max_nfev = Q.max_nfev > 0 ? Q.max_nfev : nf * 100;
    while (ctl->termination == -99) {
        __syncthreads();                                           // everybody has evaluated the loop condition
        if (tid == 0) {
            double gn = 0.0;
            for (int i = 0; i < n; ++i) gn = fmax(gn, fabs(S.g[i]));
            ctl->g_norm = gn;
            if (gn < Q.gtol) ctl->termination = 1;
            ctl->go = (ctl->termination == -99 && ctl->nfev != max_nfev) ? 1 : 0;
            ctl->actual = -1.0; ctl->accepted = 0;
        }
        __syncthreads();
        if (!ctl->go) break;
        while (ctl->actual <= 0 && ctl->nfev < max_nfev) {
            __syncthreads();                                       // everybody has evaluated the loop condition
            BA_TICK(BA_PH_SETUP);
            ba_solve_tr(S, n);
            BA_TICK(BA_PH_TR_SOLVE);
            if (tid == 0) {
                for (int i = 0; i < nf; ++i) S.x_new[i] = S.x[i];
                for (int j = 0; j < n; ++j) { const int idx = 1 + 7 * (j / 6) + 1 + j % 6; S.x_new[idx] = S.x[idx] + S.p[j]; }
            }
            __syncthreads();
            for (int c = tid; c < C; c += nt) ba_pose_from_x(S.x_new, c, S.Rt_new + 12 * c);
            __syncthreads();
            ba_cost_pass(P, Q, S, S.Rt_new, false, scratch, v3);
            ba_grid_sum3(P, S, slot, v3, tot); slot ^= 1;
            BA_TICK(BA_PH_TRIAL);
            if (tid == 0) {
                ctl->nfev += 1;
                const double cost_new = tot[0];
                const bool finite = tot[1] == 0.0;
                const double step_h_norm = ctl->step_norm;
                if (!finite) { ctl->Delta = 0.25 * step_h_norm; }
                else {
                    const double actual = ctl->cost - cost_new, pred = ctl->pred;
                    ctl->actual = actual; ctl->cost_new = cost_new;
                    double ratio;                                  // update_tr_radius
                    if (pred > 0) ratio = actual / pred;
                    else if (pred == 0 && actual == 0) ratio = 1;
                    else ratio = 0;
                    double Delta_new = ctl->Delta;
                    if (ratio < 0.25) Delta_new = 0.25 * step_h_norm;
                    else if (ratio > 0.75 && step_h_norm > 0.95 * ctl->Delta) Delta_new = ctl->Delta * 2.0;
                    const double x_norm = ba_norm2_serial(S.x, nf);   // check_termination
                    const bool ftol_ok = actual < Q.ftol * ctl->cost && ratio > 0.25;
                    const bool xtol_ok = step_h_norm < Q.xtol * (Q.xtol + x_norm);
                    if (ftol_ok && xtol_ok) ctl->termination = 4;
                    else if (ftol_ok) ctl->termination = 2;
                    else if (xtol_ok) ctl->termination = 3;
                    if (ctl->termination == -99) { ctl->alpha *= ctl->Delta / Delta_new; ctl->Delta = Delta_new; }
                }
            }
            __syncthreads();
            if (ctl->termination != -99) break;
        }
        if (ctl->actual > 0) {                                     // accept: x = x_new, new Jacobian
            __syncthreads();
            for (int i = tid; i < nf; i += nt) S.x[i] = S.x_new[i];
            for (int e = tid; e < C * 12; e += nt) S.Rt[e] = S.Rt_new[e];
            __syncthreads();
            BA_TICK(BA_PH_SETUP);
            ba_make_columns(P, Q, S);
            ba_polish_accumulate(P, Q, S);
            ba_reduce_system(P, Q, S, npair + n + 2);
            ba_load_system(P, S, n);
            BA_TICK(BA_PH_LINEARIZE);
            ba_tridiagonalise(S, n);
            BA_TICK(BA_PH_TRIDIAG);
            if (tid == 0) { ctl->cost = ba_fresh(P.fin)[npair + n]; ctl->finite = ba_fresh(P.fin)[npair + n + 1] == 0.0; ctl->njev += 1; }
        }
        if (tid == 0) ctl->iteration += 1;
        __syncthreads();
    }
    if (tid == 0) {
        double gn = 0.0;
        for (int i = 0; i < n; ++i) gn = fmax(gn, fabs(S.g[i]));
        ctl->g_norm = gn;
        if (ctl->termination == -99) ctl->termination = 0;
    }
    __syncthreads();

    // ---- result (helpers.py:290) -----------------------------------------------------------------------------------
    if (ctl->cta == 0) {
        for (int c = tid; c < C; c += nt) {
            double Rt[12];
            ba_pose_from_x(S.x, c, Rt);
            for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) P.R[9 * c + 3 * i + j] = Rt[4 * i + j]; P.t[3 * c + i] = Rt[4 * i + 3]; }
        }
        if (tid == 0 && P.report) {
            mocap_ba_report r;
            r.cost_initial = ctl->cost_initial; r.cost_final = ctl->cost; r.optimality = ctl->g_norm;
            r.n_iterations = ctl->iteration; r.n_fev = ctl->nfev; r.status = ctl->termination; r.n_residuals = ctl->n_valid;
            r.prefit_cost_initial = ctl->pf_cost0; r.prefit_cost_final = ctl->pf_cost1; r.prefit_iterations = ctl->pf_it;
            r.n_launches = 1; r.n_tr_solves = ctl->tr_calls; r.n_tr_newton = ctl->tr_its;
            const unsigned long long t_end = ba_clock();
            ctl->prof[BA_PH_SETUP] += t_end - ctl->t_last;
            for (int k = 0; k < 8; ++k) r.phase_ms[k] = (float)((double)ctl->prof[k] * 1e-6);
            *P.report = r;
        }
    }
}
BA_DEV void ba_solve_body(const BAParams& P, unsigned char* smem) { ba_solve_body(P, P, smem); }

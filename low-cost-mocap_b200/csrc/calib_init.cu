// SURVEY.md section 8(f) "next" #4: cold-start extrinsics from 2D tracks, the caller of S3/S4.
//
// Replaces the body of calculate_camera_pose (reference computer_code/api/index.py:229-270): for every
// adjacent camera pair a fundamental matrix from the common observations, E = K1^T F K0
// (cv.sfm.essentialFromFundamental with the intrinsics of cameras 0 and 1, index.py:247), the four
// (R, t) of cv.sfm.motionFromEssential, the cheirality vote with the reference's own (odd) counting rule
// (index.py:253-262), and the pose chain (index.py:264-265).  bundle_adjustment then refines the chain.
//
// The reference estimates F with cv.findFundamentalMat(FM_RANSAC, 1 px, 0.99999), whose generator starts from a
// fixed state (repeatable, but its sample sequence is not replayed here) and which returns a 7-point minimal-sample
// model.  This file's estimator: normalised 8-point over all common observations -- or, for the robust method
// (calib_ransac.cu), over the inliers of a RANSAC model -- two rounds of re-estimation on the Sampson inliers, rank
// 2 enforced.  Parity is therefore defined downstream of F (SURVEY.md section 8(c)): given the same F the
// chosen (R, t) must be the reference's, and end to end the adjusted rig must be at least as good.
//
// GPU: the 9x9 normal matrix of the epipolar constraint and the Sampson residuals are reductions over
// the correspondences (k_epipolar_normal), the cheirality vote triangulates every correspondence under
// all four candidate motions (k_cheirality).  Host: 9x9 / 3x3 eigen problems.
#include <vector>
#include <math.h>
#include "common.cuh"
#include "geom.cuh"
#include "trf_core.h"
#include "calib_pose.h"

// normal matrix (upper triangle, 45 doubles) of rows a = kron(x2h, x1h) over the inlier correspondences
__global__ void __launch_bounds__(256)
k_epipolar_normal(const double* __restrict__ p1, const double* __restrict__ p2, const uint8_t* __restrict__ inl, int n,
                  const double* __restrict__ T1, const double* __restrict__ T2, double* __restrict__ out45) {
    __shared__ double acc[45];
    for (int i = threadIdx.x; i < 45; i += blockDim.x) acc[i] = 0.0;
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (!inl[i]) continue;
        const double x1 = T1[0] * p1[2 * i] + T1[1], y1 = T1[0] * p1[2 * i + 1] + T1[2];     // isotropic normalisation
        const double x2 = T2[0] * p2[2 * i] + T2[1], y2 = T2[0] * p2[2 * i + 1] + T2[2];
        const double a[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
        int k = 0;
        for (int r = 0; r < 9; ++r)
            for (int c = r; c < 9; ++c) atomicAdd(&acc[k++], a[r] * a[c]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 45; i += blockDim.x) if (acc[i] != 0.0) atomicAdd(&out45[i], acc[i]);
}

// Sampson distance^2 of every correspondence under F (row-major, x2^T F x1 = 0); writes the inlier mask
__global__ void __launch_bounds__(256)
k_sampson_inliers(const double* __restrict__ p1, const double* __restrict__ p2, int n, const double* __restrict__ F,
                  double thresh2, uint8_t* __restrict__ inl, int* __restrict__ n_inl) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x1 = p1[2 * i], y1 = p1[2 * i + 1], x2 = p2[2 * i], y2 = p2[2 * i + 1];
    const double l0 = F[0] * x1 + F[1] * y1 + F[2], l1 = F[3] * x1 + F[4] * y1 + F[5], l2 = F[6] * x1 + F[7] * y1 + F[8];
    const double m0 = F[0] * x2 + F[3] * y2 + F[6], m1 = F[1] * x2 + F[4] * y2 + F[7];
    const double e = x2 * l0 + y2 * l1 + l2;
    const double d2 = e * e / (l0 * l0 + l1 * l1 + m0 * m0 + m1 * m1);
    const uint8_t ok = d2 <= thresh2 ? 1 : 0;
    inl[i] = ok;
    if (ok) atomicAdd(n_inl, 1);
}

// index.py:253-262: for candidate q, triangulate every correspondence with projection matrices
// P1 (previous camera) and P2[q]; count X_z > 0 plus (R_q^T X)_z > 0.
__global__ void __launch_bounds__(256)
k_cheirality(const double* __restrict__ p1, const double* __restrict__ p2, int n, const double* __restrict__ P1,
             const double* __restrict__ P2 /*[4][12]*/, const double* __restrict__ Rq /*[4][9]*/, int* __restrict__ counts) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 4 * n) return;
    const int q = idx / n, i = idx - q * n;
    Sym4 B;
    sym4_zero(B);
    dlt_add_view(B, P1, p1[2 * i], p1[2 * i + 1]);
    dlt_add_view(B, P2 + 12 * q, p2[2 * i], p2[2 * i + 1]);
    double X[3];
    dlt_solve(B, X);
    const double* R = Rq + 9 * q;
    const double zc = R[2] * X[0] + R[5] * X[1] + R[8] * X[2];       // (R^T X)_z
    const int c = (X[2] > 0 ? 1 : 0) + (zc > 0 ? 1 : 0);
    if (c) atomicAdd(&counts[q], c);
}

using namespace calib_pose;

// One adjacent pair.  p1/p2: device [n][2] common observations.  F_in (host, 9) may be given (then no
// estimation); F_out receives the matrix used.  prev_R/prev_t: accumulated pose of the first camera.
// init_inl (host, n; NULL = all points) is the set the first 8-point fit uses -- a set of fewer than 8 falls back to
// all points; thr2 is the squared Sampson threshold of the re-selection rounds; inl_out (host, n; may be NULL)
// receives the final inlier set of the rounds.
static int pair_motion(mocap_ctx* ctx, const double* d_p1, const double* d_p2, uint8_t* d_inl, double* d_work, int n,
                       const double* F_in, double* F_out, const double* K0, const double* K1, const double* prev_R,
                       const double* prev_t, double* R_rel, double* t_rel, int* votes, const uint8_t* init_inl,
                       double thr2, uint8_t* inl_out) {
    cudaStream_t s = ctx->stream;
    double F[9];
    if (F_in) memcpy(F, F_in, sizeof(F));
    else {
        // Hartley normalisation from the host copy of the points
        std::vector<double> h1(2 * (size_t)n), h2(2 * (size_t)n);
        CUDA_TRY(ctx, cudaMemcpyAsync(h1.data(), d_p1, h1.size() * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(h2.data(), d_p2, h2.size() * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        std::vector<uint8_t> inl(n, 1);
        if (init_inl) {
            int m0 = 0;
            for (int i = 0; i < n; ++i) m0 += init_inl[i] ? 1 : 0;
            if (m0 >= 8) for (int i = 0; i < n; ++i) inl[i] = init_inl[i] ? 1 : 0;
        }
        for (int round = 0; round < 3; ++round) {
            double T1[3], T2[3];
            for (int side = 0; side < 2; ++side) {
                const std::vector<double>& h = side ? h2 : h1;
                double cx = 0, cy = 0; int m = 0;
                for (int i = 0; i < n; ++i) if (inl[i]) { cx += h[2 * i]; cy += h[2 * i + 1]; ++m; }
                if (m < 8) return mocap_fail(ctx, MOCAP_EINVAL, "calibration: fewer than 8 common observations for a camera pair");
                cx /= m; cy /= m;
                double md = 0;
                for (int i = 0; i < n; ++i) if (inl[i]) md += sqrt((h[2 * i] - cx) * (h[2 * i] - cx) + (h[2 * i + 1] - cy) * (h[2 * i + 1] - cy));
                md /= m;
                const double sc = md > 0 ? sqrt(2.0) / md : 1.0;
                double* T = side ? T2 : T1;
                T[0] = sc; T[1] = -sc * cx; T[2] = -sc * cy;
            }
            double* d_T = d_work;                 // [6] T1,T2 ; [45] normal ; [9] F
            double hT[6] = {T1[0], T1[1], T1[2], T2[0], T2[1], T2[2]};
            CUDA_TRY(ctx, cudaMemcpyAsync(d_T, hT, sizeof(hT), cudaMemcpyHostToDevice, s));
            CUDA_TRY(ctx, cudaMemcpyAsync(d_inl, inl.data(), n, cudaMemcpyHostToDevice, s));
            CUDA_TRY(ctx, cudaMemsetAsync(d_work + 8, 0, 45 * 8, s));
            k_epipolar_normal<<<(n + 255) / 256 < 64 ? (n + 255) / 256 : 64, 256, 0, s>>>(d_p1, d_p2, d_inl, n, d_T, d_T + 3, d_work + 8);
            CUDA_TRY(ctx, cudaGetLastError());
            ctx->launches += 1;
            double up[45];
            CUDA_TRY(ctx, cudaMemcpyAsync(up, d_work + 8, sizeof(up), cudaMemcpyDeviceToHost, s));
            CUDA_TRY(ctx, cudaStreamSynchronize(s));
            std::vector<double> A(81), lam;
            int k = 0;
            for (int r = 0; r < 9; ++r) for (int c = r; c < 9; ++c) { A[9 * r + c] = up[k]; A[9 * c + r] = up[k]; ++k; }
            if (!trf::sym_eig(9, A, lam)) return mocap_fail(ctx, MOCAP_EINVAL, "calibration: eigen-decomposition failed");
            int best = 0;
            for (int i = 1; i < 9; ++i) if (lam[i] < lam[best]) best = i;
            double Fn[9];
            for (int i = 0; i < 9; ++i) Fn[i] = A[9 * i + best];
            // rank 2
            double U[9], sv[3], V[9];
            svd3(Fn, U, sv, V);
            double Fr[9];
            for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Fr[3 * i + j] = U[3 * i] * sv[0] * V[3 * j] + U[3 * i + 1] * sv[1] * V[3 * j + 1];
            // de-normalise: F = T2^T Fr T1 with T = [[s,0,tx],[0,s,ty],[0,0,1]]
            const double M1[9] = {T1[0], 0, T1[1], 0, T1[0], T1[2], 0, 0, 1}, M2t[9] = {T2[0], 0, 0, 0, T2[0], 0, T2[1], T2[2], 1};
            double tmp[9];
            mat3mul(M2t, Fr, tmp); mat3mul(tmp, M1, F);
            double nf = 0; for (int i = 0; i < 9; ++i) nf += F[i] * F[i];
            nf = sqrt(nf); if (nf > 0) for (int i = 0; i < 9; ++i) F[i] /= nf;
            fix_sign(F);
            if (round == 2) break;
            // Sampson inliers at thr2 (1 px: the reference's RANSAC threshold, index.py:246)
            int* d_cnt = reinterpret_cast<int*>(d_work + 64);
            CUDA_TRY(ctx, cudaMemcpyAsync(d_work + 54, F, sizeof(F), cudaMemcpyHostToDevice, s));
            CUDA_TRY(ctx, cudaMemsetAsync(d_cnt, 0, sizeof(int), s));
            k_sampson_inliers<<<(n + 255) / 256, 256, 0, s>>>(d_p1, d_p2, n, d_work + 54, thr2, d_inl, d_cnt);
            CUDA_TRY(ctx, cudaGetLastError());
            ctx->launches += 1;
            int cnt = 0;
            CUDA_TRY(ctx, cudaMemcpyAsync(&cnt, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, s));
            CUDA_TRY(ctx, cudaMemcpyAsync(inl.data(), d_inl, n, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(ctx, cudaStreamSynchronize(s));
            if (cnt < 8 || cnt == n) { if (cnt < 8) std::fill(inl.begin(), inl.end(), 1); if (cnt == n && round > 0) break; }
        }
        if (inl_out) memcpy(inl_out, inl.data(), n);
    }
    if (F_out) memcpy(F_out, F, sizeof(F));
    // E = K1^T F K0 (libmv EssentialFromFundamental(F, K1=first arg, K2=second arg) = K2^T F K1; index.py:247 passes K[0], K[1])
    double K1t[9], tmp[9], E[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) K1t[3 * i + j] = K1[3 * j + i];
    mat3mul(K1t, F, tmp); mat3mul(tmp, K0, E);
    double Rs[4][9], ts[4][3];
    motion_from_essential(E, Rs, ts);
    // cheirality vote (index.py:253-262): poses [previous camera, candidate], K of view 0 and view 1
    double P1[12], P2[4][12], Rq[4][9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) {
        double a = 0;
        for (int k = 0; k < 3; ++k) a += K0[3 * i + k] * (j < 3 ? prev_R[3 * k + j] : prev_t[k]);
        P1[4 * i + j] = a;
    }
    for (int q = 0; q < 4; ++q) {
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) {
            double a = 0;
            for (int k = 0; k < 3; ++k) a += K1[3 * i + k] * (j < 3 ? Rs[q][3 * k + j] : ts[q][k]);
            P2[q][4 * i + j] = a;
        }
        memcpy(Rq[q], Rs[q], sizeof(Rq[q]));
    }
    double* d_P = d_work;                         // [12] P1, [48] P2, [36] Rq, counts after
    int* d_counts = reinterpret_cast<int*>(d_work + 100);
    CUDA_TRY(ctx, cudaMemcpyAsync(d_P, P1, sizeof(P1), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_P + 12, P2, sizeof(P2), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_P + 60, Rq, sizeof(Rq), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemsetAsync(d_counts, 0, 4 * sizeof(int), s));
    k_cheirality<<<(4 * n + 255) / 256, 256, 0, s>>>(d_p1, d_p2, n, d_P, d_P + 12, d_P + 60, d_counts);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    int counts[4];
    CUDA_TRY(ctx, cudaMemcpyAsync(counts, d_counts, sizeof(counts), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    int best = -1, best_count = 0;
    for (int q = 0; q < 4; ++q) if (counts[q] > best_count) { best_count = counts[q]; best = q; }     // strict >, first maximum
    if (best < 0) return mocap_fail(ctx, MOCAP_EINVAL, "calibration: no candidate motion puts a point in front of the cameras");
    memcpy(R_rel, Rs[best], 9 * sizeof(double));
    memcpy(t_rel, ts[best], 3 * sizeof(double));
    if (votes) memcpy(votes, counts, sizeof(counts));
    return MOCAP_OK;
}

// The pose chain of index.py:235-265 over all adjacent pairs (see pair_motion).  init_inl (host; may be NULL) holds
// each pair's initial fit set over its common observations in frame order, pair after pair; inl_out (host,
// [n_points][C-1]; may be NULL) receives each pair's final inlier set, 0 where the frame is not common to the pair.
int calibrate_chain(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points, const double* F_given,
                    const uint8_t* init_inl, double thr2, double* R, double* t, double* F_used, int* votes, uint8_t* inl_out) {
    const int C = ctx->cfg.n_cam;
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    const size_t n = (size_t)n_points;
    int st = ensure_scratch(ctx, n * 2 * 8 * 2 + n + 4096);
    if (st) return st;
    unsigned char* base = static_cast<unsigned char*>(ctx->d_scratch);
    double* d_p1 = reinterpret_cast<double*>(base);
    double* d_p2 = d_p1 + 2 * n;
    double* d_work = d_p2 + 2 * n;                 // 256 doubles of small device scratch
    uint8_t* d_inl = reinterpret_cast<uint8_t*>(d_work + 256);
    // camera 0: (I, 0)   (index.py:235-238)
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    t[0] = t[1] = t[2] = 0.0;
    const double* K0 = ctx->h_tables.Kmat[0];
    const double* K1 = ctx->h_tables.Kmat[C > 1 ? 1 : 0];
    std::vector<double> h1, h2;
    std::vector<uint8_t> pair_inl(inl_out ? n : 0);
    size_t init_off = 0;
    if (inl_out) memset(inl_out, 0, n * (C - 1));
    for (int c = 0; c + 1 < C; ++c) {
        h1.clear(); h2.clear();
        for (int f = 0; f < n_points; ++f)
            if (mask[(size_t)f * C + c] && mask[(size_t)f * C + c + 1]) {      // index.py:242
                // the reference casts the common observations to float32 (index.py:243-244)
                h1.push_back((double)(float)obs[((size_t)f * C + c) * 2]); h1.push_back((double)(float)obs[((size_t)f * C + c) * 2 + 1]);
                h2.push_back((double)(float)obs[((size_t)f * C + c + 1) * 2]); h2.push_back((double)(float)obs[((size_t)f * C + c + 1) * 2 + 1]);
            }
        const int m = (int)(h1.size() / 2);
        if (m < 8) return mocap_fail(ctx, MOCAP_EINVAL, "calibration: cameras %d and %d share only %d observations", c, c + 1, m);
        CUDA_TRY(ctx, cudaMemcpyAsync(d_p1, h1.data(), h1.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_p2, h2.data(), h2.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
        double R_rel[9], t_rel[3];
        st = pair_motion(ctx, d_p1, d_p2, d_inl, d_work, m, F_given ? F_given + 9 * c : nullptr, F_used ? F_used + 9 * c : nullptr, K0, K1,
                         R + 9 * c, t + 3 * c, R_rel, t_rel, votes ? votes + 4 * c : nullptr, init_inl ? init_inl + init_off : nullptr,
                         thr2, inl_out ? pair_inl.data() : nullptr);
        if (st) return st;
        init_off += (size_t)m;
        if (inl_out)
            for (int f = 0, k = 0; f < n_points; ++f)
                if (mask[(size_t)f * C + c] && mask[(size_t)f * C + c + 1]) inl_out[(size_t)f * (C - 1) + c] = pair_inl[k++];
        // index.py:264-265: R = R_rel @ R_prev ; t = t_prev + R_prev @ t_rel
        mat3mul(R_rel, R + 9 * c, R + 9 * (c + 1));
        for (int i = 0; i < 3; ++i) {
            double a = t[3 * c + i];
            for (int k = 0; k < 3; ++k) a += R[9 * c + 3 * i + k] * t_rel[k];
            t[3 * (c + 1) + i] = a;
        }
    }
    return MOCAP_OK;
}

extern "C" int mocap_calibrate_init_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                         const double* F_given, double* R, double* t, double* F_used, int* votes) {
    if (!ctx) return MOCAP_EINVAL;
    const int C = ctx->cfg.n_cam;
    if (!obs || !mask || !R || !t || n_points < 8 || C < 2) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_calibrate_init_host: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    return calibrate_chain(ctx, obs, mask, n_points, F_given, nullptr, 1.0, R, t, F_used, votes, nullptr);
}

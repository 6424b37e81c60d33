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
// GPU: the 8-point re-fits of all pairs at once (calib_graph.cu's fit_pairs / select_pairs: the 9x9 normal matrices and
// the Sampson selections, summed in a fixed order), and per pair the cheirality vote, which triangulates every
// correspondence under all four candidate motions (k_cheirality).  Host: 9x9 / 3x3 eigen problems.
#include <vector>
#include <math.h>
#include "common.cuh"
#include "geom.cuh"
#include "calib_pose.h"

// index.py:253-262: for candidate q, triangulate every correspondence pts [n] {x1, y1, x2, y2} with projection matrices
// P1 (previous camera) and P2[q]; count X_z > 0 plus (R_q^T X)_z > 0.
__global__ void __launch_bounds__(256)
k_cheirality(const float4* __restrict__ pts, int n, const double* __restrict__ P1, const double* __restrict__ P2 /*[4][12]*/,
             const double* __restrict__ Rq /*[4][9]*/, int* __restrict__ counts) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 4 * n) return;
    const int q = idx / n, i = idx - q * n;
    const float4 v = pts[i];
    Sym4 B;
    sym4_zero(B);
    dlt_add_view(B, P1, v.x, v.y);
    dlt_add_view(B, P2 + 12 * q, v.z, v.w);
    double X[3];
    dlt_solve(B, X);
    const double* R = Rq + 9 * q;
    const double zc = R[2] * X[0] + R[5] * X[1] + R[8] * X[2];       // (R^T X)_z
    const int c = (X[2] > 0 ? 1 : 0) + (zc > 0 ? 1 : 0);
    if (c) atomicAdd(&counts[q], c);
}

using namespace calib_pose;

// The pose chain of index.py:235-265 over the adjacent table.  F_given (host, [C-1][9]; may be NULL) skips the fits.
int calibrate_chain(mocap_ctx* ctx, const PairTable& tab, const uint8_t* mask, int n_points, const double* F_given,
                    const uint8_t* init_inl, double thr2, double* R, double* t, double* F_used, int* votes, uint8_t* inl_out) {
    const int C = ctx->cfg.n_cam, P = tab.pairs();
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    PairDev d;
    double* d_work;
    int st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
        d.take(L, tab);
        d_work = L.take<double>(128);                // the vote's P1 [12], P2 [4][12], Rq [4][9], counts [4]
    });
    if (st) return st;
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d.pts, tab.pts.data(), tab.pts.size() * sizeof(float4), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d.off, tab.off.data(), (P + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
    std::vector<double> F(9 * (size_t)P);
    if (F_given) memcpy(F.data(), F_given, F.size() * 8);
    else {
        // Per pair: the first fit on init_inl if it holds at least 8 points (else all), three fits in all; after each
        // of the first two the Sampson selection at thr2 (1 px: the reference's RANSAC threshold, index.py:246) is the
        // next fit set, all points if it holds fewer than 8.  A pair whose selection after the second fit holds every
        // point stops there with its second F.
        std::vector<uint8_t> inl(tab.pts.size(), 1), sel(inl.size()), ok(P), live(P, 1);
        std::vector<double> Ffit(F.size());
        for (int p = 0; p < P && init_inl; ++p) {
            int k = 0;
            for (int i = tab.off[p]; i < tab.off[p + 1]; ++i) k += init_inl[i] ? 1 : 0;
            if (k >= 8) for (int i = tab.off[p]; i < tab.off[p + 1]; ++i) inl[i] = init_inl[i] ? 1 : 0;
        }
        for (int round = 0; round < 3; ++round) {
            if ((st = fit_pairs(ctx, tab, d, inl.data(), Ffit.data(), ok.data()))) return st;
            for (int p = 0; p < P; ++p) {
                if (live[p] && !ok[p]) return mocap_fail(ctx, MOCAP_EINVAL, "calibration: eigen-decomposition failed");
                if (live[p]) memcpy(&F[9 * p], &Ffit[9 * p], 9 * 8);
            }
            if (round == 2) break;
            if ((st = select_pairs(ctx, tab, d, F.data(), thr2, sel.data()))) return st;
            int n_live = 0;
            for (int p = 0; p < P; ++p) {
                if (!live[p]) continue;
                int k = 0;
                for (int i = tab.off[p]; i < tab.off[p + 1]; ++i) k += sel[i];
                for (int i = tab.off[p]; i < tab.off[p + 1]; ++i) inl[i] = k < 8 ? 1 : sel[i];
                live[p] = !(k == tab.count(p) && round > 0);
                n_live += live[p];
            }
            if (!n_live) break;
        }
        if (inl_out) scatter_pairs(tab, mask, n_points, C, inl.data(), inl_out);
    }
    if (F_used) memcpy(F_used, F.data(), F.size() * 8);
    // camera 0: (I, 0)   (index.py:235-238)
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    t[0] = t[1] = t[2] = 0.0;
    const double* K0 = ctx->h_tables.Kmat[0];
    const double* K1 = ctx->h_tables.Kmat[1];
    for (int c = 0; c < P; ++c) {
        const double *prev_R = R + 9 * c, *prev_t = t + 3 * c;
        // E = K1^T F K0 (libmv EssentialFromFundamental(F, K1=first arg, K2=second arg) = K2^T F K1; index.py:247 passes K[0], K[1])
        double K1t[9], tmp[9], E[9];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) K1t[3 * i + j] = K1[3 * j + i];
        mat3mul(K1t, &F[9 * c], tmp); mat3mul(tmp, K0, E);
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
        int* d_counts = reinterpret_cast<int*>(d_work + 100);
        CUDA_TRY(ctx, cudaMemcpyAsync(d_work, P1, sizeof(P1), cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_work + 12, P2, sizeof(P2), cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_work + 60, Rq, sizeof(Rq), cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemsetAsync(d_counts, 0, 4 * sizeof(int), s));
        const int n = tab.count(c);
        k_cheirality<<<(4 * n + 255) / 256, 256, 0, s>>>(d.pts + tab.off[c], n, d_work, d_work + 12, d_work + 60, d_counts);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        int counts[4];
        CUDA_TRY(ctx, cudaMemcpyAsync(counts, d_counts, sizeof(counts), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        int best = -1, best_count = 0;
        for (int q = 0; q < 4; ++q) if (counts[q] > best_count) { best_count = counts[q]; best = q; }     // strict >, first maximum
        if (best < 0) return mocap_fail(ctx, MOCAP_EINVAL, "calibration: no candidate motion puts a point in front of the cameras");
        if (votes) memcpy(votes + 4 * c, counts, sizeof(counts));
        // index.py:264-265: R = R_rel @ R_prev ; t = t_prev + R_prev @ t_rel
        mat3mul(Rs[best], prev_R, R + 9 * (c + 1));
        for (int i = 0; i < 3; ++i) {
            double a = prev_t[i];
            for (int k = 0; k < 3; ++k) a += prev_R[3 * i + k] * ts[best][k];
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
    PairTable tab;
    const int st = adjacent_pairs(ctx, obs, mask, n_points, "calibration", tab);
    if (st) return st;
    return calibrate_chain(ctx, tab, mask, n_points, F_given, nullptr, 1.0, R, t, F_used, votes, nullptr);
}

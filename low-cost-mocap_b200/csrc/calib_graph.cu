// Pose-graph cold start (SURVEY.md section 8(f) "next" #4, second form): every camera placed from every overlapping
// pair, instead of the chain of adjacent pairs of calib_init.cu.
//
// The reference's calculate-camera-pose handler (computer_code/api/index.py:229-270) places camera c+1 from the pair
// (c, c+1) alone, votes on the four motions of E with camera c's accumulated pose on one side and the relative
// candidate on the other (index.py:253-262), and chains t_{c+1} = t_c + R_c t_rel with every baseline taken as 1
// (index.py:264-265).  One bad pair then breaks every camera after it, the vote can pick a twisted motion however good
// F is, and from camera 2 on the centres are wrong in direction and scale.  This file departs from it deliberately:
//   1. pair table      every pair (a < b) with at least min_common common observations
//   2. RANSAC F        calib_ransac.cu's three kernels over the pair table, one launch each
//   3. re-fit          normalised 8-point fits and Sampson re-selection for all pairs at once
//                      (k_epipolar_normal_pairs, k_sampson_pairs); the 9x9 eigen problems on the host
//   4. cheirality      E = K_b^T F K_a with each pair's own intrinsics, the four candidates judged in the pair's own
//                      frame (k_pair_cheirality); a pair is dropped with fewer than min_inliers points in front of both
//                      cameras or a median triangulation angle under min_angle_deg
//   5. rotations       weighted chordal averaging with Cauchy re-weighting on the host (calib_graph.cuh); pairs off by
//                      more than rot_outlier_deg are dropped
//   6. translations    with the rotations known, the linear bearing constraints of every track, the points eliminated
//                      per track (k_translation_normal, k_translation_reduce: fixed-order sums, no floating-point
//                      atomics), smallest eigenvector on the host, irls_rounds rounds of Cauchy weights at 4 px
//                      (k_translation_residuals)
// Output: poses in camera 0's frame with |t_1| = 1 (the chain's gauge), a per-view support mask and a pair report.
// Everything the host decides from is copied back once per stage; the number of launches does not grow with the number
// of pairs.  Two calls with the same inputs give the same bits.
#include <vector>
#include <algorithm>
#include <math.h>
#include "common.cuh"
#include "calib_graph.cuh"

#define CG_THREADS      256
#define CG_TILE         16         // tracks per shared-memory tile of k_translation_normal (16 x 16 views = 256 threads)
#define CG_MAX_ENTRIES  1176       // upper triangle of the 48 x 48 reduced system
#define CG_ENT_PER_THR  ((CG_MAX_ENTRIES + CG_THREADS - 1) / CG_THREADS)
#define CG_SCALE_PX     4.0        // Cauchy scale of the translation re-weighting
#define CG_CAND         36         // per (pair, candidate): Pa 12, Pb 12, R 9, t 3

struct CgCams {
    double R[CG_MAX_CAM][9];
    double Kinv[CG_MAX_CAM][9];
    double f[CG_MAX_CAM];
};

// Normal matrix (upper triangle, 45 doubles) of rows kron(x_b, x_a) over each pair's fit set, one CTA per pair, summed
// in a fixed order: per thread over its strided points, per warp by shuffles, then over the warps.
__global__ void __launch_bounds__(CG_THREADS)
k_epipolar_normal_pairs(const float4* __restrict__ pts, const int* __restrict__ off, const uint8_t* __restrict__ inl,
                        const double* __restrict__ T /*[P][6]*/, double* __restrict__ out45 /*[P][45]*/) {
    __shared__ double part[CG_THREADS / 32][45];
    const int p = blockIdx.x, o = off[p], m = off[p + 1] - o;
    const double* Tp = T + 6 * p;
    double acc[45];
#pragma unroll
    for (int k = 0; k < 45; ++k) acc[k] = 0.0;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        if (!inl[o + i]) continue;
        const float4 v = pts[o + i];
        const double x1 = Tp[0] * (double)v.x + Tp[1], y1 = Tp[0] * (double)v.y + Tp[2];
        const double x2 = Tp[3] * (double)v.z + Tp[4], y2 = Tp[3] * (double)v.w + Tp[5];
        const double a[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
        int k = 0;
#pragma unroll
        for (int r = 0; r < 9; ++r)
#pragma unroll
            for (int c = r; c < 9; ++c) acc[k++] += a[r] * a[c];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 45; ++k) {
        double x = acc[k];
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) x += __shfl_down_sync(0xffffffffu, x, s);
        if (lane == 0) part[warp][k] = x;
    }
    __syncthreads();
    if (threadIdx.x < 45) {
        double x = 0.0;
        for (int w = 0; w < CG_THREADS / 32; ++w) x += part[w][threadIdx.x];
        out45[45 * p + threadIdx.x] = x;
    }
}

// Sampson distance^2 of every pair's correspondences under its F [P][9] (x_b^T F x_a = 0) against thr2 -> mask
__global__ void __launch_bounds__(CG_THREADS)
k_sampson_pairs(const float4* __restrict__ pts, const int* __restrict__ off, const double* __restrict__ Fp, double thr2,
                uint8_t* __restrict__ inl) {
    const int p = blockIdx.y, o = off[p], m = off[p + 1] - o;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const double* F = Fp + 9 * p;
    const float4 v = pts[o + i];
    const double x1 = v.x, y1 = v.y, x2 = v.z, y2 = v.w;
    const double l0 = F[0] * x1 + F[1] * y1 + F[2], l1 = F[3] * x1 + F[4] * y1 + F[5], l2 = F[6] * x1 + F[7] * y1 + F[8];
    const double m0 = F[0] * x2 + F[3] * y2 + F[6], m1 = F[1] * x2 + F[4] * y2 + F[7];
    const double e = x2 * l0 + y2 * l1 + l2;
    const double d2 = e * e / (l0 * l0 + l1 * l1 + m0 * m0 + m1 * m1);
    inl[o + i] = d2 <= thr2 ? 1 : 0;
}

// One thread per (pair, correspondence, candidate): cheirality in the pair's own frame (calib_graph.cuh).  counts
// [P][4] (integer atomics: the same sums in any order); ang [total][4] the triangulation angle in degrees of each
// candidate, -1 where the correspondence is not an inlier or not in front of both cameras.
__global__ void __launch_bounds__(CG_THREADS)
k_pair_cheirality(const float4* __restrict__ pts, const int* __restrict__ off, const uint8_t* __restrict__ inl,
                  const double* __restrict__ cand /*[P][4][CG_CAND]*/, int* __restrict__ counts, double* __restrict__ ang) {
    const int p = blockIdx.y, o = off[p], m = off[p + 1] - o;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = idx >> 2, q = idx & 3;
    if (i >= m) return;
    double a = -1.0;
    if (inl[o + i]) {
        const double* c = cand + (size_t)(4 * p + q) * CG_CAND;
        const float4 v = pts[o + i];
        bool front;
        const double ang_deg = cg_cheirality_point(c, c + 12, c + 24, c + 33, v.x, v.y, v.z, v.w, front);
        if (front) { a = ang_deg; atomicAdd(&counts[4 * p + q], 1); }
    }
    ang[(size_t)(o + i) * 4 + q] = a;
}

// Reduced translation system.  CTA g takes the tracks [g * chunk, (g+1) * chunk) in tiles of CG_TILE: thread (track,
// view) forms its view's terms, one thread per track sums H_xx over the views in camera order and inverts it, then each
// thread adds its entries of the reduced system over the tile's tracks in order.  partial [gridDim.x][E], no atomics.
// w [n][C]: the view weights (0: out).
__global__ void __launch_bounds__(CG_THREADS)
k_translation_normal(const double* __restrict__ obs, const double* __restrict__ w, int n, int C, const CgCams* __restrict__ cams,
                     int chunk, double* __restrict__ partial) {
    __shared__ double sR[CG_MAX_CAM][9], sKi[CG_MAX_CAM][9];
    __shared__ double sN[CG_TILE][CG_MAX_CAM][9];
    __shared__ double sQ[CG_TILE][CG_MAX_CAM][6];
    __shared__ double sHi[CG_TILE][6];
    __shared__ unsigned sViews[CG_TILE];
    for (int i = threadIdx.x; i < C * 9; i += blockDim.x) { sR[i / 9][i % 9] = cams->R[i / 9][i % 9]; sKi[i / 9][i % 9] = cams->Kinv[i / 9][i % 9]; }
    const int n3 = 3 * C, E = n3 * (n3 + 1) / 2;
    int er[CG_ENT_PER_THR], ec[CG_ENT_PER_THR];
    double acc[CG_ENT_PER_THR];
#pragma unroll
    for (int k = 0; k < CG_ENT_PER_THR; ++k) {
        acc[k] = 0.0;
        const int e = threadIdx.x + k * CG_THREADS;
        er[k] = -1; ec[k] = -1;
        if (e < E) cg_entry_rc(n3, e, er[k], ec[k]);
    }
    const int f0 = blockIdx.x * chunk, f1 = min(n, f0 + chunk);
    const int tr = threadIdx.x / CG_MAX_CAM, vc = threadIdx.x % CG_MAX_CAM;
    for (int base = f0; base < f1; base += CG_TILE) {
        __syncthreads();
        const int f = base + tr;
        double RtQR[6];
        bool on = false;
        if (f < f1 && vc < C) {
            const double wv = w[(size_t)f * C + vc];
            if (wv > 0.0) {
                double x[3];
                cg_bearing(sKi[vc], obs[((size_t)f * C + vc) * 2], obs[((size_t)f * C + vc) * 2 + 1], x);
                cg_view_terms(x, wv, sR[vc], sQ[tr][vc], sN[tr][vc], RtQR);
                on = true;
            }
        }
        // H_xx in camera order: gather the RtQR of the track's views through shared memory (reuse sHi-sized slots)
        __shared__ double sH[CG_TILE][CG_MAX_CAM][6];
        __shared__ unsigned char sOn[CG_TILE][CG_MAX_CAM];
#pragma unroll
        for (int k = 0; k < 6; ++k) sH[tr][vc][k] = on ? RtQR[k] : 0.0;
        sOn[tr][vc] = on ? 1 : 0;
        __syncthreads();
        if (vc == 0) {
            double H[6] = {0, 0, 0, 0, 0, 0};
            unsigned views = 0u;
            int nv = 0;
            for (int c = 0; c < C; ++c)
                if (sOn[tr][c]) {
                    views |= 1u << c; ++nv;
#pragma unroll
                    for (int k = 0; k < 6; ++k) H[k] += sH[tr][c][k];
                }
            if (nv < 2 || !cg_inv_sym3(H, sHi[tr])) views = 0u;
            sViews[tr] = views;
        }
        __syncthreads();
        const int nt = min(CG_TILE, f1 - base);
#pragma unroll
        for (int k = 0; k < CG_ENT_PER_THR; ++k) {
            if (er[k] < 0) continue;
            const int ca = er[k] / 3, i = er[k] % 3, cb = ec[k] / 3, j = ec[k] % 3;
            for (int t = 0; t < nt; ++t) {
                const unsigned v = sViews[t];
                if (!((v >> ca) & 1u) || !((v >> cb) & 1u)) continue;
                double x = -cg_coupling(sN[t][ca], sHi[t], sN[t][cb], i, j);
                if (ca == cb) x += sQ[t][ca][cg_s6(i, j)];
                acc[k] += x;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < CG_ENT_PER_THR; ++k)
        if (er[k] >= 0) partial[(size_t)blockIdx.x * E + threadIdx.x + k * CG_THREADS] = acc[k];
}

// out[e] = sum over the CTAs in order of partial[g][e]
__global__ void __launch_bounds__(CG_THREADS)
k_translation_reduce(const double* __restrict__ partial, int G, int E, double* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    double x = 0.0;
    for (int g = 0; g < G; ++g) x += partial[(size_t)g * E + e];
    out[e] = x;
}

// One thread per (track, view): the track's point from its views weighted by w_old (the H_xx of k_translation_normal,
// summed in the same order), then the view's angular residual against it and its new Cauchy weight.  Views outside
// `init` keep weight 0; front: the point lies in front of the view's camera.
__global__ void __launch_bounds__(CG_THREADS)
k_translation_residuals(const double* __restrict__ obs, const uint8_t* __restrict__ init, const double* __restrict__ w_old, int n, int C,
                        const CgCams* __restrict__ cams, const double* __restrict__ t, double scale_px, double* __restrict__ w_new,
                        uint8_t* __restrict__ front) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * C) return;
    const int f = idx / C, cv = idx - f * C;
    double H[6] = {0, 0, 0, 0, 0, 0};
    double N[CG_MAX_CAM * 9];
    double xv[3] = {0, 0, 0};
    unsigned views = 0u;
    int nv = 0;
    for (int c = 0; c < C; ++c) {
        const double wv = w_old[(size_t)f * C + c];
        if (!(wv > 0.0)) continue;
        double x[3], Q[6], RtQR[6];
        cg_bearing(cams->Kinv[c], obs[((size_t)f * C + c) * 2], obs[((size_t)f * C + c) * 2 + 1], x);
        cg_view_terms(x, wv, cams->R[c], Q, N + 9 * c, RtQR);
#pragma unroll
        for (int k = 0; k < 6; ++k) H[k] += RtQR[k];
        views |= 1u << c; ++nv;
    }
    double Hi[6];
    double wn = 0.0;
    uint8_t fr = 0;
    if (init[idx] && nv >= 2 && cg_inv_sym3(H, Hi)) {
        double X[3];
        cg_track_point(Hi, N, t, views, C, X);
        cg_bearing(cams->Kinv[cv], obs[(size_t)idx * 2], obs[(size_t)idx * 2 + 1], xv);
        bool fb;
        const double r = cg_view_residual_px(xv, cams->R[cv], t + 3 * cv, X, cams->f[cv], fb);
        wn = cg_cauchy(r, scale_px);
        fr = fb ? 1 : 0;
    }
    w_new[idx] = wn;
    front[idx] = fr;
}

int fit_pairs(mocap_ctx* ctx, const PairTable& tab, const PairDev& d, const uint8_t* inl, double* F, uint8_t* ok) {
    const int P = tab.pairs();
    std::vector<double> hT(6 * (size_t)P), h45(45 * (size_t)P);
    for (int p = 0; p < P; ++p)
        calib_pose::hartley(reinterpret_cast<const float*>(&tab.pts[tab.off[p]]), tab.count(p), inl + tab.off[p], &hT[6 * p]);
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d.T, hT.data(), hT.size() * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d.inl, inl, tab.pts.size(), cudaMemcpyHostToDevice, s));
    k_epipolar_normal_pairs<<<P, CG_THREADS, 0, s>>>(d.pts, d.off, d.inl, d.T, d.n45);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaMemcpyAsync(h45.data(), d.n45, h45.size() * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    for (int p = 0; p < P; ++p) ok[p] = calib_pose::fit_from_normal(&h45[45 * p], &hT[6 * p], F + 9 * p) ? 1 : 0;
    return MOCAP_OK;
}

int select_pairs(mocap_ctx* ctx, const PairTable& tab, const PairDev& d, const double* F, double thr2, uint8_t* sel) {
    const int P = tab.pairs();
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d.F, F, (size_t)P * 9 * 8, cudaMemcpyHostToDevice, s));
    k_sampson_pairs<<<dim3((tab.max_count() + CG_THREADS - 1) / CG_THREADS, P), CG_THREADS, 0, s>>>(d.pts, d.off, d.F, thr2, d.inl);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaMemcpyAsync(sel, d.inl, tab.pts.size(), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return MOCAP_OK;
}

static void inv3(const double* K, double* Ki) {
    const double det = calib_pose::det3m(K);
    Ki[0] = (K[4] * K[8] - K[5] * K[7]) / det; Ki[1] = (K[2] * K[7] - K[1] * K[8]) / det; Ki[2] = (K[1] * K[5] - K[2] * K[4]) / det;
    Ki[3] = (K[5] * K[6] - K[3] * K[8]) / det; Ki[4] = (K[0] * K[8] - K[2] * K[6]) / det; Ki[5] = (K[2] * K[3] - K[0] * K[5]) / det;
    Ki[6] = (K[3] * K[7] - K[4] * K[6]) / det; Ki[7] = (K[1] * K[6] - K[0] * K[7]) / det; Ki[8] = (K[0] * K[4] - K[1] * K[3]) / det;
}

static int fail_cameras(mocap_ctx* ctx, unsigned cams, const char* what) {
    char list[128];
    int k = 0;
    list[0] = 0;
    for (int c = 0; c < 32 && k < 120; ++c)
        if ((cams >> c) & 1u) k += snprintf(list + k, sizeof(list) - k, "%s%d", k ? ", " : "", c);
    return mocap_fail(ctx, MOCAP_EINVAL, "mocap_calibrate_graph_host: %s; camera(s) %s not connected to camera 0", what, list);
}

extern "C" void mocap_graph_default_options(mocap_graph_options* opt) {
    if (!opt) return;
    opt->min_common = 30;
    opt->min_inliers = 30;
    opt->min_angle_deg = 2.0;
    opt->rot_outlier_deg = 5.0;
    opt->irls_rounds = 4;
}

extern "C" int mocap_calibrate_graph_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                          const mocap_ransac_options* ropt, const mocap_graph_options* gopt, double* R, double* t,
                                          mocap_graph_pair* pairs_out, int* n_pairs, uint8_t* support) {
    using namespace calib_pose;
    static const char* who = "mocap_calibrate_graph_host";
    if (!ctx) return MOCAP_EINVAL;
    const int C = ctx->cfg.n_cam;
    if (!obs || !mask || !R || !t || n_points < 8 || C < 2 || C > CG_MAX_CAM) return mocap_fail(ctx, MOCAP_EINVAL, "%s: bad argument", who);
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    mocap_ransac_options ro;
    int st = ransac_check_options(ctx, ropt, &ro, who);
    if (st) return st;
    mocap_graph_options go;
    mocap_graph_default_options(&go);
    if (gopt) go = *gopt;
    if (go.min_common < 8 || go.min_inliers < 1 || !(go.min_angle_deg >= 0.0) || !(go.min_angle_deg < 90.0) || !(go.rot_outlier_deg > 0.0) ||
        !(go.rot_outlier_deg <= 180.0) || go.irls_rounds < 1 || go.irls_rounds > 64)
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: min_common must be >= 8, min_inliers >= 1, min_angle_deg in [0, 90), rot_outlier_deg in "
                          "(0, 180] and irls_rounds in 1..64 (got %d, %d, %g, %g, %d)", who, go.min_common, go.min_inliers,
                          go.min_angle_deg, go.rot_outlier_deg, go.irls_rounds);
    // 1. pair table
    std::vector<int> pa, pb;
    for (int a = 0; a < C; ++a)
        for (int b = a + 1; b < C; ++b) {
            int m = 0;
            for (int f = 0; f < n_points; ++f) m += (mask[(size_t)f * C + a] && mask[(size_t)f * C + b]) ? 1 : 0;
            if (m >= go.min_common) { pa.push_back(a); pb.push_back(b); }
        }
    const PairTable tab = pair_table(obs, mask, n_points, C, pa, pb);
    const std::vector<int>& off = tab.off;
    const int P = tab.pairs();
    {
        std::vector<uint8_t> all(P, 1);
        const unsigned lost = P ? cg_disconnected(C, P, pa.data(), pb.data(), all.data()) : ((1u << C) - 2u);
        if (lost) return fail_cameras(ctx, lost, "too few common observations (min_common) to link every camera");
    }
    // 2. RANSAC over the pair table
    std::vector<double> F(9 * (size_t)P);
    std::vector<uint8_t> inl(tab.pts.size());
    std::vector<unsigned long long> keys(P);
    st = ransac_run(ctx, tab, ro, F.data(), inl.data(), keys.data());
    if (st) { cudaGetLastError(); return st; }
    // device buffers of the later stages
    const size_t total = tab.pts.size(), nv = (size_t)n_points * C;
    const int mmax = tab.max_count();
    const int n3 = 3 * C, E = n3 * (n3 + 1) / 2;
    const int chunk = 64;
    const int G = (n_points + chunk - 1) / chunk;
    PairDev d;
    int* d_cnt; uint8_t *d_init, *d_front; CgCams* d_cams;
    double *d_cand, *d_ang, *d_obs, *d_w[2], *d_t, *d_part, *d_H;
    st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
        d.take(L, tab);
        d_cand = L.take<double>((size_t)P * 4 * CG_CAND); d_cnt = L.take<int>((size_t)P * 4); d_ang = L.take<double>(total * 4);
        d_obs = L.take<double>(nv * 2); d_init = L.take<uint8_t>(nv); d_w[0] = L.take<double>(nv); d_w[1] = L.take<double>(nv);
        d_front = L.take<uint8_t>(nv); d_cams = L.take<CgCams>(1);
        d_t = L.take<double>(n3); d_part = L.take<double>((size_t)G * E); d_H = L.take<double>(E);
    });
    if (st) { cudaGetLastError(); return st; }
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d.pts, tab.pts.data(), total * sizeof(float4), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d.off, off.data(), (P + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
    // 3. re-fits: three 8-point fits, each followed by a Sampson re-selection at the RANSAC threshold; the last
    //    selection is the pair's inlier set.  A pair without a model, or whose selection falls under 8 points, keeps
    //    its previous set.
    std::vector<uint8_t> ok(P), fitted(P);
    for (int p = 0; p < P; ++p) {
        ok[p] = keys[p] ? 1 : 0;
        int k = 0;
        for (int i = off[p]; i < off[p + 1]; ++i) k += inl[i];
        if (k < 8) for (int i = off[p]; i < off[p + 1]; ++i) inl[i] = 1;
    }
    const double thr2 = ro.threshold_px * ro.threshold_px;
    std::vector<uint8_t> sel(total);
    for (int round = 0; round < 3; ++round) {
        if ((st = fit_pairs(ctx, tab, d, inl.data(), F.data(), fitted.data()))) return st;
        for (int p = 0; p < P; ++p) ok[p] &= fitted[p];
        if ((st = select_pairs(ctx, tab, d, F.data(), thr2, sel.data()))) return st;
        for (int p = 0; p < P; ++p) {
            int k = 0;
            for (int i = off[p]; i < off[p + 1]; ++i) k += sel[i];
            if (k >= 8) for (int i = off[p]; i < off[p + 1]; ++i) inl[i] = sel[i];
        }
    }
    // 4. cheirality in each pair's own frame
    std::vector<double> cand((size_t)P * 4 * CG_CAND, 0.0), Rs_all((size_t)P * 4 * 9), ts_all((size_t)P * 4 * 3);
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z3[3] = {0, 0, 0};
    for (int p = 0; p < P; ++p) {
        const double* Ka = ctx->h_tables.Kmat[pa[p]];
        const double* Kb = ctx->h_tables.Kmat[pb[p]];
        double Kbt[9], tmp[9], Ess[9], Rs[4][9], ts[4][3];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Kbt[3 * i + j] = Kb[3 * j + i];
        mat3mul(Kbt, &F[9 * p], tmp); mat3mul(tmp, Ka, Ess);
        motion_from_essential(Ess, Rs, ts);
        for (int q = 0; q < 4; ++q) {
            double* c = &cand[(size_t)(4 * p + q) * CG_CAND];
            cg_make_P(Ka, I3, z3, c);
            cg_make_P(Kb, Rs[q], ts[q], c + 12);
            memcpy(c + 24, Rs[q], 9 * 8); memcpy(c + 33, ts[q], 3 * 8);
            memcpy(&Rs_all[(size_t)(4 * p + q) * 9], Rs[q], 9 * 8); memcpy(&ts_all[(size_t)(4 * p + q) * 3], ts[q], 3 * 8);
        }
    }
    std::vector<int> counts((size_t)P * 4);
    std::vector<double> ang(total * 4);
    CUDA_TRY(ctx, cudaMemcpyAsync(d_cand, cand.data(), cand.size() * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d.inl, inl.data(), total, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemsetAsync(d_cnt, 0, (size_t)P * 4 * sizeof(int), s));
    k_pair_cheirality<<<dim3((4 * mmax + CG_THREADS - 1) / CG_THREADS, P), CG_THREADS, 0, s>>>(d.pts, d.off, d.inl, d_cand, d_cnt, d_ang);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaMemcpyAsync(counts.data(), d_cnt, counts.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(ang.data(), d_ang, ang.size() * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    std::vector<mocap_graph_pair> rep(P);
    std::vector<double> Rab((size_t)P * 9), wrot(P), resid(P, NAN);
    std::vector<uint8_t> use(P, 0);
    for (int p = 0; p < P; ++p) {
        mocap_graph_pair& r = rep[p];
        r.a = pa[p]; r.b = pb[p]; r.common = tab.count(p);
        r.inliers = 0;
        for (int i = off[p]; i < off[p + 1]; ++i) r.inliers += inl[i];
        int best = -1, bc = 0;
        for (int q = 0; q < 4; ++q) if (counts[4 * p + q] > bc) { bc = counts[4 * p + q]; best = q; }     // strict >, first maximum
        r.candidate = ok[p] ? best : -1;
        r.in_front = ok[p] ? bc : 0;
        r.median_angle_deg = NAN;
        r.rot_residual_deg = NAN;
        r.used = 0;
        if (r.candidate < 0) continue;
        std::vector<double> av;
        for (int i = off[p]; i < off[p + 1]; ++i) if (ang[(size_t)i * 4 + best] >= 0.0) av.push_back(ang[(size_t)i * 4 + best]);
        std::sort(av.begin(), av.end());
        const size_t h = av.size();
        r.median_angle_deg = h ? (h % 2 ? av[h / 2] : 0.5 * (av[h / 2 - 1] + av[h / 2])) : 0.0;
        memcpy(&Rab[9 * (size_t)p], &Rs_all[(size_t)(4 * p + best) * 9], 9 * 8);
        wrot[p] = bc;
        use[p] = (bc >= go.min_inliers && r.median_angle_deg >= go.min_angle_deg) ? 1 : 0;
    }
    // 5. rotation averaging
    {
        const unsigned lost = cg_disconnected(C, P, pa.data(), pb.data(), use.data());
        if (lost) return fail_cameras(ctx, lost, "too few pairs pass the cheirality and angle checks");
    }
    std::vector<double> Rh(9 * (size_t)C);
    if (!cg_rotation_average(C, P, pa.data(), pb.data(), Rab.data(), wrot.data(), go.rot_outlier_deg, use.data(), Rh.data(), resid.data())) {
        const unsigned lost = cg_disconnected(C, P, pa.data(), pb.data(), use.data());
        return lost ? fail_cameras(ctx, lost, "the pairs that agree on the rotations do not link every camera")
                    : mocap_fail(ctx, MOCAP_EINVAL, "%s: rotation averaging failed", who);
    }
    for (int p = 0; p < P; ++p) { rep[p].used = use[p]; if (rep[p].candidate >= 0) rep[p].rot_residual_deg = resid[p]; }
    // 6. translations.  A view enters if it is an inlier of at least 2 used pairs (1 for a camera with one used pair).
    std::vector<int> npairs(C, 0), hits(nv, 0);
    for (int p = 0; p < P; ++p) {
        if (!use[p]) continue;
        ++npairs[pa[p]]; ++npairs[pb[p]];
        for (int f = 0, i = off[p]; f < n_points; ++f)
            if (mask[(size_t)f * C + pa[p]] && mask[(size_t)f * C + pb[p]]) {
                if (inl[i]) { ++hits[(size_t)f * C + pa[p]]; ++hits[(size_t)f * C + pb[p]]; }
                ++i;
            }
    }
    std::vector<uint8_t> init(nv);
    std::vector<double> w0(nv);
    for (size_t k = 0; k < nv; ++k) {
        const int c = (int)(k % C);
        init[k] = mask[k] && hits[k] >= (npairs[c] >= 2 ? 2 : 1) ? 1 : 0;
        w0[k] = init[k] ? 1.0 : 0.0;
    }
    CgCams cams;
    memset(&cams, 0, sizeof(cams));
    for (int c = 0; c < C; ++c) {
        memcpy(cams.R[c], &Rh[9 * (size_t)c], 9 * 8);
        inv3(ctx->h_tables.Kmat[c], cams.Kinv[c]);
        cams.f[c] = ctx->h_tables.Kmat[c][0];
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(d_obs, obs, nv * 2 * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_init, init.data(), nv, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_w[0], w0.data(), nv * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_cams, &cams, sizeof(cams), cudaMemcpyHostToDevice, s));
    std::vector<double> Hu(E), th(n3);
    int cur = 0;
    for (int round = 0; round < go.irls_rounds; ++round) {
        k_translation_normal<<<G, CG_THREADS, 0, s>>>(d_obs, d_w[cur], n_points, C, d_cams, chunk, d_part);
        CUDA_TRY(ctx, cudaGetLastError());
        k_translation_reduce<<<(E + CG_THREADS - 1) / CG_THREADS, CG_THREADS, 0, s>>>(d_part, G, E, d_H);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 2;
        CUDA_TRY(ctx, cudaMemcpyAsync(Hu.data(), d_H, E * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        if (!cg_translation_solve(C, Hu.data(), th.data())) return mocap_fail(ctx, MOCAP_EINVAL, "%s: translation eigen-decomposition failed", who);
        CUDA_TRY(ctx, cudaMemcpyAsync(d_t, th.data(), n3 * 8, cudaMemcpyHostToDevice, s));
        k_translation_residuals<<<(int)((nv + CG_THREADS - 1) / CG_THREADS), CG_THREADS, 0, s>>>(d_obs, d_init, d_w[cur], n_points, C, d_cams,
                                                                                                  d_t, CG_SCALE_PX, d_w[cur ^ 1], d_front);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        cur ^= 1;
    }
    std::vector<double> wf(nv);
    std::vector<uint8_t> front(nv);
    CUDA_TRY(ctx, cudaMemcpyAsync(wf.data(), d_w[cur], nv * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(front.data(), d_front, nv, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    // 7. output: sign by the views in front, the chain's gauge, support = weight >= 0.5 on tracks that keep 2 views
    std::vector<uint8_t> sup(nv, 0);
    long n_front = 0, n_back = 0;
    for (int f = 0; f < n_points; ++f) {
        int k = 0;
        for (int c = 0; c < C; ++c) k += wf[(size_t)f * C + c] >= 0.5 ? 1 : 0;
        if (k < 2) continue;
        for (int c = 0; c < C; ++c) {
            const size_t i = (size_t)f * C + c;
            if (wf[i] < 0.5) continue;
            sup[i] = 1;
            if (front[i]) ++n_front; else ++n_back;
        }
    }
    cg_gauge(C, th.data(), n_front, n_back);
    memcpy(R, Rh.data(), 9 * (size_t)C * 8);
    memcpy(t, th.data(), n3 * 8);
    if (support) memcpy(support, sup.data(), nv);
    if (pairs_out) memcpy(pairs_out, rep.data(), P * sizeof(mocap_graph_pair));
    if (n_pairs) *n_pairs = P;
    return MOCAP_OK;
}

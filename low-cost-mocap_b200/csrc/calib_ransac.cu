// Robust cold-start calibration: RANSAC fundamental matrices for all C-1 adjacent camera pairs on the device, then
// the pose chain of calib_init.cu refined from each pair's RANSAC inliers.
//
// The reference's calculate-camera-pose handler estimates each pair's F with cv.findFundamentalMat(FM_RANSAC, 1 px,
// 0.99999) (index.py:246); mocap_calibrate_init_host fits a normalised 8-point model to all common observations,
// which a single mismatched point can pull away.  Here (calib_ransac.cuh for the per-hypothesis arithmetic):
//   k_ransac_hypotheses  one thread per (pair, hypothesis): deterministic 7-point sample, 7-point solver, 1-3 models
//   k_ransac_score       one warp per hypothesis, its models scored over the pair's points staged through shared
//                        memory; per-model inlier counts by ballot / popc, the winner by one 64-bit atomicMax of a
//                        packed (count, ~index) key per pair -- the most inliers, ties to the lowest (hypothesis, root)
//   k_ransac_mask        the winning model's inlier mask over every pair's points
// One launch of each for all pairs, whatever the number of cameras.  cv2 stops adaptively (confidence 0.99999, at
// most 1000 iterations); a fixed budget of H >= 1000 hypotheses per pair needs no sequential stopping rule.
#include <vector>
#include <math.h>
#include "common.cuh"
#include "calib_ransac.cuh"

#define RS_HYP_THREADS  128
#define RS_SCORE_WARPS  8       // hypotheses per CTA of k_ransac_score
#define RS_TILE         1024    // correspondences per shared-memory tile (16 KB)
#define RS_MAX_HYP      65536

// pts: every pair's common observations {x1, y1, x2, y2} (float32, as the reference casts them), pair p at
// [off[p], off[p+1]); models [P][H][3][9], n_models [P][H]
__global__ void __launch_bounds__(RS_HYP_THREADS)
k_ransac_hypotheses(const float4* __restrict__ pts, const int* __restrict__ off, int H, unsigned long long seed,
                    double* __restrict__ models, int* __restrict__ n_models) {
    const int p = blockIdx.y, h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    const int o = off[p], m = off[p + 1] - o;
    double F[3][9];
    const int n = rs_hypothesis(pts + o, m, seed, p, h, F);
    double* out = models + ((size_t)p * H + h) * 27;
    for (int k = 0; k < n; ++k)
        for (int i = 0; i < 9; ++i) out[9 * k + i] = F[k][i];
    n_models[(size_t)p * H + h] = n;
}

__global__ void __launch_bounds__(RS_SCORE_WARPS * 32)
k_ransac_score(const float4* __restrict__ pts, const int* __restrict__ off, int H, double thr2, const double* __restrict__ models,
               const int* __restrict__ n_models, unsigned long long* __restrict__ best) {
    __shared__ float4 tile[RS_TILE];
    const int p = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int h = blockIdx.x * RS_SCORE_WARPS + warp;
    const int n = h < H ? n_models[(size_t)p * H + h] : 0;
    double F[3][9];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int i = 0; i < 9; ++i) F[k][i] = k < n ? models[((size_t)p * H + h) * 27 + 9 * k + i] : 0.0;
    int cnt[3] = {0, 0, 0};
    const int o = off[p], m = off[p + 1] - o;
    for (int base = 0; base < m; base += RS_TILE) {
        const int tc = min(RS_TILE, m - base);
        __syncthreads();
        for (int i = threadIdx.x; i < tc; i += blockDim.x) tile[i] = pts[o + base + i];
        __syncthreads();
        if (n == 0) continue;
        for (int i0 = 0; i0 < tc; i0 += 32) {
            const int i = i0 + lane;
            const float4 v = tile[i < tc ? i : 0];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (k >= n) break;
                const bool ok = i < tc && rs_is_inlier(F[k], v.x, v.y, v.z, v.w, thr2);
                cnt[k] += __popc(__ballot_sync(0xffffffffu, ok));
            }
        }
    }
    if (lane == 0)
        for (int k = 0; k < n; ++k) atomicMax(best + p, rs_key(cnt[k], h, k));
}

// inl: mask over pts (same layout); F_best [P][9] the winning models (zeros for a pair without any model)
__global__ void __launch_bounds__(256)
k_ransac_mask(const float4* __restrict__ pts, const int* __restrict__ off, int H, double thr2, const double* __restrict__ models,
              const unsigned long long* __restrict__ best, uint8_t* __restrict__ inl, double* __restrict__ F_best) {
    const int p = blockIdx.y;
    const unsigned long long key = best[p];
    const uint32_t idx = ~(uint32_t)key;
    double F[9];
    for (int i = 0; i < 9; ++i) F[i] = key ? models[((size_t)p * H + idx / 3) * 27 + 9 * (idx % 3) + i] : 0.0;
    if (blockIdx.x == 0 && threadIdx.x < 9) F_best[9 * p + threadIdx.x] = F[threadIdx.x];
    const int o = off[p], m = off[p + 1] - o;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const float4 v = pts[o + i];
        inl[o + i] = key && rs_is_inlier(F, v.x, v.y, v.z, v.w, thr2) ? 1 : 0;
    }
}

int ransac_check_options(mocap_ctx* ctx, const mocap_ransac_options* opt, mocap_ransac_options* o, const char* who) {
    mocap_ransac_default_options(o);
    if (opt) *o = *opt;
    if (!(o->threshold_px > 0) || !isfinite(o->threshold_px) || o->hypotheses < 1 || o->hypotheses > RS_MAX_HYP)
        return mocap_fail(ctx, MOCAP_EINVAL, "%s: threshold_px must be positive and finite and hypotheses in 1..%d (got %g, %d)", who,
                          RS_MAX_HYP, o->threshold_px, o->hypotheses);
    return MOCAP_OK;
}

int ransac_run(mocap_ctx* ctx, const PairTable& tab, const mocap_ransac_options& o, double* F_best, uint8_t* inl, unsigned long long* keys) {
    const int H = o.hypotheses, P = tab.pairs();
    const double thr2 = o.threshold_px * o.threshold_px;
    const size_t total = tab.pts.size();
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    float4* d_pts; int *d_off, *d_n; double *d_models, *d_F; unsigned long long* d_best; uint8_t* d_inl;
    int st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
        d_pts = L.take<float4>(total); d_off = L.take<int>(P + 1);
        d_models = L.take<double>((size_t)P * H * 27); d_n = L.take<int>((size_t)P * H);
        d_best = L.take<unsigned long long>(P); d_F = L.take<double>((size_t)P * 9); d_inl = L.take<uint8_t>(total);
    });
    if (st) return st;
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(d_pts, tab.pts.data(), total * sizeof(float4), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(d_off, tab.off.data(), (P + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemsetAsync(d_best, 0, P * sizeof(unsigned long long), s));
    k_ransac_hypotheses<<<dim3((H + RS_HYP_THREADS - 1) / RS_HYP_THREADS, P), RS_HYP_THREADS, 0, s>>>(
        d_pts, d_off, H, (unsigned long long)o.seed, d_models, d_n);
    CUDA_TRY(ctx, cudaGetLastError());
    k_ransac_score<<<dim3((H + RS_SCORE_WARPS - 1) / RS_SCORE_WARPS, P), RS_SCORE_WARPS * 32, 0, s>>>(d_pts, d_off, H, thr2, d_models,
                                                                                                      d_n, d_best);
    CUDA_TRY(ctx, cudaGetLastError());
    const int mmax = tab.max_count();
    k_ransac_mask<<<dim3((mmax + 255) / 256 < 32 ? (mmax + 255) / 256 : 32, P), 256, 0, s>>>(d_pts, d_off, H, thr2, d_models, d_best,
                                                                                            d_inl, d_F);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 3;
    CUDA_TRY(ctx, cudaMemcpyAsync(keys, d_best, P * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(F_best, d_F, P * 9 * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(inl, d_inl, total, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    return MOCAP_OK;
}

PairTable pair_table(const double* obs, const uint8_t* mask, int n_points, int C, const std::vector<int>& a, const std::vector<int>& b) {
    PairTable tab{a, b, {}, {0}};
    for (size_t k = 0; k < a.size(); ++k) {
        for (int f = 0; f < n_points; ++f)
            if (mask[(size_t)f * C + a[k]] && mask[(size_t)f * C + b[k]]) {      // index.py:242-244
                const double* xa = obs + ((size_t)f * C + a[k]) * 2;
                const double* xb = obs + ((size_t)f * C + b[k]) * 2;
                tab.pts.push_back(make_float4((float)xa[0], (float)xa[1], (float)xb[0], (float)xb[1]));
            }
        tab.off.push_back((int)tab.pts.size());
    }
    return tab;
}

int adjacent_pairs(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points, const char* who, PairTable& tab) {
    const int C = ctx->cfg.n_cam;
    std::vector<int> a, b;
    for (int c = 0; c + 1 < C; ++c) { a.push_back(c); b.push_back(c + 1); }
    tab = pair_table(obs, mask, n_points, C, a, b);
    for (int c = 0; c + 1 < C; ++c)
        if (tab.count(c) < 8) return mocap_fail(ctx, MOCAP_EINVAL, "%s: cameras %d and %d share only %d observations", who, c, c + 1, tab.count(c));
    return MOCAP_OK;
}

void scatter_pairs(const PairTable& tab, const uint8_t* mask, int n_points, int C, const uint8_t* sel, uint8_t* out) {
    const int P = tab.pairs();
    memset(out, 0, (size_t)n_points * P);
    for (int p = 0; p < P; ++p)
        for (int f = 0, k = tab.off[p]; f < n_points; ++f)
            if (mask[(size_t)f * C + tab.a[p]] && mask[(size_t)f * C + tab.b[p]]) out[(size_t)f * P + p] = sel[k++];
}

// RANSAC over every adjacent pair: F_best [C-1][9], the adjacent table and the inlier mask over it.  Validates
// everything before any launch.
static int ransac_pairs(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points, const mocap_ransac_options* opt,
                        double* F_best, std::vector<uint8_t>& inl, PairTable& tab, const char* who) {
    const int C = ctx->cfg.n_cam, P = C - 1;
    if (!obs || !mask || n_points < 8 || C < 2) return mocap_fail(ctx, MOCAP_EINVAL, "%s: bad argument", who);
    mocap_ransac_options o;
    int st = ransac_check_options(ctx, opt, &o, who);
    if (st) return st;
    st = adjacent_pairs(ctx, obs, mask, n_points, who, tab);
    if (st) return st;
    std::vector<unsigned long long> keys(P);
    inl.resize(tab.pts.size());
    st = ransac_run(ctx, tab, o, F_best, inl.data(), keys.data());
    if (st) return st;
    for (int c = 0; c < P; ++c)
        if (!keys[c]) return mocap_fail(ctx, MOCAP_EINVAL, "%s: no 7-point sample of cameras %d and %d gave a model", who, c, c + 1);
    return MOCAP_OK;
}

extern "C" void mocap_ransac_default_options(mocap_ransac_options* opt) {
    if (!opt) return;
    opt->threshold_px = 1.0;
    opt->hypotheses = 2048;
    opt->seed = 0;
}

extern "C" int mocap_fundamental_ransac_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                             const mocap_ransac_options* opt, double* F, uint8_t* inliers) {
    if (!ctx) return MOCAP_EINVAL;
    if (!F) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_fundamental_ransac_host: bad argument");
    std::vector<uint8_t> inl;
    PairTable tab;
    const int st = ransac_pairs(ctx, obs, mask, n_points, opt, F, inl, tab, "mocap_fundamental_ransac_host");
    if (st) return st;
    if (inliers) scatter_pairs(tab, mask, n_points, ctx->cfg.n_cam, inl.data(), inliers);
    return MOCAP_OK;
}

extern "C" int mocap_calibrate_init_ransac_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                                                const mocap_ransac_options* opt, double* R, double* t, double* F_used, int* votes,
                                                uint8_t* inliers) {
    if (!ctx) return MOCAP_EINVAL;
    if (!R || !t) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_calibrate_init_ransac_host: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    std::vector<double> F_best(9 * (size_t)(ctx->cfg.n_cam > 1 ? ctx->cfg.n_cam - 1 : 1));
    std::vector<uint8_t> inl;
    PairTable tab;
    int st = ransac_pairs(ctx, obs, mask, n_points, opt, F_best.data(), inl, tab, "mocap_calibrate_init_ransac_host");
    if (st) return st;
    const double thr = opt ? opt->threshold_px : 1.0;
    return calibrate_chain(ctx, tab, mask, n_points, nullptr, inl.data(), thr * thr, R, t, F_used, votes, inliers);
}

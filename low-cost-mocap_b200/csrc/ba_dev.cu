// S4 on the device, launch side: k_ba_solve (ba_device.cuh) as ONE cooperative launch, plus the two small
// kernels that turn the matcher's tracks of a batch into the explicit correspondences S4 consumes, so that
// "S1-S3, then one bundle adjustment per batch" (BASELINE config 3) never touches the host.
//
// Replaces bundle_adjustment (reference computer_code/api/helpers.py:244-290) behind
// mocap_bundle_adjust_dev / mocap_bundle_adjust_host.
#include "common.cuh"
#include "ba_device.cuh"

#define BA_THREADS 512

// one launch runs B.n independent problems, each on its own range of CTAs; a single solve is a batch of one.
// __grid_constant__: the table is read in place, without a per-thread copy.  Each CTA copies its problem to shared
// memory once (the body reads its per-problem pointers from there, ba_fresh); what all problems share comes from
// problem 0 at fixed parameter offsets
__global__ void __launch_bounds__(BA_THREADS, 1) k_ba_solve(const __grid_constant__ BABatch B) {
    extern __shared__ __align__(16) unsigned char ba_smem_raw[];
    __shared__ BAParams problem;
    if (threadIdx.x == 0) problem = B.p[ba_problem_of(B)];
    __syncthreads();
    ba_solve_body(problem, B.p[0], ba_smem_raw);
}

// ---- tracks -> observations --------------------------------------------------------------------------------
// kept[s] = tracks of frame-set s that go to S4 (every track the matcher emitted has >= 2 views; max_err > 0 drops
// those whose reprojection error exceeds it); exclusive scan over the frame-sets -> offs, total -> n_points
__global__ void __launch_bounds__(1024)
k_track_offsets(const int32_t* __restrict__ n_obj, const double* __restrict__ err, int n_sets, int RMAX, double max_err,
                int capacity, int32_t* __restrict__ offs, int32_t* __restrict__ n_points) {
    __shared__ int warp_sum[32];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int s0 = 0; s0 < n_sets; s0 += blockDim.x) {
        const int s = s0 + tid;
        int kept = 0;
        if (s < n_sets) {
            const int k = min(n_obj[s], RMAX);
            if (max_err > 0.0) { for (int r = 0; r < k; ++r) kept += (err[(size_t)s * RMAX + r] <= max_err) ? 1 : 0; }
            else kept = k;
        }
        int v = kept;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
        if (lane == 31) warp_sum[wid] = v;
        __syncthreads();
        if (wid == 0) {
            int w = lane < (int)(blockDim.x >> 5) ? warp_sum[lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
            warp_sum[lane] = w;
        }
        __syncthreads();
        const int before = carry + (wid > 0 ? warp_sum[wid - 1] : 0) + v - kept;
        if (s < n_sets) offs[s] = before;
        __syncthreads();
        if (tid == (int)blockDim.x - 1) carry = before + kept;
        __syncthreads();
    }
    if (tid == 0) *n_points = carry < capacity ? carry : capacity;
}

__global__ void __launch_bounds__(256)
k_tracks_to_obs(const int32_t* __restrict__ track_xy, const int32_t* __restrict__ n_obj, const double* __restrict__ err,
                const int32_t* __restrict__ offs, int n_sets, int RMAX, int C, double max_err, int capacity,
                double* __restrict__ obs, uint8_t* __restrict__ mask) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n_sets * RMAX) return;
    const int s = (int)(idx / RMAX), r = (int)(idx - (long long)s * RMAX);
    if (r >= min(n_obj[s], RMAX)) return;
    int rank = r;
    if (max_err > 0.0) {
        if (!(err[(size_t)s * RMAX + r] <= max_err)) return;
        rank = 0;
        for (int q = 0; q < r; ++q) rank += (err[(size_t)s * RMAX + q] <= max_err) ? 1 : 0;
    }
    const int p = offs[s] + rank;
    if (p >= capacity) return;
    const int32_t* t = track_xy + ((size_t)s * RMAX + r) * C * 2;
    for (int c = 0; c < C; ++c) {
        const int x = t[2 * c], y = t[2 * c + 1];
        const bool seen = x >= 0;
        obs[((size_t)p * C + c) * 2] = seen ? (double)x : 0.0;
        obs[((size_t)p * C + c) * 2 + 1] = seen ? (double)y : 0.0;
        mask[(size_t)p * C + c] = seen ? 1 : 0;
    }
}

// ---- host side ---------------------------------------------------------------------------------------------
int ba_dev_init(mocap_ctx* ctx) {
    const int C = ctx->cfg.n_cam;
    ctx->ba_threads = BA_THREADS;
    ctx->ba_smem = ba_smem_bytes(C, BA_THREADS);
    ctx->ba_grid = 0;
    if (C < 2) return MOCAP_OK;                                   // no bundle adjustment with one camera
    if (ctx->ba_smem > 227 * 1024) return MOCAP_OK;               // entry point reports it
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_ba_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->ba_smem));
    int per_sm = 0;
    CUDA_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_ba_solve, BA_THREADS, ctx->ba_smem));
    if (per_sm < 1) return MOCAP_OK;
    ctx->ba_grid = ctx->num_sms;                                  // one CTA per SM, all co-resident (cooperative launch)
    const char* g = getenv("MOCAP_BA_GRID");                      // measurement switch
    if (g && atoi(g) > 0 && atoi(g) <= ctx->num_sms * per_sm) ctx->ba_grid = atoi(g);
    return MOCAP_OK;
}

// per-problem carve of the context's workspace
struct BAProblemWS { double* X; double* Xnew; uint8_t* valid; double* part; double* fin; double* cpart; unsigned* bar; };
struct BAWorkspace {
    BAProblemWS pr[MOCAP_BA_MAX_BATCH];
    double* Rt_io; int32_t* offs; mocap_ba_report* report;
};

#define BA_BAR_LINE 128                                           // bytes: each problem's barrier words on a line of their own

// carve the workspace for K problems of m_max[k] points on g[k] CTAs (K = 0: none, the offsets of n_sets frame-sets only)
static int ba_workspace(mocap_ctx* ctx, int K, const int* m_max, const int* g, int n_sets, BAWorkspace& W, int* pstride_out) {
    const int C = ctx->cfg.n_cam, n = 6 * (C - 1), npair = n * (n + 1) / 2;
    const int pstride = npair + 2 * n + 8;
    const size_t sets = n_sets > 0 ? n_sets : 1;
    // the whole workspace is zeroed when it grows (the grid barriers start at zero); the barrier words come FIRST so
    // that they keep their place (and their generation counts) when nothing grows
    int st = grow_carved(ctx, ctx->ba_ws, Drain::stream, [&](Layout& L) {
        uint8_t* bars = L.take<uint8_t>((size_t)MOCAP_BA_MAX_BATCH * BA_BAR_LINE);
        for (int k = 0; k < K; ++k) {
            BAProblemWS& w = W.pr[k];
            const size_t m = (size_t)m_max[k], G = (size_t)g[k];
            w.bar = bars ? (unsigned*)(bars + (size_t)k * BA_BAR_LINE) : nullptr;
            w.X = L.take<double>(m * 3); w.Xnew = L.take<double>(m * 3); w.valid = L.take<uint8_t>(m);
            w.part = L.take<double>(G * pstride); w.fin = L.take<double>(pstride); w.cpart = L.take<double>(2 * G * 4);
        }
        W.Rt_io = L.take<double>((size_t)C * 12); W.offs = L.take<int32_t>(sets);
        W.report = L.take<mocap_ba_report>(1);
        L.zero_so_far();
    });
    if (st) return st;
    *pstride_out = pstride;
    return MOCAP_OK;
}

// one cooperative launch of k_ba_solve over the K problems (arguments checked by the caller): problem k gets
// G / K + (k < G % K) of the context's G CTAs
static int ba_launch(mocap_ctx* ctx, const mocap_ba_problem* pr, int K, const mocap_ba_options* opt_in) {
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    mocap_ba_options opt;
    if (opt_in) opt = *opt_in; else mocap_ba_default_options(&opt);
    const int G = ctx->ba_grid;
    int m_max[MOCAP_BA_MAX_BATCH], g[MOCAP_BA_MAX_BATCH];
    for (int k = 0; k < K; ++k) { m_max[k] = pr[k].n_points_max; g[k] = G / K + (k < G % K ? 1 : 0); }
    BAWorkspace W;
    int pstride = 0;
    int st = ba_workspace(ctx, K, m_max, g, 0, W, &pstride);
    if (st) return st;
    BABatch B;
    memset(&B, 0, sizeof(B));
    B.n = K;
    for (int k = 0, cta0 = 0; k < K; cta0 += g[k], ++k) {
        BAParams& P = B.p[k];
        const BAProblemWS& w = W.pr[k];
        P.tb = ctx->d_tables; P.obs = pr[k].obs; P.mask = pr[k].mask; P.m_dev = pr[k].n_points; P.m_max = pr[k].n_points_max;
        P.C = ctx->cfg.n_cam; P.R = pr[k].R; P.t = pr[k].t;
        P.ftol = opt.ftol; P.xtol = opt.xtol; P.gtol = opt.gtol; P.max_nfev = opt.max_nfev;
        P.jac_mode = opt.jacobian ? 1 : 0; P.prefit = opt.prefit ? 1 : 0; P.prefit_max_iter = opt.prefit_max_iter;
        P.X = w.X; P.Xnew = w.Xnew; P.valid = w.valid; P.part = w.part; P.pstride = pstride; P.fin = w.fin; P.cpart = w.cpart;
        P.bar = w.bar; P.report = pr[k].report;
        P.cta0 = cta0; P.ncta = g[k];
    }
    void* args[] = {&B};
    CUDA_TRY(ctx, cudaLaunchCooperativeKernel((const void*)k_ba_solve, dim3(G), dim3(ctx->ba_threads), args, ctx->ba_smem, ctx->stream));
    ctx->launches += 1;
    return MOCAP_OK;
}

extern "C" {

int mocap_set_ba_grid(mocap_ctx* ctx, int n_ctas) {
    if (!ctx) return MOCAP_EINVAL;
    if (ctx->ba_grid < 1) return mocap_fail(ctx, MOCAP_EINVAL, "bundle adjustment is not available for this context (cameras: %d)", ctx->cfg.n_cam);
    if (n_ctas < 0 || n_ctas > ctx->num_sms)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_set_ba_grid: %d CTAs asked, 1 .. %d possible (0: default)", n_ctas, ctx->num_sms);
    // the workspace is carved per call from the grid in force (ba_workspace), the barrier words keep their place
    ctx->ba_grid = n_ctas == 0 ? ctx->num_sms : n_ctas;
    return MOCAP_OK;
}

int mocap_tracks_to_observations_dev(mocap_ctx* ctx, const int32_t* track_xy, const int32_t* n_obj, const double* err,
                                     int n_frame_sets, double max_err, double* obs, uint8_t* mask, int32_t* n_points,
                                     int capacity) {
    if (!ctx) return MOCAP_EINVAL;
    if (!track_xy || !n_obj || !obs || !mask || !n_points || n_frame_sets < 0 || capacity < 1 || (max_err > 0.0 && !err))
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_tracks_to_observations_dev: bad argument");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    BAWorkspace W;
    int pstride = 0;
    if (ctx->ba_grid < 1) return mocap_fail(ctx, MOCAP_EINVAL, "bundle adjustment needs at least two cameras");
    int st = ba_workspace(ctx, 0, nullptr, nullptr, n_frame_sets, W, &pstride);
    if (st) return st;
    const int RM = ctx->cfg.max_roots, C = ctx->cfg.n_cam;
    k_track_offsets<<<1, 1024, 0, ctx->stream>>>(n_obj, err, n_frame_sets, RM, max_err, capacity, W.offs, n_points);
    CUDA_TRY(ctx, cudaGetLastError());
    const long long total = (long long)n_frame_sets * RM;
    if (total > 0) {
        k_tracks_to_obs<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(track_xy, n_obj, err, W.offs, n_frame_sets, RM, C,
                                                                                 max_err, capacity, obs, mask);
        CUDA_TRY(ctx, cudaGetLastError());
    }
    ctx->launches += 2;
    return MOCAP_OK;
}

int mocap_bundle_adjust_dev(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points_max, const int32_t* n_points,
                            double* R, double* t, const mocap_ba_options* opt_in, mocap_ba_report* report) {
    if (!ctx) return MOCAP_EINVAL;
    if (!obs || !mask || !R || !t || n_points_max <= 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_bundle_adjust_dev: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    if (ctx->cfg.n_cam < 2) return mocap_fail(ctx, MOCAP_EINVAL, "bundle adjustment needs at least two cameras");
    if (ctx->ba_grid < 1) return mocap_fail(ctx, MOCAP_EINVAL, "k_ba_solve needs %zu bytes of shared memory per CTA for %d cameras", ctx->ba_smem, ctx->cfg.n_cam);
    // a batch of one on all the context's CTAs
    const mocap_ba_problem pr = {obs, mask, n_points_max, n_points, R, t, report};
    return ba_launch(ctx, &pr, 1, opt_in);
}

int mocap_bundle_adjust_batch_dev(mocap_ctx* ctx, const mocap_ba_problem* problems, int n_problems, const mocap_ba_options* opt) {
    if (!ctx) return MOCAP_EINVAL;
    if (!problems) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_bundle_adjust_batch_dev: problems is NULL");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    if (ctx->cfg.n_cam < 2) return mocap_fail(ctx, MOCAP_EINVAL, "bundle adjustment needs at least two cameras");
    if (ctx->ba_grid < 1) return mocap_fail(ctx, MOCAP_EINVAL, "k_ba_solve needs %zu bytes of shared memory per CTA for %d cameras", ctx->ba_smem, ctx->cfg.n_cam);
    if (n_problems < 1 || n_problems > MOCAP_BA_MAX_BATCH || n_problems > ctx->ba_grid)
        return mocap_fail(ctx, MOCAP_EINVAL, "mocap_bundle_adjust_batch_dev: %d problems, 1 .. %d possible (MOCAP_BA_MAX_BATCH, and at most the %d CTAs of the context)",
                          n_problems, MOCAP_BA_MAX_BATCH < ctx->ba_grid ? MOCAP_BA_MAX_BATCH : ctx->ba_grid, ctx->ba_grid);
    for (int k = 0; k < n_problems; ++k) {
        const mocap_ba_problem& p = problems[k];
        if (!p.obs || !p.mask || !p.R || !p.t || p.n_points_max <= 0)
            return mocap_fail(ctx, MOCAP_EINVAL, "mocap_bundle_adjust_batch_dev: bad argument in problem %d", k);
    }
    return ba_launch(ctx, problems, n_problems, opt);
}

}  // extern "C"

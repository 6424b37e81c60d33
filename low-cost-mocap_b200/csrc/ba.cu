// S4 on sm_90a: bundle adjustment of the camera poses.
//
// Replaces bundle_adjustment (reference computer_code/api/helpers.py:244-290):
//   x = [f0, (f_i, rotvec_i, t_i) i = 1..C-1]; residual_j(x) = float32(mean squared reprojection
//   error of point j after DLT re-triangulation with the poses of x) (helpers.py:264-276);
//   scipy least_squares(loss="cauchy", ftol=1e-2) -> TRF, 2-point finite-difference Jacobian.
//
// What runs where
//   GPU  k_ba_eval         residuals of every point for the current poses AND for every one-parameter
//                          perturbation in one launch (the reference pays 1 + 6(C-1) Python passes,
//                          each re-triangulating every point)
//        k_ba_rows/_gram   finite differences, Cauchy scaling of J and f (scipy
//                          scale_for_robust_loss_function), reduction to J^T J, J^T f, cost
//        k_sba_*           optional prefit: classic Levenberg-Marquardt BA over poses AND points with
//                          analytic Jacobians; each thread owns a point, eliminates its 3x3 block in
//                          registers (Schur complement) and adds its share of the dense reduced
//                          camera system, accumulated in shared memory
//   host trf_core.h        the n <= 90 dense eigen/Cholesky solves and the accept/reject logic
//
// The reference's objective is kept exactly (same residual definition, same float32 cast, same
// Cauchy cost); `prefit` and `jacobian == 1` only change HOW the minimum is approached -- the
// reference's own path is chaotic because it differentiates float32-quantised residuals with
// steps of 1.5e-8 (SURVEY.md section 7) -- and are switched off with prefit = 0, jacobian = 0.
#include <vector>
#include "common.cuh"
#include "geom.cuh"
#include "trf_core.h"
#include "ba_device.cuh"          // BA_PREFIT_REL_STOP and the device-resident solve's declarations

struct BAColumn { int cam; int pad; double Rt[12]; };     // pose of ONE camera replaced (cam < 0: none)

// K_k [R|t] summed like the BLAS micro-kernel the reference's numpy call runs (see mocap_set_cameras)
__device__ __forceinline__ void make_P(const double* __restrict__ Kk, const double* __restrict__ Rt, double P[12]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double acc = __dmul_rn(Kk[3 * i + 0], Rt[j]);
            acc = fma(Kk[3 * i + 1], Rt[4 + j], acc);
            acc = fma(Kk[3 * i + 2], Rt[8 + j], acc);
            P[4 * i + j] = acc;
        }
}

// residual_function of the reference for point p under (base poses with column col applied)
__device__ __forceinline__ double ba_point_residual(const CameraTables* __restrict__ tb, const double* __restrict__ baseRt,
                                                    const BAColumn& col, const double* __restrict__ o,
                                                    const uint8_t* __restrict__ mk, int C, double X[3]) {
    Sym4 B;
    sym4_zero(B);
    int k = 0;
    for (int c = 0; c < C; ++c)
        if (mk[c]) {
            const double* Rt = (c == col.cam) ? col.Rt : baseRt + 12 * c;
            double P[12];
            make_P(tb->Kmat[k], Rt, P);                  // K of the k-th present view (helpers.py:305-307)
            dlt_add_view(B, P, o[2 * c], o[2 * c + 1]);
            ++k;
        }
    dlt_solve(B, X);
    double sq[2 * MOCAP_MAX_CAM];
    k = 0;
    for (int c = 0; c < C; ++c)
        if (mk[c]) {
            const double* Rt = (c == col.cam) ? col.Rt : baseRt + 12 * c;
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

// one thread per (column, point).  f64[col][p] = residual in double, f32 = its float32 cast
// (helpers.py:273).  Threads whose column does not touch any view of the point are skipped:
// their finite difference is exactly zero in the reference as well.
__global__ void __launch_bounds__(128)
k_ba_eval(const CameraTables* __restrict__ tb, const double* __restrict__ baseRt, const BAColumn* __restrict__ cols,
          int ncol, const double* __restrict__ obs, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ valid,
          int m, int C, float* __restrict__ f32, double* __restrict__ f64, double* __restrict__ X_out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)m * ncol) return;
    const int col = (int)(idx / m), p = (int)(idx - (long long)col * m);
    if (!valid[p]) return;
    const BAColumn cc = cols[col];
    const uint8_t* mk = mask + (size_t)p * C;
    if (cc.cam >= 0 && !mk[cc.cam]) return;
    double X[3];
    const double r = ba_point_residual(tb, baseRt, cc, obs + (size_t)p * C * 2, mk, C, X);
    f64[(size_t)col * m + p] = r;
    f32[(size_t)col * m + p] = (float)r;
    if (X_out && col == 0) { X_out[3 * p] = X[0]; X_out[3 * p + 1] = X[1]; X_out[3 * p + 2] = X[2]; }
}

// per point: Cauchy pieces in the precisions scipy uses when the residual vector is float32
// (z, log1p, 1/t, -1/t^2 in float32; J_scale in float64; scaled f cast back to float32), and
// the scaled Jacobian row.  Js [n][m], fs [m], cterm [m].
__global__ void __launch_bounds__(128)
k_ba_rows(const float* __restrict__ f32, const double* __restrict__ f64, const BAColumn* __restrict__ cols,
          const double* __restrict__ dx, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ valid,
          int m, int C, int n, int jac_mode, double* __restrict__ Js, double* __restrict__ fs,
          double* __restrict__ cterm, int* __restrict__ nonfinite) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    if (!valid[p]) {
        fs[p] = 0.0; cterm[p] = 0.0;
        for (int j = 0; j < n; ++j) Js[(size_t)j * m + p] = 0.0;
        return;
    }
    const float fv = f32[p];
    if (!isfinite(fv)) atomicOr(nonfinite, 1);
    const float z = __fmul_rn(fv, fv), t = __fadd_rn(1.0f, z);
    const float rho1 = __fdiv_rn(1.0f, t), rho2 = -__fdiv_rn(1.0f, __fmul_rn(t, t));
    cterm[p] = (double)log1pf(z);
    double js = (double)rho1 + 2.0 * (double)rho2 * (double)z;
    if (js < 2.220446049250313e-16) js = 2.220446049250313e-16;
    js = sqrt(js);
    fs[p] = (double)(float)((double)fv * ((double)rho1 / js));
    const double f0d = f64[p];
    for (int j = 0; j < n; ++j) {
        double Jv = 0.0;
        if (mask[(size_t)p * C + cols[j + 1].cam]) {
            if (jac_mode == 0) Jv = (double)__fsub_rn(f32[(size_t)(j + 1) * m + p], fv) / dx[j];
            else Jv = (f64[(size_t)(j + 1) * m + p] - f0d) / dx[j];
        }
        Js[(size_t)j * m + p] = Jv * js;
    }
}

// one warp per output: the n(n+1)/2 entries of Js^T Js, the n entries of Js^T fs, the cost.
__global__ void __launch_bounds__(128)
k_ba_gram(const double* __restrict__ Js, const double* __restrict__ fs, const double* __restrict__ cterm,
          int m, int n, double* __restrict__ out /* A[n*n], g[n], cost */) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int n_pairs = n * (n + 1) / 2;
    if (w > n_pairs + n) return;
    const double* a; const double* b;
    int i = 0, j = 0;
    if (w < n_pairs) {
        int rem = w;
        while (rem >= n - i) { rem -= n - i; ++i; }
        j = i + rem;
        a = Js + (size_t)i * m; b = Js + (size_t)j * m;
    } else if (w < n_pairs + n) { i = w - n_pairs; a = Js + (size_t)i * m; b = fs; }
    else { a = cterm; b = nullptr; }
    double s = 0.0;
    for (int p = lane; p < m; p += 32) s += b ? a[p] * b[p] : a[p];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
        if (w < n_pairs) { out[(size_t)i * n + j] = s; out[(size_t)j * n + i] = s; }
        else if (w < n_pairs + n) out[(size_t)n * n + i] = s;
        else out[(size_t)n * n + n] = 0.5 * s;
    }
}

// trial point: cost only (loss_function(f_new, cost_only=True))
__global__ void __launch_bounds__(256)
k_ba_cost(const float* __restrict__ f32, const uint8_t* __restrict__ valid, int m, double* __restrict__ out, int* __restrict__ nonfinite) {
    __shared__ double part[8];
    double s = 0.0;
    for (int p = threadIdx.x; p < m; p += blockDim.x)
        if (valid[p]) {
            const float fv = f32[p];
            if (!isfinite(fv)) atomicOr(nonfinite, 1);
            s += (double)log1pf(__fmul_rn(fv, fv));
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += part[w];
        out[0] = 0.5 * tot;
    }
}

// ---------------------------------------------------------------------------------------------
// prefit: Levenberg-Marquardt over poses and points, Schur complement on the point blocks
// ---------------------------------------------------------------------------------------------
struct ViewJac { double e[2]; double Jc[2][6]; double Jp[2][3]; };

__device__ __forceinline__ void view_jacobian(const double* __restrict__ Rt, double fx, double fy, double cx, double cy,
                                              const double X[3], double uo, double vo, ViewJac& J) {
    const double rx = Rt[0] * X[0] + Rt[1] * X[1] + Rt[2] * X[2];
    const double ry = Rt[4] * X[0] + Rt[5] * X[1] + Rt[6] * X[2];
    const double rz = Rt[8] * X[0] + Rt[9] * X[1] + Rt[10] * X[2];
    const double x = rx + Rt[3], y = ry + Rt[7], z = rz + Rt[11];
    const double iz = 1.0 / z;
    J.e[0] = fx * x * iz + cx - uo;
    J.e[1] = fy * y * iz + cy - vo;
    const double du[3] = {fx * iz, 0.0, -fx * x * iz * iz};      // d u / d Xc
    const double dv[3] = {0.0, fy * iz, -fy * y * iz * iz};
    // Xc = Exp(w) (R X) + t + dt  ->  dXc/dw = -[R X]x , dXc/ddt = I
    J.Jc[0][0] = du[1] * (-rz) + du[2] * ry;  J.Jc[0][1] = du[0] * rz + du[2] * (-rx);  J.Jc[0][2] = du[0] * (-ry) + du[1] * rx;
    J.Jc[1][0] = dv[1] * (-rz) + dv[2] * ry;  J.Jc[1][1] = dv[0] * rz + dv[2] * (-rx);  J.Jc[1][2] = dv[0] * (-ry) + dv[1] * rx;
    for (int q = 0; q < 3; ++q) { J.Jc[0][3 + q] = du[q]; J.Jc[1][3 + q] = dv[q]; }
    for (int q = 0; q < 3; ++q) {
        J.Jp[0][q] = du[0] * Rt[q] + du[1] * Rt[4 + q] + du[2] * Rt[8 + q];
        J.Jp[1][q] = dv[0] * Rt[q] + dv[1] * Rt[4 + q] + dv[2] * Rt[8 + q];
    }
}

__device__ __forceinline__ bool inv_sym3(const double H[6], double Hi[6]) {   // 00 01 02 11 12 22
    const double c00 = H[3] * H[5] - H[4] * H[4], c01 = H[2] * H[4] - H[1] * H[5], c02 = H[1] * H[4] - H[2] * H[3];
    const double det = H[0] * c00 + H[1] * c01 + H[2] * c02;
    if (!(fabs(det) > 0.0)) return false;
    const double id = 1.0 / det;
    Hi[0] = c00 * id; Hi[1] = c01 * id; Hi[2] = c02 * id;
    Hi[3] = (H[0] * H[5] - H[2] * H[2]) * id; Hi[4] = (H[1] * H[2] - H[0] * H[4]) * id; Hi[5] = (H[0] * H[3] - H[1] * H[1]) * id;
    return true;
}
__device__ __forceinline__ void sym3_mul(const double Hi[6], const double v[3], double o[3]) {
    o[0] = Hi[0] * v[0] + Hi[1] * v[1] + Hi[2] * v[2];
    o[1] = Hi[1] * v[0] + Hi[3] * v[1] + Hi[4] * v[2];
    o[2] = Hi[2] * v[0] + Hi[4] * v[1] + Hi[5] * v[2];
}

// mode 0: accumulate the reduced camera system  S dc = -r  (+ undamped diagonal D, cost)
// mode 1: given dc, back-substitute dp and write X_new
// shared memory: S [n*n], r [n], D [n], cost [1]   (mode 0)
__global__ void __launch_bounds__(128)
k_sba(const CameraTables* __restrict__ tb, const double* __restrict__ Rt_all, const double* __restrict__ X,
      const double* __restrict__ obs, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ valid,
      int m, int C, double lambda, int mode, const double* __restrict__ dc, double* __restrict__ X_new,
      double* __restrict__ out /* S[n*n], r[n], D[n], cost */) {
    extern __shared__ double sh[];
    const int n = 6 * (C - 1);
    double* S = sh; double* r = S + (size_t)n * n; double* D = r + n; double* cost = D + n;
    if (mode == 0) {
        for (int i = threadIdx.x; i < n * n + 2 * n + 1; i += blockDim.x) sh[i] = 0.0;
        __syncthreads();
    }
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < m; p += gridDim.x * blockDim.x) {
        if (!valid[p]) continue;
        const double Xp[3] = {X[3 * p], X[3 * p + 1], X[3 * p + 2]};
        const uint8_t* mk = mask + (size_t)p * C;
        const double* o = obs + (size_t)p * C * 2;
        double Hpp[6] = {0, 0, 0, 0, 0, 0}, gp[3] = {0, 0, 0};
        double W[MOCAP_MAX_CAM][6][3];
        int cam_of[MOCAP_MAX_CAM];
        double my_cost = 0.0;
        int nv = 0, k = 0;
        for (int c = 0; c < C; ++c) {
            if (!mk[c]) continue;
            ViewJac J;
            view_jacobian(Rt_all + 12 * c, tb->fx[k], tb->fy[k], tb->cx[k], tb->cy[k], Xp, o[2 * c], o[2 * c + 1], J);
            ++k;
            my_cost += J.e[0] * J.e[0] + J.e[1] * J.e[1];
            Hpp[0] += J.Jp[0][0] * J.Jp[0][0] + J.Jp[1][0] * J.Jp[1][0];
            Hpp[1] += J.Jp[0][0] * J.Jp[0][1] + J.Jp[1][0] * J.Jp[1][1];
            Hpp[2] += J.Jp[0][0] * J.Jp[0][2] + J.Jp[1][0] * J.Jp[1][2];
            Hpp[3] += J.Jp[0][1] * J.Jp[0][1] + J.Jp[1][1] * J.Jp[1][1];
            Hpp[4] += J.Jp[0][1] * J.Jp[0][2] + J.Jp[1][1] * J.Jp[1][2];
            Hpp[5] += J.Jp[0][2] * J.Jp[0][2] + J.Jp[1][2] * J.Jp[1][2];
            for (int q = 0; q < 3; ++q) gp[q] += J.Jp[0][q] * J.e[0] + J.Jp[1][q] * J.e[1];
            if (c == 0) continue;                                   // camera 0 is pinned (helpers.py:250-253)
            cam_of[nv] = c;
            for (int a = 0; a < 6; ++a)
                for (int q = 0; q < 3; ++q) W[nv][a][q] = J.Jc[0][a] * J.Jp[0][q] + J.Jc[1][a] * J.Jp[1][q];
            if (mode == 0) {
                const int base = 6 * (c - 1);
                for (int a = 0; a < 6; ++a) {
                    for (int b = 0; b < 6; ++b)
                        atomicAdd(&S[(size_t)(base + a) * n + base + b], J.Jc[0][a] * J.Jc[0][b] + J.Jc[1][a] * J.Jc[1][b]);
                    atomicAdd(&r[base + a], J.Jc[0][a] * J.e[0] + J.Jc[1][a] * J.e[1]);
                    atomicAdd(&D[base + a], J.Jc[0][a] * J.Jc[0][a] + J.Jc[1][a] * J.Jc[1][a]);
                }
            }
            ++nv;
        }
        double Hd[6] = {Hpp[0] * (1.0 + lambda), Hpp[1], Hpp[2], Hpp[3] * (1.0 + lambda), Hpp[4], Hpp[5] * (1.0 + lambda)};
        double Hi[6];
        if (!inv_sym3(Hd, Hi)) { Hi[0] = Hi[3] = Hi[5] = 0.0; Hi[1] = Hi[2] = Hi[4] = 0.0; }
        if (mode == 0) {
            atomicAdd(cost, 0.5 * my_cost);
            double Hig[3];
            sym3_mul(Hi, gp, Hig);
            for (int a = 0; a < nv; ++a) {
                const int ba = 6 * (cam_of[a] - 1);
                double WH[6][3];                                      // W_a Hpp^-1
                for (int i = 0; i < 6; ++i) {
                    const double v[3] = {W[a][i][0], W[a][i][1], W[a][i][2]};
                    sym3_mul(Hi, v, WH[i]);
                    atomicAdd(&r[ba + i], -(v[0] * Hig[0] + v[1] * Hig[1] + v[2] * Hig[2]));
                }
                for (int b = 0; b < nv; ++b) {
                    const int bb = 6 * (cam_of[b] - 1);
                    for (int i = 0; i < 6; ++i)
                        for (int j = 0; j < 6; ++j)
                            atomicAdd(&S[(size_t)(ba + i) * n + bb + j],
                                      -(WH[i][0] * W[b][j][0] + WH[i][1] * W[b][j][1] + WH[i][2] * W[b][j][2]));
                }
            }
        } else {
            double rhs[3] = {gp[0], gp[1], gp[2]};                   // dp = -Hpp^-1 (gp + W^T dc)
            for (int a = 0; a < nv; ++a) {
                const double* d = dc + 6 * (cam_of[a] - 1);
                for (int q = 0; q < 3; ++q)
                    for (int i = 0; i < 6; ++i) rhs[q] += W[a][i][q] * d[i];
            }
            double dp[3];
            sym3_mul(Hi, rhs, dp);
            X_new[3 * p] = Xp[0] - dp[0]; X_new[3 * p + 1] = Xp[1] - dp[1]; X_new[3 * p + 2] = Xp[2] - dp[2];
        }
    }
    if (mode == 0) {
        __syncthreads();
        for (int i = threadIdx.x; i < n * n + 2 * n + 1; i += blockDim.x)
            if (sh[i] != 0.0) atomicAdd(&out[i], sh[i]);
    }
}

// 0.5 * sum of squared pixel residuals of (poses, X)
__global__ void __launch_bounds__(256)
k_sba_cost(const CameraTables* __restrict__ tb, const double* __restrict__ Rt_all, const double* __restrict__ X,
           const double* __restrict__ obs, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ valid,
           int m, int C, double* __restrict__ out) {
    __shared__ double part[8];
    double s = 0.0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < m; p += gridDim.x * blockDim.x) {
        if (!valid[p]) continue;
        const double Xp[3] = {X[3 * p], X[3 * p + 1], X[3 * p + 2]};
        int k = 0;
        for (int c = 0; c < C; ++c)
            if (mask[(size_t)p * C + c]) {
                const double* Rt = Rt_all + 12 * c;
                const double x = Rt[0] * Xp[0] + Rt[1] * Xp[1] + Rt[2] * Xp[2] + Rt[3];
                const double y = Rt[4] * Xp[0] + Rt[5] * Xp[1] + Rt[6] * Xp[2] + Rt[7];
                const double z = Rt[8] * Xp[0] + Rt[9] * Xp[1] + Rt[10] * Xp[2] + Rt[11];
                const double eu = tb->fx[k] * x / z + tb->cx[k] - obs[((size_t)p * C + c) * 2];
                const double ev = tb->fy[k] * y / z + tb->cy[k] - obs[((size_t)p * C + c) * 2 + 1];
                s += eu * eu + ev * ev;
                ++k;
            }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double tot = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += part[w];
        atomicAdd(out, 0.5 * tot);
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
namespace {

struct DeviceBA : trf::Problem {
    mocap_ctx* ctx;
    int m, C, jac_mode;
    std::vector<int> live_idx;
    // device
    double* d_obs; uint8_t* d_mask; uint8_t* d_valid; double* d_baseRt; BAColumn* d_cols; double* d_dx;
    float* d_f32; double* d_f64; double* d_Js; double* d_fs; double* d_cterm; double* d_out; int* d_flag;
    double* d_X; double* d_Xnew; double* d_dc; double* d_sba;
    int n_valid;
    int status;     // first CUDA failure

    static void poses_from_x(const double* x, int C, std::vector<double>& Rt) {
        Rt.assign((size_t)C * 12, 0.0);
        Rt[0] = Rt[5] = Rt[10] = 1.0;                              // camera 0: (I, 0), helpers.py:250-253
        for (int c = 1; c < C; ++c) {
            const double* q = x + 1 + 7 * (c - 1);
            double R[9];
            trf::rotvec_to_matrix(q + 1, R);
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) Rt[(size_t)c * 12 + 4 * i + j] = R[3 * i + j];
                Rt[(size_t)c * 12 + 4 * i + 3] = q[4 + i];
            }
        }
    }

    int eval(const double* x, bool with_columns) {
        const int n = n_live;
        std::vector<double> Rt;
        poses_from_x(x, C, Rt);
        std::vector<BAColumn> cols(1 + (with_columns ? n : 0));
        std::vector<double> dx(n > 0 ? n : 1, 1.0);
        cols[0].cam = -1; cols[0].pad = 0;
        memset(cols[0].Rt, 0, sizeof(cols[0].Rt));
        if (with_columns) {
            std::vector<double> xp(x, x + n_full), Rtp;
            for (int j = 0; j < n; ++j) {
                const int idx = live_idx[j];
                const double x0 = x[idx];
                // scipy _compute_absolute_step: sqrt(eps) * sign(x0) * max(1, |x0|), sign(0) = +1
                const double h = 1.4901161193847656e-08 * (x0 >= 0 ? 1.0 : -1.0) * fmax(1.0, fabs(x0));
                xp[idx] = x0 + h;
                dx[j] = xp[idx] - x0;
                const int cam = 1 + (idx - 1) / 7;
                poses_from_x(xp.data(), C, Rtp);
                cols[j + 1].cam = cam; cols[j + 1].pad = 0;
                memcpy(cols[j + 1].Rt, Rtp.data() + (size_t)cam * 12, 12 * sizeof(double));
                xp[idx] = x0;
            }
        }
        cudaStream_t st = ctx->stream;
        CUDA_TRY(ctx, cudaMemcpyAsync(d_baseRt, Rt.data(), Rt.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_cols, cols.data(), cols.size() * sizeof(BAColumn), cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_dx, dx.data(), dx.size() * sizeof(double), cudaMemcpyHostToDevice, st));
        CUDA_TRY(ctx, cudaMemsetAsync(d_flag, 0, sizeof(int), st));
        const long long total = (long long)m * (long long)cols.size();
        k_ba_eval<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(ctx->d_tables, d_baseRt, d_cols, (int)cols.size(), d_obs, d_mask,
                                                                   d_valid, m, C, d_f32, d_f64, d_X);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        // the pageable host vectors above are consumed by the copies before this returns
        CUDA_TRY(ctx, cudaStreamSynchronize(st));
        return MOCAP_OK;
    }

    int linearize(const double* x, double* A, double* g, double* cost, int* finite) override {
        const int n = n_live;
        int st = eval(x, true);
        if (st) return st;
        cudaStream_t s = ctx->stream;
        k_ba_rows<<<(m + 127) / 128, 128, 0, s>>>(d_f32, d_f64, d_cols, d_dx, d_mask, d_valid, m, C, n, jac_mode, d_Js, d_fs, d_cterm, d_flag);
        CUDA_TRY(ctx, cudaGetLastError());
        const int warps = n * (n + 1) / 2 + n + 1;
        k_ba_gram<<<(warps * 32 + 127) / 128, 128, 0, s>>>(d_Js, d_fs, d_cterm, m, n, d_out);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 2;
        std::vector<double> out((size_t)n * n + n + 1);
        int flag = 0;
        CUDA_TRY(ctx, cudaMemcpyAsync(out.data(), d_out, out.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        memcpy(A, out.data(), (size_t)n * n * sizeof(double));
        memcpy(g, out.data() + (size_t)n * n, n * sizeof(double));
        *cost = out[(size_t)n * n + n];
        *finite = flag ? 0 : 1;
        return MOCAP_OK;
    }

    int trial_cost(const double* x, double* cost, int* finite) override {
        int st = eval(x, false);
        if (st) return st;
        cudaStream_t s = ctx->stream;
        k_ba_cost<<<1, 256, 0, s>>>(d_f32, d_valid, m, d_out, d_flag);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        int flag = 0;
        CUDA_TRY(ctx, cudaMemcpyAsync(cost, d_out, sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        *finite = flag ? 0 : 1;
        return MOCAP_OK;
    }
};

// dense Cholesky solve of the reduced camera system (n <= 90), in place.  false: not positive definite
bool cholesky_solve(int n, std::vector<double>& A, std::vector<double>& b) {
    for (int j = 0; j < n; ++j) {
        double d = A[(size_t)j * n + j];
        for (int k = 0; k < j; ++k) d -= A[(size_t)j * n + k] * A[(size_t)j * n + k];
        if (!(d > 0.0)) return false;
        d = sqrt(d);
        A[(size_t)j * n + j] = d;
        for (int i = j + 1; i < n; ++i) {
            double s = A[(size_t)i * n + j];
            for (int k = 0; k < j; ++k) s -= A[(size_t)i * n + k] * A[(size_t)j * n + k];
            A[(size_t)i * n + j] = s / d;
        }
    }
    for (int i = 0; i < n; ++i) {
        double s = b[i];
        for (int k = 0; k < i; ++k) s -= A[(size_t)i * n + k] * b[k];
        b[i] = s / A[(size_t)i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
        double s = b[i];
        for (int k = i + 1; k < n; ++k) s -= A[(size_t)k * n + i] * b[k];
        b[i] = s / A[(size_t)i * n + i];
    }
    return true;
}

void exp_so3(const double w[3], double E[9]) {
    const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    double a, b;
    if (th < 1e-8) { a = 1.0 - th * th / 6.0; b = 0.5 - th * th / 24.0; }
    else { a = sin(th) / th; b = (1.0 - cos(th)) / (th * th); }
    const double K[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
    double K2[9];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += K[3 * i + k] * K[3 * k + j]; K2[3 * i + j] = s; }
    for (int i = 0; i < 9; ++i) E[i] = (i % 4 == 0 ? 1.0 : 0.0) + a * K[i] + b * K2[i];
}

// Levenberg-Marquardt over poses + points.  Rt: [C][12] in/out; *taken: whether a step was accepted.
int prefit(DeviceBA& P, std::vector<double>& Rt, int max_iter, mocap_ba_report* rep, bool* taken) {
    mocap_ctx* ctx = P.ctx;
    cudaStream_t s = ctx->stream;
    const int C = P.C, m = P.m, n = 6 * (C - 1);
    const size_t n_out = (size_t)n * n + 2 * n + 1;
    const size_t smem = n_out * sizeof(double);
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_sba, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = (m + 127) / 128;
    if (grid > 2 * ctx->num_sms) grid = 2 * ctx->num_sms;
    std::vector<double> out(n_out), Rt_new, S, rhs;
    double lambda = 1e-3, cost = 0.0;
    auto upload = [&](const std::vector<double>& r) { return cudaMemcpyAsync(P.d_baseRt, r.data(), r.size() * sizeof(double), cudaMemcpyHostToDevice, s); };
    auto eval_cost = [&](const double* dX, double* c) -> int {
        CUDA_TRY(ctx, cudaMemsetAsync(P.d_sba, 0, sizeof(double), s));
        k_sba_cost<<<grid, 256, 0, s>>>(ctx->d_tables, P.d_baseRt, dX, P.d_obs, P.d_mask, P.d_valid, m, C, P.d_sba);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        CUDA_TRY(ctx, cudaMemcpyAsync(c, P.d_sba, sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        return MOCAP_OK;
    };
    CUDA_TRY(ctx, upload(Rt));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    int st = eval_cost(P.d_X, &cost);
    if (st) return st;
    rep->prefit_cost_initial = cost;
    *taken = false;
    int it = 0;
    for (; it < max_iter; ++it) {
        CUDA_TRY(ctx, cudaMemsetAsync(P.d_sba, 0, n_out * sizeof(double), s));
        k_sba<<<grid, 128, smem, s>>>(ctx->d_tables, P.d_baseRt, P.d_X, P.d_obs, P.d_mask, P.d_valid, m, C, lambda, 0, nullptr, nullptr, P.d_sba);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        CUDA_TRY(ctx, cudaMemcpyAsync(out.data(), P.d_sba, n_out * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        S.assign(out.begin(), out.begin() + (size_t)n * n);
        rhs.assign(n, 0.0);
        for (int i = 0; i < n; ++i) { S[(size_t)i * n + i] += lambda * out[(size_t)n * n + n + i]; rhs[i] = -out[(size_t)n * n + i]; }
        // a parameter with a zero diagonal belongs to a camera that sees no point: pinned, its step is 0 (ba_device.cuh)
        for (int i = 0; i < n; ++i)
            if (out[(size_t)n * n + n + i] == 0.0) {
                for (int j = 0; j < n; ++j) S[(size_t)i * n + j] = S[(size_t)j * n + i] = 0.0;
                S[(size_t)i * n + i] = 1.0; rhs[i] = 0.0;
            }
        if (!cholesky_solve(n, S, rhs)) { lambda *= 10.0; if (lambda > 1e12) { ++it; break; } continue; }
        // candidate poses: R' = Exp(dw) R, t' = t + dt
        Rt_new = Rt;
        for (int c = 1; c < C; ++c) {
            const double* d = rhs.data() + 6 * (c - 1);
            double E[9];
            exp_so3(d, E);
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) {
                    double v = 0;
                    for (int k = 0; k < 3; ++k) v += E[3 * i + k] * Rt[(size_t)c * 12 + 4 * k + j];
                    Rt_new[(size_t)c * 12 + 4 * i + j] = v;
                }
                Rt_new[(size_t)c * 12 + 4 * i + 3] = Rt[(size_t)c * 12 + 4 * i + 3] + d[3 + i];
            }
        }
        CUDA_TRY(ctx, cudaMemcpyAsync(P.d_dc, rhs.data(), n * sizeof(double), cudaMemcpyHostToDevice, s));
        k_sba<<<grid, 128, smem, s>>>(ctx->d_tables, P.d_baseRt, P.d_X, P.d_obs, P.d_mask, P.d_valid, m, C, lambda, 1, P.d_dc, P.d_Xnew, P.d_sba);
        CUDA_TRY(ctx, cudaGetLastError());
        ctx->launches += 1;
        CUDA_TRY(ctx, upload(Rt_new));
        double cost_new = 0.0;
        st = eval_cost(P.d_Xnew, &cost_new);
        if (st) return st;
        if (cost_new < cost && isfinite(cost_new)) {
            const double rel = (cost - cost_new) / fmax(cost, 1e-300);
            Rt = Rt_new;
            double* tmp = P.d_X; P.d_X = P.d_Xnew; P.d_Xnew = tmp;
            cost = cost_new;
            *taken = true;
            lambda = fmax(lambda * 0.3, 1e-12);
            if (rel < BA_PREFIT_REL_STOP) { ++it; break; }
        } else {
            CUDA_TRY(ctx, upload(Rt));                       // back to the accepted poses
            CUDA_TRY(ctx, cudaStreamSynchronize(s));
            lambda *= 10.0;
            if (lambda > 1e12) { ++it; break; }
        }
    }
    CUDA_TRY(ctx, upload(Rt));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    rep->prefit_cost_final = cost;
    rep->prefit_iterations = it;
    return MOCAP_OK;
}

int setup_problem(mocap_ctx* ctx, DeviceBA& P, const double* obs, const uint8_t* mask, int n_points, int jac_mode) {
    const int C = ctx->cfg.n_cam, m = n_points;
    P.ctx = ctx; P.m = m; P.C = C; P.jac_mode = jac_mode;
    P.n_full = 1 + 7 * (C - 1);
    P.live_idx.clear();
    for (int c = 1; c < C; ++c) for (int q = 1; q < 7; ++q) P.live_idx.push_back(1 + 7 * (c - 1) + q);
    P.n_live = (int)P.live_idx.size();
    P.live = P.live_idx.data();
    const int n = P.n_live;
    std::vector<uint8_t> valid(m);
    P.n_valid = 0;
    for (int f = 0; f < m; ++f) {
        int nv = 0;
        for (int c = 0; c < C; ++c) nv += mask[(size_t)f * C + c] ? 1 : 0;
        valid[f] = nv > 1;                                      // helpers.py:207-208,222-223: <= 1 view is skipped
        P.n_valid += valid[f];
    }
    const size_t ncol = (size_t)n + 1;
    int st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
        P.d_obs = L.take<double>((size_t)m * C * 2); P.d_mask = L.take<uint8_t>((size_t)m * C); P.d_valid = L.take<uint8_t>(m);
        P.d_baseRt = L.take<double>((size_t)C * 12); P.d_cols = L.take<BAColumn>(ncol); P.d_dx = L.take<double>(ncol);
        P.d_f32 = L.take<float>(ncol * m); P.d_f64 = L.take<double>(ncol * m); P.d_Js = L.take<double>((size_t)(n > 0 ? n : 1) * m);
        P.d_fs = L.take<double>(m); P.d_cterm = L.take<double>(m); P.d_out = L.take<double>((size_t)n * n + 2 * n + 8);
        P.d_flag = L.take<int>(64); P.d_X = L.take<double>((size_t)m * 3); P.d_Xnew = L.take<double>((size_t)m * 3);
        P.d_dc = L.take<double>((size_t)n + 1); P.d_sba = L.take<double>((size_t)n * n + 2 * n + 8);
    });
    if (st) return st;
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(P.d_obs, obs, (size_t)m * C * 2 * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(P.d_mask, mask, (size_t)m * C, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(P.d_valid, valid.data(), (size_t)m, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemsetAsync(P.d_f32, 0, ncol * m * 4, s));
    CUDA_TRY(ctx, cudaMemsetAsync(P.d_f64, 0, ncol * m * 8, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));                   // `valid` is a pageable temporary
    return MOCAP_OK;
}

void x_from_poses(const mocap_ctx* ctx, const double* R, const double* t, int C, std::vector<double>& x) {
    x.assign(1 + 7 * (C - 1), 0.0);
    x[0] = ctx->h_tables.Kmat[0][0];
    for (int c = 1; c < C; ++c) {
        double* q = x.data() + 1 + 7 * (c - 1);
        q[0] = ctx->h_tables.Kmat[c - 1][0];                    // helpers.py:281-282: K[i], i enumerating poses[1:]
        trf::matrix_to_rotvec(R + 9 * c, q + 1);
        q[4] = t[3 * c]; q[5] = t[3 * c + 1]; q[6] = t[3 * c + 2];
    }
}

}  // namespace

extern "C" {

void mocap_ba_default_options(mocap_ba_options* opt) {
    opt->ftol = 1e-2; opt->xtol = 1e-8; opt->gtol = 1e-8; opt->max_nfev = 0;
    opt->jacobian = 1; opt->prefit = 1; opt->prefit_max_iter = 50; opt->engine = 0;
}

int mocap_ba_residuals_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points,
                            const double* R, const double* t, float* r, uint8_t* valid, int* n_valid) {
    if (!ctx) return MOCAP_EINVAL;
    if (!obs || !mask || !R || !t || !r || !valid || n_points <= 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_ba_residuals_host: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    DeviceBA P;
    int st = setup_problem(ctx, P, obs, mask, n_points, 1);
    if (st) return st;
    std::vector<double> x;
    x_from_poses(ctx, R, t, P.C, x);
    // exact poses as given (no rotvec round trip): upload R|t directly as the base and evaluate column 0
    std::vector<double> Rt((size_t)P.C * 12);
    for (int c = 0; c < P.C; ++c)
        for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) Rt[(size_t)c * 12 + 4 * i + j] = R[9 * c + 3 * i + j]; Rt[(size_t)c * 12 + 4 * i + 3] = t[3 * c + i]; }
    BAColumn c0; c0.cam = -1; c0.pad = 0; memset(c0.Rt, 0, sizeof(c0.Rt));
    cudaStream_t s = ctx->stream;
    CUDA_TRY(ctx, cudaMemcpyAsync(P.d_baseRt, Rt.data(), Rt.size() * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(P.d_cols, &c0, sizeof(c0), cudaMemcpyHostToDevice, s));
    k_ba_eval<<<(n_points + 127) / 128, 128, 0, s>>>(ctx->d_tables, P.d_baseRt, P.d_cols, 1, P.d_obs, P.d_mask, P.d_valid, n_points, P.C,
                                                     P.d_f32, P.d_f64, P.d_X);
    CUDA_TRY(ctx, cudaGetLastError());
    ctx->launches += 1;
    CUDA_TRY(ctx, cudaMemcpyAsync(r, P.d_f32, (size_t)n_points * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(valid, P.d_valid, (size_t)n_points, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    if (n_valid) *n_valid = P.n_valid;
    return MOCAP_OK;
}

int mocap_bundle_adjust_host(mocap_ctx* ctx, const double* obs, const uint8_t* mask, int n_points, double* R, double* t,
                             const mocap_ba_options* opt_in, mocap_ba_report* report) {
    if (!ctx) return MOCAP_EINVAL;
    if (!obs || !mask || !R || !t || n_points <= 0) return mocap_fail(ctx, MOCAP_EINVAL, "mocap_bundle_adjust_host: bad argument");
    if (!ctx->cameras_set) return mocap_fail(ctx, MOCAP_ESTATE, "mocap_set_cameras has not been called (intrinsics are needed)");
    if (ctx->cfg.n_cam < 2) return mocap_fail(ctx, MOCAP_EINVAL, "bundle adjustment needs at least two cameras");
    CUDA_TRY(ctx, cudaSetDevice(ctx->cfg.device));
    mocap_ba_options opt;
    if (opt_in) opt = *opt_in; else mocap_ba_default_options(&opt);
    if (opt.engine == 0) {
        // default: copy in, ONE launch of the device-resident solve (mocap_bundle_adjust_dev), copy out
        const int C = ctx->cfg.n_cam;
        double *d_obs, *d_R, *d_t;
        uint8_t* d_mask;
        mocap_ba_report* d_rep;
        int st = grow_carved(ctx, ctx->scratch, Drain::stream, [&](Layout& L) {
            d_obs = L.take<double>((size_t)n_points * C * 2); d_mask = L.take<uint8_t>((size_t)n_points * C);
            d_R = L.take<double>((size_t)C * 9); d_t = L.take<double>((size_t)C * 3); d_rep = L.take<mocap_ba_report>(1);
        });
        if (st) return st;
        cudaStream_t s = ctx->stream;
        CUDA_TRY(ctx, cudaMemcpyAsync(d_obs, obs, (size_t)n_points * C * 2 * 8, cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_mask, mask, (size_t)n_points * C, cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_R, R, (size_t)C * 9 * 8, cudaMemcpyHostToDevice, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(d_t, t, (size_t)C * 3 * 8, cudaMemcpyHostToDevice, s));
        st = mocap_bundle_adjust_dev(ctx, d_obs, d_mask, n_points, nullptr, d_R, d_t, &opt, d_rep);
        if (st) return st;
        mocap_ba_report rep;
        CUDA_TRY(ctx, cudaMemcpyAsync(R, d_R, (size_t)C * 9 * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(t, d_t, (size_t)C * 3 * 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaMemcpyAsync(&rep, d_rep, sizeof(rep), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(ctx, cudaStreamSynchronize(s));
        if (rep.status == -3) return mocap_fail(ctx, MOCAP_EINVAL, "no point is seen by two cameras");
        if (report) *report = rep;
        return MOCAP_OK;
    }
    // engine 1: the host-stepped solve (optimiser control in trf_core.h, one launch per phase): kept as the
    // cross-check of the device-resident solve
    mocap_ba_report rep;
    memset(&rep, 0, sizeof(rep));
    const uint64_t launches0 = ctx->launches;
    DeviceBA P;
    int st = setup_problem(ctx, P, obs, mask, n_points, opt.jacobian ? 1 : 0);
    if (st) return st;
    if (P.n_valid == 0) return mocap_fail(ctx, MOCAP_EINVAL, "no point is seen by two cameras");
    const int C = P.C;
    std::vector<double> x;
    x_from_poses(ctx, R, t, C, x);                              // helpers.py:278-285

    bool taken = false;
    if (opt.prefit) {
        // start from the DLT points of the initial poses (k_ba_eval writes them to d_X)
        st = P.eval(x.data(), false);
        if (st) return st;
        std::vector<double> Rt;
        DeviceBA::poses_from_x(x.data(), C, Rt);
        st = prefit(P, Rt, opt.prefit_max_iter > 0 ? opt.prefit_max_iter : 50, &rep, &taken);
        if (st) return st;
        for (int c = 1; c < C; ++c) {
            double Rc[9];
            for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rc[3 * i + j] = Rt[(size_t)c * 12 + 4 * i + j];
            double* q = x.data() + 1 + 7 * (c - 1);
            trf::matrix_to_rotvec(Rc, q + 1);
            q[4] = Rt[(size_t)c * 12 + 3]; q[5] = Rt[(size_t)c * 12 + 7]; q[6] = Rt[(size_t)c * 12 + 11];
        }
    }

    // after a prefit that took a step the start is already close: begin the polish with a trust region of
    // BA_POLISH_RADIUS (rad / pose units) instead of scipy's ||x0|| (~ the focal length), which would burn its evaluations
    // shrinking.  A prefit that took no step left the start where it was: the polish starts as scipy does
    trf::Options topt{opt.ftol, opt.xtol, opt.gtol, opt.max_nfev, taken ? BA_POLISH_RADIUS : 0.0};
    trf::Report trep{};
    st = trf::minimize(P, x.data(), topt, trep);
    if (st) return st;
    if (opt.prefit) {
        // cost_initial must describe the caller's start, not the prefit result
        std::vector<double> x0;
        x_from_poses(ctx, R, t, C, x0);
        double c0 = 0.0; int fin = 1;
        st = P.trial_cost(x0.data(), &c0, &fin);
        if (st) return st;
        trep.cost_initial = c0;
    }
    std::vector<double> Rt;
    DeviceBA::poses_from_x(x.data(), C, Rt);                   // helpers.py:290
    for (int c = 0; c < C; ++c)
        for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) R[9 * c + 3 * i + j] = Rt[(size_t)c * 12 + 4 * i + j]; t[3 * c + i] = Rt[(size_t)c * 12 + 4 * i + 3]; }
    rep.cost_initial = trep.cost_initial; rep.cost_final = trep.cost_final; rep.optimality = trep.optimality;
    rep.n_iterations = trep.n_iterations; rep.n_fev = trep.n_fev; rep.status = trep.status; rep.n_residuals = P.n_valid;
    rep.n_launches = (int)(ctx->launches - launches0);
    if (report) *report = rep;
    return MOCAP_OK;
}

}  // extern "C"

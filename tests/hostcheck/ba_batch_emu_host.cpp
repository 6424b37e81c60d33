// Test-only: a BATCHED launch of the device-resident bundle adjustment (csrc/ba_device.cuh: BABatch, one sub-grid
// of CTAs per problem, each with its own barrier words and workspace) run unchanged on the host through the SIMT
// emulation in simt_emu.h, so that every problem of a batch can be compared bit for bit with the single-solve hook
// (ba_dev_emu_host.cpp) on a grid of the same size.  NOT part of libmocap_b200.so and never used by the product path.
#include "simt_emu.h"
#include "../../low-cost-mocap_b200/csrc/ba_device.cuh"
#include "../../low-cost-mocap_b200/csrc/camera_tables.h"

// K problems sharing the cameras K_cam [C][9] and the options; problem k: obs[k] [m[k]][C][2], mask[k] [m[k]][C],
// R[k] [C][9] / t[k] [C][3] in-out (its own starting poses), on ctas[k] CTAs of n_threads threads; the camera tables
// are built from problem 0's poses, as a context's are from its mocap_set_cameras.  report[k] [13] as hc_ba_solve_dev
extern "C" int hc_ba_solve_batch(int K, const double* const* obs, const uint8_t* const* mask, const int* m, int C, const double* K_cam,
                                 double* const* R, double* const* t, double ftol, int max_nfev, int jac_mode, int prefit,
                                 int prefit_max_iter, const int* ctas, int n_threads, double* const* report) {
    if (K < 1 || K > MOCAP_BA_MAX_BATCH) return -1;
    static CameraTables T;
    memset(&T, 0, sizeof(T));
    build_camera_tables(T, C, K_cam, R[0], t[0]);
    const int n = 6 * (C - 1), npair = n * (n + 1) / 2, pstride = npair + 2 * n + 8;
    std::vector<std::vector<double>> X(K), Xnew(K), part(K), fin(K), cpart(K);
    std::vector<std::vector<uint8_t>> valid(K);
    std::vector<unsigned> bars(2 * K, 0u);
    std::vector<mocap_ba_report> rep(K);
    BABatch B;
    memset(&B, 0, sizeof(B));
    B.n = K;
    int G = 0;
    for (int k = 0; k < K; ++k) {
        const size_t mk = m[k] > 0 ? (size_t)m[k] : 1;
        X[k].resize(mk * 3); Xnew[k].resize(mk * 3); valid[k].resize(mk);
        part[k].resize((size_t)ctas[k] * pstride); fin[k].resize(pstride); cpart[k].resize((size_t)2 * ctas[k] * 4);
        memset(&rep[k], 0, sizeof(mocap_ba_report));
        BAParams& P = B.p[k];
        P.tb = &T; P.obs = obs[k]; P.mask = mask[k]; P.m_dev = nullptr; P.m_max = (int)mk; P.C = C; P.R = R[k]; P.t = t[k];
        P.ftol = ftol; P.xtol = 1e-8; P.gtol = 1e-8; P.max_nfev = max_nfev; P.jac_mode = jac_mode; P.prefit = prefit;
        P.prefit_max_iter = prefit_max_iter;
        P.X = X[k].data(); P.Xnew = Xnew[k].data(); P.valid = valid[k].data(); P.part = part[k].data(); P.pstride = pstride;
        P.fin = fin[k].data(); P.cpart = cpart[k].data(); P.bar = &bars[2 * k]; P.report = &rep[k];
        P.cta0 = G; P.ncta = ctas[k];
        G += ctas[k];
    }
    // m[k] == 0: a problem without points, read through a device-style count of 0
    static int32_t zero = 0;
    for (int k = 0; k < K; ++k) if (m[k] <= 0) B.p[k].m_dev = &zero;
    const size_t smem = ba_smem_bytes(C, n_threads);
    std::vector<std::vector<unsigned char>> sm(G, std::vector<unsigned char>(smem + 16));
    simt::launch_grid(G, n_threads, [&] {
        unsigned char* base = sm[blockIdx.x].data();
        base += (16 - ((uintptr_t)base & 15)) & 15;
        ba_solve_body(B.p[ba_problem_of(B)], B.p[0], base);
    });
    for (int k = 0; k < K; ++k) {
        const mocap_ba_report& r = rep[k];
        double* o = report[k];
        o[0] = r.cost_initial; o[1] = r.cost_final; o[2] = r.optimality; o[3] = r.n_iterations; o[4] = r.n_fev; o[5] = r.status;
        o[6] = r.n_residuals; o[7] = r.prefit_cost_initial; o[8] = r.prefit_cost_final; o[9] = r.prefit_iterations; o[10] = (double)smem;
        o[11] = r.n_tr_solves; o[12] = r.n_tr_newton;
    }
    return 0;
}

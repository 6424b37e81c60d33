// Test-only: the building blocks of S4's prefit and parameterisation (csrc/ba_device.cuh, csrc/trf_core.h) as plain
// host functions, so that tests/test_ba_prefit_on_host.py can hold each of them to scipy and to complex-step
// derivatives.  NOT part of libmocap_b200.so.
#include "simt_emu.h"
#include "../../low-cost-mocap_b200/csrc/ba_device.cuh"
#include "../../low-cost-mocap_b200/csrc/trf_core.h"

extern "C" {
// Rt [12] row-major [R|t], K4 = fx fy cx cy, X [3], uv [2] -> out [2 + 12 + 6]: e, Jc (2 x 6), Jp (2 x 3)
void hc_ba_view_jacobian(const double* Rt, const double* K4, const double* X, const double* uv, double* out) {
    BAViewJac J;
    ba_view_jacobian(Rt, K4[0], K4[1], K4[2], K4[3], X, uv[0], uv[1], J);
    out[0] = J.e[0]; out[1] = J.e[1];
    for (int r = 0; r < 2; ++r) for (int a = 0; a < 6; ++a) out[2 + 6 * r + a] = J.Jc[r][a];
    for (int r = 0; r < 2; ++r) for (int a = 0; a < 3; ++a) out[14 + 3 * r + a] = J.Jp[r][a];
}
void hc_ba_exp_so3(const double* w, double* E) { ba_exp_so3(w, E); }
void hc_ba_rotvec_to_matrix(const double* rv, double* R) { ba_rotvec_to_matrix(rv, R); }
void hc_ba_matrix_to_rotvec(const double* R, double* rv) { ba_matrix_to_rotvec(R, rv); }
void hc_trf_rotvec_to_matrix(const double* rv, double* R) { trf::rotvec_to_matrix(rv, R); }
void hc_trf_matrix_to_rotvec(const double* R, double* rv) { trf::matrix_to_rotvec(R, rv); }
}

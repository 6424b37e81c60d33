"""S4's Levenberg-Marquardt prefit held to a float64 model written from the algorithm (tests/ba_prefit_util.py), on a
machine without a GPU.

* The building blocks of csrc/ba_device.cuh and csrc/trf_core.h (view Jacobian, Exp, rotation-vector conversions)
  against complex-step derivatives and scipy.
* The device engine's solve (k_ba_solve's body, run unchanged on the host through the SIMT emulation of
  tests/hostcheck/simt_emu.h) against the model, iteration by iteration: `prefit_max_iter = k` with `max_nfev = 1`
  returns the poses after k prefit iterations (the polish evaluates once and takes no step).
* A camera that sees no point: it is held where it is, and the others are fitted as if it were not in the rig."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from tests import ba_prefit_util as bu
from tests import hostbuild
from tests.hostbuild import ptr
from tests.util import ROOT, synth

KEYS = ["cost_initial", "cost_final", "optimality", "n_iterations", "n_fev", "status", "n_residuals", "prefit_cost_initial",
        "prefit_cost_final", "prefit_iterations", "smem", "n_tr_solves", "n_tr_newton"]


@pytest.fixture(scope="module")
def libs():
    return hostbuild.load("ba_dev_emu"), hostbuild.load("ba_parts")


def solve(emu, obs, mask, K, R, t, prefit_max_iter=50, max_nfev=1, n_ctas=2, n_threads=64, prefit=True):
    """The device engine on the host.  K: one 3x3 matrix or [C, 3, 3] (K[k] for the k-th present view)."""
    C = mask.shape[1]
    obs = np.ascontiguousarray(obs, np.float64); mask = np.ascontiguousarray(mask, np.uint8)
    K = np.asarray(K, np.float64)
    Ks = np.ascontiguousarray(np.stack([K] * C) if K.ndim == 2 else K)
    R = np.ascontiguousarray(np.array(R, np.float64)); t = np.ascontiguousarray(np.array(t, np.float64).reshape(C, 3))
    rep = np.zeros(13)
    assert emu.hc_ba_solve_dev(ptr(obs), ptr(mask), obs.shape[0], C, ptr(Ks), ptr(R), ptr(t), 1e-2, max_nfev, 1, int(prefit),
                               prefit_max_iter, n_ctas, n_threads, ptr(rep)) == 0
    return R, t, dict(zip(KEYS, rep))


def tracks(C, F, seed, **kw):
    return bu.tracks_case(synth, C, F, seed, **kw)


def golden(name):
    return bu.golden_case(ROOT, name)


def check_against_model(emu, case, ks=(1, 2, 3), **kw):
    """k prefit iterations of the engine equal the model's, for each k in ks and for the whole prefit."""
    obs, mask, K, R0, t0 = case
    M = bu.prefit(obs, mask, K, R0, t0)
    for k in ks:
        if k <= M["iterations"]:
            bu.assert_iteration(M, k, *solve(emu, obs, mask, K, R0, t0, prefit_max_iter=k, **kw))
    R, t, r = solve(emu, obs, mask, K, R0, t0, **kw)
    bu.assert_prefit(M, R, t, r)
    return M, r


# ---- building blocks -----------------------------------------------------------------------------------------------
def _cs_view(Rt, K4, X, uv):
    """e, d e / d (w, dt), d e / d X of one view by complex step, w and dt applied as Exp(w) R X + t + dt."""
    def e(p):
        Xc = bu._exp_series(p[:3]) @ (Rt[:, :3] @ (X + p[6:])) + Rt[:, 3] + p[3:6]
        return np.array([K4[0] * Xc[0] / Xc[2] + K4[2] - uv[0], K4[1] * Xc[1] / Xc[2] + K4[3] - uv[1]])
    J = np.empty((2, 9))
    for j in range(9):
        d = np.zeros(9, complex)
        d[j] = 1e-30j
        J[:, j] = e(d).imag / 1e-30
    return e(np.zeros(9, complex)).real, J


WHERE = ["centre", "left_edge", "corner", "small_depth", "behind_tilt"]


@pytest.mark.parametrize("where", WHERE)
def test_view_jacobian_equals_complex_step(libs, where):
    """ba_view_jacobian's residual and its 2x6 camera and 2x3 point Jacobians, for points in the middle of the image,
    at its edges and corner, at 5 cm depth and seen by a strongly rotated camera."""
    _, parts = libs
    rng = np.random.default_rng(WHERE.index(where))
    K4 = np.array([600.0, 640.0, 320.0, 240.0])
    R = Rotation.from_rotvec(rng.normal(scale=0.3, size=3)).as_matrix()
    t = rng.normal(size=3)
    z = {"small_depth": 0.05}.get(where, 3.0)
    u, v = {"centre": (330.0, 250.0), "left_edge": (0.5, 240.0), "corner": (639.5, 479.5)}.get(where, (100.0, 400.0))
    if where == "behind_tilt":
        R = Rotation.from_rotvec([0.0, 1.4, 0.3]).as_matrix()
    Xc = np.array([(u - K4[2]) * z / K4[0], (v - K4[3]) * z / K4[1], z])
    X = R.T @ (Xc - t)                                   # the point that lands at (u, v) at depth z
    uv = np.array([u + 3.0, v - 2.0])
    Rt = np.ascontiguousarray(np.c_[R, t])
    out = np.zeros(20)
    parts.hc_ba_view_jacobian(ptr(Rt), ptr(K4), ptr(np.ascontiguousarray(X)), ptr(uv), ptr(out))
    e_ref, J_ref = _cs_view(Rt, K4, X, uv)
    scale = np.abs(J_ref).max()
    assert np.abs(out[:2] - e_ref).max() < 1e-9
    assert np.abs(out[2:14].reshape(2, 6) - J_ref[:, :6]).max() < 1e-12 * scale
    assert np.abs(out[14:].reshape(2, 3) - J_ref[:, 6:]).max() < 1e-12 * scale


ANGLES = [0.0, 1e-12, 5e-9, 1e-8, 1e-3, 1.0, np.pi - 1e-6, np.pi]


@pytest.mark.parametrize("angle", ANGLES)
def test_exp_so3_equals_scipy(libs, angle):
    """ba_exp_so3 (the prefit's pose update R' = Exp(w) R) on both sides of its th < 1e-8 series and up to pi."""
    _, parts = libs
    rng = np.random.default_rng(3)
    for _ in range(8):
        a = rng.normal(size=3)
        w = np.ascontiguousarray(a / np.linalg.norm(a) * angle)
        E = np.zeros(9)
        parts.hc_ba_exp_so3(ptr(w), ptr(E))
        assert np.abs(E.reshape(3, 3) - Rotation.from_rotvec(w).as_matrix()).max() < 1e-15


def _rotvecs():
    """Rotation vectors across the 1e-3 series switch, at pi exactly, and on every branch of the quaternion choice (the
    largest of R00, R11, R22 and the trace: near-pi turns about x, y and z pick 0, 1, 2; small turns pick the trace)."""
    out = []
    rng = np.random.default_rng(5)
    for a in (0.0, 1e-7, 1e-3 * (1 - 1e-9), 1e-3, 1e-3 * (1 + 1e-9), 0.5, 2.0, np.pi - 1e-7, np.pi):
        for _ in range(4):
            d = rng.normal(size=3)
            out.append(d / np.linalg.norm(d) * a)
    for axis in np.eye(3):
        for a in (np.pi, np.pi - 1e-4, 2.5):
            out.append(axis * a + 1e-3 * rng.normal(size=3) * (a < np.pi))
    return [np.ascontiguousarray(v) for v in out]


def test_rotvec_conversions_equal_scipy_and_trf(libs):
    """ba_rotvec_to_matrix / ba_matrix_to_rotvec equal scipy's Rotation (the reference's parameterisation), and the
    trf:: copies that engine 1 uses give the same bits."""
    _, parts = libs
    branches = set()
    for rv in _rotvecs():
        R, R2 = np.zeros(9), np.zeros(9)
        parts.hc_ba_rotvec_to_matrix(ptr(rv), ptr(R))
        parts.hc_trf_rotvec_to_matrix(ptr(rv), ptr(R2))
        ref = Rotation.from_rotvec(rv).as_matrix()
        assert np.array_equal(R, R2) and np.abs(R.reshape(3, 3) - ref).max() < 1e-15
        Rm = np.ascontiguousarray(ref.reshape(9))
        branches.add(int(np.argmax([Rm[0], Rm[4], Rm[8], Rm[0] + Rm[4] + Rm[8]])))
        v, v2 = np.zeros(3), np.zeros(3)
        parts.hc_ba_matrix_to_rotvec(ptr(Rm), ptr(v))
        parts.hc_trf_matrix_to_rotvec(ptr(Rm), ptr(v2))
        vref = Rotation.from_matrix(ref).as_rotvec()
        assert np.array_equal(v, v2)
        if np.linalg.norm(vref) > np.pi - 1e-6:          # at pi, w and -w are the same turn
            assert min(np.abs(v - vref).max(), np.abs(v + vref).max()) < 1e-9
        else:
            assert np.abs(v - vref).max() < 1e-13 * max(1.0, np.linalg.norm(vref))
    assert branches == {0, 1, 2, 3}


# ---- the model itself ----------------------------------------------------------------------------------------------
def test_model_dense_and_schur_forms_agree():
    """The model's dense solve over poses and points and its Schur form give the same trajectory."""
    case = tracks(4, 40, 10, rot=0.5, tsig=0.3)
    a, b = bu.prefit(*case, dense=True), bu.prefit(*case, dense=False)
    assert a["iterations"] == b["iterations"] and [s["accepted"] for s in a["trace"]] == [s["accepted"] for s in b["trace"]]
    assert abs(a["cost_final"] - b["cost_final"]) <= 1e-10 * a["cost_final"]
    assert np.abs(a["R"] - b["R"]).max() < 1e-10


def test_model_descends_to_the_true_rig():
    """From exact projections (no rounding of the pixels) the model's prefit reaches the true rig up to its scale."""
    o, poses, K, _ = synth.make_tracks(5, 60, seed=2, missing_frac=0.0, round_to_int=False)
    st = synth.perturb_poses(poses, seed=3)
    obs = np.array([[[v for v in cam] for cam in fr] for fr in o], dtype=np.float64)
    M = bu.prefit(obs, np.ones(obs.shape[:2], np.uint8), K, np.stack([p["R"] for p in st]), np.stack([p["t"] for p in st]))
    assert M["cost_final"] < 1e-12 * M["cost_initial"]
    for c in range(5):
        assert np.abs(M["R"][c] - poses[c]["R"]).max() < 1e-7
    assert np.abs(bu.scale_free(M["t"]) - bu.scale_free(np.stack([p["t"] for p in poses]))).max() < 1e-7


# ---- the device engine's prefit against the model ------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ba_c4", "ba_c8"])
def test_engine_prefit_equals_model_on_goldens(libs, name):
    check_against_model(libs[0], golden(name))


@pytest.mark.parametrize("C,F", [(2, 40), (3, 50), (16, 90)])
def test_engine_prefit_equals_model_on_synthetic_rigs(libs, C, F):
    """C = 16 is n = 90 camera parameters (BA_MAX_N)."""
    check_against_model(libs[0], tracks(C, F, 20 + C))


@pytest.mark.parametrize("m", [31, 32, 33, 65])
def test_engine_prefit_equals_model_at_tile_boundaries(libs, m):
    """Point counts around BA_TILE (32), with points of a single view (not valid) on the tile boundaries."""
    obs, mask, K, R0, t0 = tracks(4, m, 40 + m)
    for p in (0, 30, 31, 32, 63, 64):
        if p < m:
            mask[p] = 0
            mask[p, p % 4] = 1
    check_against_model(libs[0], (obs, mask, K, R0, t0))


def test_engine_prefit_indexes_intrinsics_by_present_view(libs):
    """Distinct intrinsics per camera, and views missing from low-index cameras, so that a point's k-th present view
    is often not camera k: the engine uses K[k], as the reference and the model do."""
    obs, mask, K, R0, t0 = tracks(5, 60, 7)
    rng = np.random.default_rng(8)
    Ks = np.stack([K] * 5)
    for c in range(5):
        Ks[c, 0, 0] += 40 * c; Ks[c, 1, 1] -= 25 * c; Ks[c, 0, 2] += 7 * c; Ks[c, 1, 2] -= 5 * c
    drop = rng.uniform(size=60) < 0.5
    mask[drop, 0] = 0
    mask[rng.uniform(size=60) < 0.4, 1] = 0
    assert (mask.sum(1) >= 2).sum() > 40
    M, _ = check_against_model(libs[0], (obs, mask, Ks, R0, t0))
    # the same problem with K[camera] is a different problem: the model tells them apart
    pb = bu.Problem(obs, mask, Ks)
    assert np.any(pb.v_k != pb.v_cam)


@pytest.mark.parametrize("n_ctas", [1, 3])
def test_engine_prefit_equals_model_on_any_grid(libs, n_ctas):
    check_against_model(libs[0], golden("ba_c4"), n_ctas=n_ctas)


def test_engine_prefit_equals_model_when_steps_are_rejected(libs):
    """A start 0.5 rad and 0.3 pose units off: steps get rejected and lambda climbs before the prefit converges."""
    case = tracks(4, 40, 10, rot=0.5, tsig=0.3)
    M, _ = check_against_model(libs[0], case, ks=(1, 2, 3, 4, 5, 6, 7))
    acc = [s["accepted"] for s in M["trace"]]
    assert not all(acc) and acc[-1]
    assert max(s["lam"] for s in M["trace"]) > 1e-3


def test_prefit_that_takes_no_step_leaves_the_polish_as_the_reference(libs):
    """The first step of this start is rejected; with one prefit iteration nothing is accepted.  The prefit then reports
    its initial cost as its final one, and the polish starts as scipy does (radius ||x0||): the same solve as without
    the prefit."""
    emu = libs[0]
    obs, mask, K, R0, t0 = tracks(4, 40, 11, rot=0.5, tsig=0.3)
    M = bu.prefit(obs, mask, K, R0, t0, max_iter=1)
    assert not M["trace"][0]["accepted"]
    R, t, r = solve(emu, obs, mask, K, R0, t0, prefit_max_iter=1, max_nfev=0)
    assert r["prefit_iterations"] == 1
    assert abs(r["prefit_cost_final"] - M["cost_initial"]) <= bu.COST_RTOL * M["cost_initial"]
    assert r["prefit_cost_final"] == r["prefit_cost_initial"]
    Rn, tn, rn = solve(emu, obs, mask, K, R0, t0, max_nfev=0, prefit=False)
    assert (r["status"], r["n_fev"], r["n_iterations"]) == (rn["status"], rn["n_fev"], rn["n_iterations"])
    assert abs(r["cost_final"] - rn["cost_final"]) <= 1e-9 * rn["cost_final"]


# ---- a camera that sees no point -----------------------------------------------------------------------------------
UNSEEN_COST_RTOL = 1e-6      # final robust cost of the masked rig against the rig without that camera


@pytest.mark.parametrize("n_ctas", [1, 2])
def test_unseen_camera_is_held_and_the_rest_fitted_as_without_it(libs, n_ctas):
    """Golden ba_c4 with every view of camera 3 masked out, against the same data as a 3-camera rig.  Before camera 3
    was held, its zero rows made the reduced system singular at every lambda: the prefit gave up after 16 iterations
    with prefit_cost_final 0, and the polish, started at the small radius meant for a converged prefit, stopped at a
    cost of 201 where the 3-camera rig reaches 0.055."""
    emu = libs[0]
    obs, mask, K, R0, t0 = golden("ba_c4")
    mask = mask.copy()
    mask[:, 3] = 0
    M = bu.prefit(obs, mask, K, R0, t0)
    M3 = bu.prefit(obs[:, :3], mask[:, :3], K, R0[:3], t0[:3])
    assert M["iterations"] == M3["iterations"] and np.abs(M["R"][:3] - M3["R"]).max() < 1e-12
    assert np.array_equal(M["R"][3], R0[3]) and np.array_equal(M["t"][3], t0[3])
    R, t, r = solve(emu, obs, mask, K, R0, t0, n_ctas=n_ctas)
    assert r["prefit_iterations"] == M["iterations"]
    assert abs(r["prefit_cost_final"] - M["cost_final"]) <= bu.COST_RTOL * M["cost_final"]
    assert np.abs(R[:3] - bu.rotvec_round_trip(M["R"][:3])).max() < 1e-8
    assert np.abs(bu.scale_free(t[:3]) - bu.scale_free(M["t"][:3])).max() < 1e-8
    assert np.abs(R[3] - R0[3]).max() < 1e-15 and np.array_equal(t[3], t0[3])
    # the whole solve, prefit and polish, against the 3-camera rig
    Rf, tf, rf = solve(emu, obs, mask, K, R0, t0, max_nfev=0, n_ctas=n_ctas)
    R3, t3, r3 = solve(emu, obs[:, :3], mask[:, :3], K, R0[:3], t0[:3], max_nfev=0, n_ctas=n_ctas)
    assert rf["status"] in (1, 2, 3, 4) and rf["prefit_iterations"] == r3["prefit_iterations"]
    assert abs(rf["cost_final"] - r3["cost_final"]) <= UNSEEN_COST_RTOL * r3["cost_final"], (rf["cost_final"], r3["cost_final"])
    assert np.abs(Rf[:3] - R3).max() < 1e-8 and np.abs(tf[:3] - t3).max() < 1e-8
    assert np.abs(Rf[3] - R0[3]).max() < 1e-15 and np.array_equal(tf[3], t0[3])


def test_unseen_low_index_camera_in_a_larger_rig(libs):
    """Camera 1 of a 6-camera rig sees nothing: the model holds it and fits the rest, and the engine follows."""
    obs, mask, K, R0, t0 = tracks(6, 80, 31)
    mask[:, 1] = 0
    keep = mask.sum(1) >= 2
    obs, mask = obs[keep], mask[keep]
    M, r = check_against_model(libs[0], (obs, mask, K, R0, t0))
    assert np.array_equal(M["R"][1], R0[1])

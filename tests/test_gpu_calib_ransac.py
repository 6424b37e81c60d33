"""The robust cold-start calibration on the GPU (csrc/calib_ransac.cu): RANSAC fundamental matrices for all adjacent
camera pairs, the pose chain refined from their inliers, and calculate_camera_poses(robust=True), on rigs whose
tracks carry mismatched points.  Run with ``-m gpu`` on an H100."""
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth
EINVAL = -1


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def contaminated_tracks(C, n, frac, seed):
    """synth.make_tracks with, in each camera, a fraction `frac` of its observations replaced by uniform random
    pixels (a stray reflection recorded instead of the marker).  Returns (obs, mask, obs_obj, bad [n, C], poses, K,
    true points)."""
    obs_obj, poses, K, pts = synth.make_tracks(C, n, seed=seed, missing_frac=0.1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    rng = np.random.default_rng(seed + 7919)
    bad = np.zeros(mask.shape, dtype=bool)
    for c in range(C):
        seen = np.flatnonzero(mask[:, c])
        pick = rng.choice(seen, int(round(frac * len(seen))), replace=False)
        bad[pick, c] = True
        obs[pick, c] = np.floor(rng.uniform([0, 0], [synth.WIDTH, synth.HEIGHT], size=(len(pick), 2)))
    out = np.empty(obs_obj.shape, dtype=object)
    for f in range(n):
        for c in range(C):
            out[f, c] = [int(obs[f, c, 0]), int(obs[f, c, 1])] if mask[f, c] else [None, None]
    return obs, mask, out, bad, poses, K, pts


def hypotheses_for(frac):
    """Per camera `frac` outliers leave a pair (1 - frac)^2 inliers; the budget is the number of 7-point samples that
    gives a clean one with confidence 0.99999 (cv2's setting), at least the default 2048: 16384 at 40 %."""
    w7 = ((1 - frac) ** 2) ** 7
    need = np.log(1e-5) / np.log1p(-w7) if w7 < 1 else 1.0
    return 2048 if need <= 2048 else 1 << int(np.ceil(np.log2(need)))


def rel_rot_errors(chain, poses):
    out = []
    for c in range(len(poses) - 1):
        Rt = np.asarray(poses[c + 1]["R"]) @ np.asarray(poses[c]["R"]).T
        Re = np.asarray(chain[c + 1]["R"], dtype=np.float64) @ np.asarray(chain[c]["R"], dtype=np.float64).T
        out.append(np.degrees(np.arccos(np.clip((np.trace(Rt.T @ Re) - 1) / 2, -1, 1))))
    return np.array(out)


def _ctx(C, K):
    ctx = pkg.MocapContext(C, 640, 480)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    return ctx


def e_rotation_error_deg(F, K, R_true):
    """Error of the better of the two rotations of E = K^T F K: the quality of F, whichever candidate a vote picks."""
    import cv2
    R1, R2, _ = cv2.decomposeEssentialMat(K.T @ F @ K)
    ang = lambda R: np.degrees(np.arccos(np.clip((np.trace(R.T @ R_true) - 1) / 2, -1, 1)))
    return min(ang(R1), ang(R2))


@pytest.mark.parametrize("C", [4, 8, 16])
@pytest.mark.parametrize("frac", [0.0, 0.1, 0.2, 0.3, 0.4])
def test_ransac_chain_and_masks(torch, C, frac):
    """Per pair, the relative rotation F_used gives (the better of E's two rotations) is within 2 degrees of the truth
    and within cv2 FM_RANSAC's (the reference's estimator) + 0.5 degrees; on the 4-camera ring the chain itself meets
    the same bar against the cv2 chain.  Over the rig's pairs the inlier masks keep >= 95 % of the true inliers and
    <= 3 % of the outliers.

    The chain is checked on 4 cameras only because the cheirality vote is the reference's (index.py:253-262): it
    triangulates camera c's pixel with camera c's pose in camera 0's frame and camera c+1's pixel with the relative
    candidate, so past the first pair it can pick the twisted pair however good F is (on the 16-camera arc the cv2 chain
    and this one each flip pairs the other does not)."""
    import cv2
    from oracle.ref_port import RefPort
    obs, mask, obs_obj, bad, poses, K, _ = contaminated_tracks(C, 1000, frac, seed=100 + C)
    ctx = _ctx(C, K)
    chain, F_used, votes, inl = ctx.calibrate_init(obs, mask, method="ransac", hypotheses=hypotheses_for(frac))
    assert (votes.max(axis=1) > 0).all()
    kept_in = n_in = kept_out = n_out = 0
    for c in range(C - 1):
        common = (mask[:, c] & mask[:, c + 1]).astype(bool)
        R_true = np.asarray(poses[c + 1]["R"]) @ np.asarray(poses[c]["R"]).T
        F_cv2, _ = cv2.findFundamentalMat(obs[common, c].astype(np.float32), obs[common, c + 1].astype(np.float32), cv2.FM_RANSAC, 1, 0.99999)
        e, e_cv2 = e_rotation_error_deg(F_used[c], K, R_true), e_rotation_error_deg(F_cv2, K, R_true)
        assert e < 2.0 and e <= e_cv2 + 0.5, (c, e, e_cv2)
        assert not inl[~common, c].any()
        got = inl[:, c].astype(bool)
        true_in = common & ~bad[:, c] & ~bad[:, c + 1]
        out = common & (bad[:, c] | bad[:, c + 1])
        kept_in += int(got[true_in].sum()); n_in += int(true_in.sum())
        kept_out += int(got[out].sum()); n_out += int(out.sum())
    assert kept_in >= 0.95 * n_in, (kept_in, n_in)
    assert kept_out <= 0.03 * n_out, (kept_out, n_out)
    if C == 4:
        err = rel_rot_errors(chain, poses)
        ref_err = rel_rot_errors(RefPort([K] * C).calibrate_init(obs_obj.tolist(), rng_seed=0), poses)
        assert (err < 2.0).all() and (err <= ref_err + 0.5).all(), (err, ref_err)


def test_calculate_camera_poses_robust_end_to_end(torch):
    """8 cameras, 20 % of each camera's observations mismatched: the final robust cost is at most 1.05 x that of a
    bundle adjustment started from the cv2 chain, and after a similarity alignment the points triangulated from their
    true views lie at least as close to the truth as with that adjustment's poses (+ 0.01).  The adjustment keeps every
    track, mismatched views included, as the reference's does, so neither reaches the clean-track bar of 0.03.  (Tracks
    on which the reference's cheirality vote picks the true motion for every pair: the adjustment cannot undo a
    twisted pair, see test_ransac_chain_and_masks.)"""
    from oracle.ref_port import RefPort
    C = 8
    obs, mask, obs_obj, bad, poses, K, pts = contaminated_tracks(C, 300, 0.2, seed=108)
    start = _ctx(C, K).calibrate_init(obs, mask, method="ransac")[0]
    assert (rel_rot_errors(start, poses) < 2.0).all()
    final = pkg.calculate_camera_poses(obs_obj.tolist(), session=pkg.MocapSession([K] * C), robust=True)
    ctx = _ctx(C, K)
    ctx.set_cameras([K] * C, final)
    cost = 0.5 * np.sum(np.log1p(ctx.ba_residuals(obs, mask, final).astype(np.float64) ** 2))
    ref_chain = RefPort([K] * C).calibrate_init(obs_obj.tolist(), rng_seed=0)
    ref_start = [{"R": np.asarray(p["R"], dtype=np.float64), "t": np.asarray(p["t"], dtype=np.float64).ravel()} for p in ref_chain]
    ctx.set_cameras([K] * C, ref_start)
    ref_final, rep = ctx.bundle_adjust(obs, mask, ref_start)
    assert cost <= rep["cost_final"] * 1.05 + 1e-6, (cost, rep["cost_final"])
    clean = (mask.astype(bool) & ~bad).astype(np.uint8)
    keep = clean.sum(axis=1) >= 2

    def aligned_error(rig):
        ctx.set_cameras([K] * C, rig)
        X, _, valid = ctx.triangulate(obs[keep], clean[keep])
        assert valid.all()
        A = X - X.mean(0); Bm = pts[keep] - pts[keep].mean(0)
        A *= np.linalg.norm(Bm) / np.linalg.norm(A)
        U, _, Vt = np.linalg.svd(A.T @ Bm)
        return np.abs(A @ (U @ Vt) - Bm).max()
    own, ref = aligned_error(final), aligned_error(ref_final)
    assert own <= ref + 0.01, (own, ref)


def test_clean_tracks_meet_the_8point_bar(torch):
    """On the clean tracks of test_calibrate_init_vs_oracle, the RANSAC chain meets that test's bar (ii): at least as
    close to the truth as the cv2 chain (+ 0.5 degrees), epipolar distances with median < 1 px, and after bundle
    adjustment a cost within 1.05 x and points within 0.03 of the truth."""
    from oracle.ref_port import RefPort
    C = 4
    obs_obj, poses, K, pts = synth.make_tracks(C, 80, seed=14, missing_frac=0.1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    ref_chain = RefPort([K] * C).calibrate_init(obs_obj.tolist(), rng_seed=0)
    ctx = _ctx(C, K)

    def rot_err_deg(chain_):
        return max(np.degrees(np.arccos(np.clip((np.trace(np.asarray(poses[c]["R"]).T @ np.asarray(chain_[c]["R"], dtype=np.float64)) - 1) / 2,
                                                -1, 1))) for c in range(1, C))
    own, F_own, _, _ = ctx.calibrate_init(obs, mask, method="ransac")
    assert rot_err_deg(own) <= rot_err_deg(ref_chain) + 0.5
    for c in range(C - 1):
        both = (mask[:, c] & mask[:, c + 1]).astype(bool)
        x1 = np.c_[obs[both, c], np.ones(both.sum())]; x2 = np.c_[obs[both, c + 1], np.ones(both.sum())]
        l = x1 @ F_own[c].T
        assert np.median(np.abs(np.sum(x2 * l, axis=1)) / np.sqrt(l[:, 0] ** 2 + l[:, 1] ** 2)) < 1.0
    final = pkg.calculate_camera_poses(obs_obj.tolist(), session=pkg.MocapSession([K] * C), robust=True)
    ctx.set_cameras([K] * C, final)
    cost_own = 0.5 * np.sum(np.log1p(ctx.ba_residuals(obs, mask, final).astype(np.float64) ** 2))
    ref_start = [{"R": np.asarray(p["R"], dtype=np.float64), "t": np.asarray(p["t"], dtype=np.float64).ravel()} for p in ref_chain]
    ctx.set_cameras([K] * C, ref_start)
    _, rep = ctx.bundle_adjust(obs, mask, ref_start)
    assert cost_own <= rep["cost_final"] * 1.05 + 1e-6
    ctx.set_cameras([K] * C, final)
    X, _, _ = ctx.triangulate(obs, mask)
    A = X - X.mean(0); Bm = pts - pts.mean(0)
    A *= np.linalg.norm(Bm) / np.linalg.norm(A)
    U, _, Vt = np.linalg.svd(A.T @ Bm)
    assert np.abs(A @ (U @ Vt) - Bm).max() < 0.03


def test_determinism(torch):
    """The RANSAC stage gives the same bits on every call.  The chain after it agrees to rounding: the 8-point
    re-fits (shared with the default method) sum their normal matrix with floating-point atomics, whose order varies.
    Another seed gives the same chain within 0.1 degrees, and a RANSAC call between two default calls does not change
    the default result."""
    C = 8
    obs, mask, _, _, poses, K, _ = contaminated_tracks(C, 300, 0.2, seed=5)
    ctx = _ctx(C, K)
    F1, m1 = ctx.fundamental_ransac(obs, mask)
    base = ctx.calibrate_init(obs, mask)
    a = ctx.calibrate_init(obs, mask, method="ransac")
    F2, m2 = ctx.fundamental_ransac(obs, mask)
    b = ctx.calibrate_init(obs, mask, method="ransac")
    again = ctx.calibrate_init(obs, mask)
    assert np.array_equal(F1, F2) and np.array_equal(m1, m2)
    for x, y in list(zip(a[0], b[0])) + list(zip(base[0], again[0])):
        assert np.abs(x["R"] - y["R"]).max() < 1e-9 and np.abs(x["t"] - y["t"]).max() < 1e-9
    assert np.abs(a[1] - b[1]).max() < 1e-9 and np.abs(base[1] - again[1]).max() < 1e-9
    assert np.array_equal(a[2], b[2]) and np.array_equal(base[2], again[2])
    assert (a[3] == b[3]).mean() >= 0.999
    other = ctx.calibrate_init(obs, mask, method="ransac", seed=12345)
    for c in range(C):
        Ra, Ro = a[0][c]["R"], other[0][c]["R"]
        assert np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Ro) - 1) / 2, -1, 1))) < 0.1


def test_ransac_stage_is_one_launch_per_kernel(torch):
    """The RANSAC stage launches the same number of kernels (one hypothesis, one scoring and one mask kernel) at 4
    and at 16 cameras."""
    deltas = []
    for C in (4, 16):
        obs, mask, _, _, _, K, _ = contaminated_tracks(C, 200, 0.1, seed=9)
        ctx = _ctx(C, K)
        n0 = ctx.launch_count()
        F, inl = ctx.fundamental_ransac(obs, mask)
        deltas.append(ctx.launch_count() - n0)
        assert F.shape == (C - 1, 3, 3) and np.allclose(np.linalg.norm(F.reshape(C - 1, 9), axis=1), 1.0)
    assert deltas[0] == deltas[1] == 3


def test_refusals_launch_nothing(torch):
    C = 4
    obs, mask, _, _, _, K, _ = contaminated_tracks(C, 100, 0.1, seed=2)
    ctx = _ctx(C, K)
    few = mask.copy()
    few[8:, 2] = 0                                   # cameras 1-2 and 2-3 share at most 8 frames ...
    few[1:8, 3] = 0                                  # ... and 2-3 fewer than 8
    n0 = ctx.launch_count()
    cases = [dict(threshold=0.0), dict(threshold=-1.0), dict(threshold=float("nan")), dict(threshold=float("inf")),
             dict(hypotheses=0), dict(hypotheses=65537)]
    for kw in cases:
        for call in (lambda: ctx.calibrate_init(obs, mask, method="ransac", **kw), lambda: ctx.fundamental_ransac(obs, mask, **kw)):
            with pytest.raises(pkg.MocapError) as e:
                call()
            assert e.value.status == EINVAL
    for call in (lambda: ctx.calibrate_init(obs, few, method="ransac"), lambda: ctx.fundamental_ransac(obs, few),
                 lambda: ctx.calibrate_init(obs[:7], mask[:7], method="ransac")):
        with pytest.raises(pkg.MocapError) as e:
            call()
        assert e.value.status == EINVAL
    assert ctx.launch_count() == n0
    with pytest.raises(ValueError):
        ctx.calibrate_init(obs, mask, method="lmeds")
    with pytest.raises(ValueError):
        ctx.calibrate_init(obs, mask, F_given=np.zeros((C - 1, 3, 3)), method="ransac")

"""The RANSAC pieces of the robust cold-start calibration (csrc/calib_ransac.cuh), compiled for the host with g++:
the 7-point solver against cv2's FM_7POINT, cv2's fundamental-matrix error and inlier masks, the counter-based
sampler, and the per-pair selection stepped on the host over contaminated pairs."""
import ctypes
import importlib

import cv2
import numpy as np
import pytest
from scipy import stats

from tests import hostbuild
from tests.calib_util import eight_point_refit
from tests.hostbuild import ptr

synth = importlib.import_module("low-cost-mocap_b200.synth")


@pytest.fixture(scope="module")
def rs():
    return hostbuild.load("calib_ransac")


def _draw(rs, seed, p, h0, count, m, attempt=0):
    idx = np.zeros((count, 7), dtype=np.int32)
    rs.hc_draw7(seed, p, h0, count, attempt, m, ptr(idx))
    return idx


def contaminated_pair(seed, frac, n=200):
    """Cameras 0 and 1 of the 8-camera rig (29 degrees apart), integer pixels; a fraction `frac` of the second view's
    observations replaced by uniform random pixels.  Returns (x1, x2, true relative rotation, K, outlier mask)."""
    obs, poses, K, _ = synth.make_tracks(8, n, seed=seed, missing_frac=0.0)
    x1 = np.array(obs[:, 0].tolist(), dtype=np.float64)
    x2 = np.array(obs[:, 1].tolist(), dtype=np.float64)
    rng = np.random.default_rng(seed + 1000)
    bad = np.zeros(n, dtype=bool)
    bad[rng.choice(n, int(round(frac * n)), replace=False)] = True
    x2[bad] = np.floor(rng.uniform([0, 0], [synth.WIDTH, synth.HEIGHT], size=(bad.sum(), 2)))
    return x1, x2, np.asarray(poses[1]["R"]), K, bad


def rotation_error_deg(F, K, R_true):
    """Error of the better of the two rotations of E = K^T F K."""
    R1, R2, _ = cv2.decomposeEssentialMat(K.T @ F @ K)
    ang = lambda R: np.degrees(np.arccos(np.clip((np.trace(R.T @ R_true) - 1) / 2, -1, 1)))
    return min(ang(R1), ang(R2))


def _normalised(q):
    c = q.mean(0)
    return (q - c) * (np.sqrt(2) / np.linalg.norm(q - c, axis=1).mean())


def _well_conditioned(a, b):
    """The normalised 7x9 epipolar system has a clear rank 7 (smallest / largest singular value >= 0.05)."""
    x1, x2 = _normalised(a.astype(np.float64)), _normalised(b.astype(np.float64))
    A = np.einsum("ni,nj->nij", np.c_[x2, np.ones(7)], np.c_[x1, np.ones(7)]).reshape(7, 9)
    s = np.linalg.svd(A, compute_uv=False)
    return s[6] / s[0] >= 0.05


def test_seven_point_matches_cv2(rs):
    """On random well-conditioned 7-point sets (a clear rank 7, distinct models): the same number of real roots as
    cv2's FM_7POINT, every model equal up to scale and sign to 1e-8 relative."""
    rng = np.random.default_rng(3)
    roots = set()
    tried = 0
    while tried < 300:
        a = rng.uniform(0, 640, (7, 2)).astype(np.float32)
        b = rng.uniform(0, 480, (7, 2)).astype(np.float32)
        if not _well_conditioned(a, b):
            continue
        F, _ = cv2.findFundamentalMat(a, b, cv2.FM_7POINT)
        ref = [] if F is None else [F[3 * i:3 * i + 3].ravel() / np.linalg.norm(F[3 * i:3 * i + 3]) for i in range(F.shape[0] // 3)]
        # nearly coincident roots make each model as sensitive as their separation is small: skip those sets
        if any(min(np.abs(r - q).max(), np.abs(r + q).max()) < 0.05 for i, r in enumerate(ref) for q in ref[:i]):
            continue
        tried += 1
        out = np.zeros(27)
        n = rs.hc_seven_point(ptr(np.ascontiguousarray(a.astype(np.float64).ravel())),
                              ptr(np.ascontiguousarray(b.astype(np.float64).ravel())), ptr(out))
        assert n == len(ref)
        roots.add(n)
        for k in range(n):
            g = out[9 * k:9 * k + 9]
            assert abs(np.linalg.norm(g) - 1) < 1e-12
            assert min(min(np.abs(g - r).max(), np.abs(g + r).max()) for r in ref) < 1e-8
    assert roots == {1, 3}


def test_seven_point_degenerate_samples_give_no_model(rs):
    """Coincident points, or all seven on one line in a view: no model."""
    rng = np.random.default_rng(4)
    b = rng.uniform(0, 480, 14)
    out = np.zeros(27)
    assert rs.hc_seven_point(ptr(np.full(14, 100.0)), ptr(b), ptr(out)) == 0
    t = np.sort(rng.uniform(0, 1, 7))
    line = np.ascontiguousarray(np.c_[100 + 300 * t, 50 + 200 * t].ravel())
    assert rs.hc_seven_point(ptr(line), ptr(b), ptr(out)) == 0
    assert rs.hc_has_collinear(ptr(line)) == 1


def test_fm_error_matches_numpy(rs):
    rng = np.random.default_rng(5)
    F = rng.normal(size=9)
    pts = np.ascontiguousarray(rng.uniform(0, 640, (1000, 4)))
    err = np.zeros(1000)
    rs.hc_fm_error(ptr(F), ptr(pts), 1000, ptr(err))
    Fm = F.reshape(3, 3)
    x1 = np.c_[pts[:, :2], np.ones(1000)]
    x2 = np.c_[pts[:, 2:], np.ones(1000)]
    l2 = x1 @ Fm.T                  # line of x1 in view 2
    l1 = x2 @ Fm                    # line of x2 in view 1
    d = (x2 * l2).sum(1)
    ref = np.maximum(d ** 2 / (l1[:, 0] ** 2 + l1[:, 1] ** 2), d ** 2 / (l2[:, 0] ** 2 + l2[:, 1] ** 2))
    assert np.allclose(err, ref, rtol=1e-10, atol=0)


@pytest.mark.parametrize("frac", [0.0, 0.2, 0.4])
def test_inlier_mask_agrees_with_cv2(rs, frac):
    """Under cv2's returned F, the inlier test gives cv2's returned mask on >= 99 % of the points."""
    for seed in range(3):
        x1, x2, _, _, _ = contaminated_pair(seed, frac)
        a, b = x1.astype(np.float32), x2.astype(np.float32)
        F, mask = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, 1, 0.99999)
        pts = np.ascontiguousarray(np.c_[a, b].astype(np.float64))
        mine = np.zeros(len(a), dtype=np.uint8)
        rs.hc_inlier_mask(ptr(np.ascontiguousarray(F.ravel())), ptr(pts), len(a), 1.0, ptr(mine))
        assert (mine == mask.ravel()).mean() >= 0.99


def test_sampler_distinct_in_range_and_repeatable(rs):
    for m in (7, 8, 13, 5000):
        idx = _draw(rs, 0, 2, 0, 2000, m)
        assert idx.min() >= 0 and idx.max() < m
        assert all(len(set(r)) == 7 for r in idx.tolist())
        assert np.array_equal(idx, _draw(rs, 0, 2, 0, 2000, m))
    base = _draw(rs, 0, 2, 0, 500, 1000)
    assert np.array_equal(base[100:], _draw(rs, 0, 2, 100, 400, 1000))       # a hypothesis does not depend on its neighbours
    for other in (_draw(rs, 1, 2, 0, 500, 1000), _draw(rs, 0, 3, 0, 500, 1000), _draw(rs, 0, 2, 0, 500, 1000, attempt=1)):
        assert (other != base).any(axis=1).mean() > 0.99


def test_sampler_has_no_gross_bias(rs):
    """10^5 draws over m = 50: index frequencies (all 7 slots, and the first slot alone) pass a chi-square test."""
    m = 50
    idx = _draw(rs, 12345, 0, 0, 100000, m)
    for sample in (idx.ravel(), idx[:, 0]):
        counts = np.bincount(sample, minlength=m)
        assert stats.chisquare(counts).pvalue > 1e-4
    # slot k never repeats an earlier slot, so every slot is uniform on its own too
    assert stats.chisquare(np.bincount(idx[:, 6], minlength=m)).pvalue > 1e-4


@pytest.mark.parametrize("frac", [0.0, 0.1, 0.2, 0.3, 0.4])
def test_host_selection_recovers_rotation(rs, frac):
    """The selection rule stepped on the host (2048 hypotheses, 1 px) over contaminated pairs, then the 8-point
    re-fits from the winner's inliers: relative rotation within 2 degrees.  The winner, a minimal 7-point model on
    integer pixels, keeps most true inliers and drops the outliers."""
    for seed in range(3):
        x1, x2, R_true, K, bad = contaminated_pair(seed, frac)
        pts = np.ascontiguousarray(np.c_[x1, x2].astype(np.float32))
        F = np.zeros(9)
        mask = np.zeros(len(x1), dtype=np.uint8)
        cnt = ctypes.c_int()
        assert rs.hc_ransac_select(ptr(pts), len(x1), 0, 2048, 0, 1.0, ptr(F), ptr(mask), ctypes.byref(cnt)) == 1
        inl = mask.astype(bool)
        assert cnt.value == inl.sum()
        assert inl[~bad].mean() >= 0.75 and (inl[bad].mean() if bad.any() else 0) <= 0.05
        assert rotation_error_deg(eight_point_refit(x1, x2, inl), K, R_true) < 2.0

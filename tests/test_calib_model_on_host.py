"""The host model of the calibration's device paths (tests/calib_util.py), pinned on its own, without a GPU: the full
pose-graph model recovers the true rig from noise-free tracks, and the chain model's re-fit -- the product's eigen
solver through the g++ build -- equals the numpy restatement of the 8-point chain."""
import numpy as np
import pytest

from tests import calib_util as cu
from tests.hostbuild import ptr
from tests.test_calib_ransac_on_host import contaminated_pair


@pytest.fixture(scope="module")
def libs():
    return cu.Libs()


@pytest.mark.parametrize("C", [4, 8, 16])
def test_graph_model_recovers_the_true_rig(libs, C):
    """Noise-free float tracks, 300 points: every pair used, rotations and translations (|t_1| = 1) within 1e-6 of the
    truth, and every view that enters the translation stage keeps weight >= 0.5.  1e-6 is the floor the float32 cast of
    the common observations sets (the reference casts them, index.py:243-244; measured 1.4e-7 and 3.2e-7): the
    translation stage alone reaches 1e-9 (test_calib_graph_on_host.py)."""
    obs, mask, poses, K = cu.float_tracks(C, 300, seed=5)
    g = cu.graph_model(libs, obs, mask, [K] * C)
    assert all(r["used"] and r["candidate"] >= 0 for r in g["pairs"])
    assert len(g["pairs"]) == C * (C - 1) // 2
    R_true = np.stack([np.asarray(q["R"]) for q in poses])
    t_true = np.stack([np.asarray(q["t"]).reshape(3) for q in poses])
    t_true = t_true / np.linalg.norm(t_true[1])
    assert np.abs(g["R"] - R_true).max() < 1e-6
    assert np.abs(g["t"] - t_true).max() < 1e-6
    assert np.array_equal(g["support"], g["init"])
    # every view of a track seen by 3 or more cameras enters
    many = mask.sum(1) >= 3
    assert np.array_equal(g["init"][many], mask[many])
    for r in g["pairs"]:
        assert r["inliers"] == r["common"] and r["in_front"] == r["inliers"]


@pytest.mark.parametrize("frac", [0.0, 0.2, 0.4])
def test_chain_model_fit_equals_numpy_refit(libs, frac):
    """The 2-camera case of test_calib_ransac_on_host.py: from the host RANSAC winner's inliers, the chain model's F
    (the product's trf::sym_eig / svd3 on the normal matrix) equals eight_point_refit's (numpy eigh / svd) up to sign,
    to 1e-9 relative, and the chain model of calibrate_init(method="ransac") on the same tracks gives that F."""
    for seed in range(3):
        x1, x2, _, K, _ = contaminated_pair(seed, frac)
        pts = np.ascontiguousarray(np.c_[x1, x2].astype(np.float32))
        r = cu.host_ransac(libs, pts, 0, 2048, 0, 1.0)
        assert r["ok"] and r["count"] == r["mask"].sum()
        want = cu.eight_point_refit(x1, x2, r["mask"])
        got, _, _ = cu.chain_refit(x1, x2, r["mask"], 1.0, cu.fit_product(libs))
        assert abs(np.linalg.norm(got) - 1) < 1e-12
        assert min(np.abs(got - want).max(), np.abs(got + want).max()) < 1e-9
        obs = np.stack([x1, x2], axis=1)
        ch = cu.chain_model(libs, obs, np.ones((len(x1), 2), dtype=np.uint8), [K, K], method="ransac")
        assert np.array_equal(ch["F"][0], got)
        assert np.array_equal(ch["inliers"][:, 0].astype(bool), cu.chain_refit(x1, x2, r["mask"], 1.0, cu.fit_product(libs))[1])


def test_chain_vote_picks_the_true_motion(libs):
    """On noise-free tracks the chain model's vote picks, for the first pair, the motion of the truth (the later pairs
    follow index.py's quirk, which needs no such property), and its F annihilates the common observations."""
    obs, mask, poses, K = cu.float_tracks(4, 200, seed=9)
    ch = cu.chain_model(libs, obs, mask, [K] * 4)
    R_rel = np.asarray(poses[1]["R"]) @ np.asarray(poses[0]["R"]).T
    assert np.abs(ch["R"][1] - R_rel).max() < 1e-6
    for c, (a, b, frames) in enumerate(cu.chain_pairs(mask)):
        assert np.sqrt(cu.sampson(ch["F"][c], obs[frames, a], obs[frames, b])).max() < 1e-3


def test_ransac_models_scan_equals_selection(libs):
    """hc_ransac_models' per-(hypothesis, root) counts give hc_ransac_select's winner: the most inliers, ties to the
    lowest index."""
    x1, x2, _, _, _ = contaminated_pair(1, 0.2)
    pts = np.ascontiguousarray(np.c_[x1, x2].astype(np.float32))
    r = cu.host_ransac(libs, pts, 3, 300, 7, 1.0)
    n, counts, F = cu.ransac_models(libs, pts, 3, 300, 7, 1.0)
    assert ((counts >= 0).sum(1) == n).all()
    flat = counts.ravel()
    k = int(np.argmax(flat))                                      # first maximum: lowest 3h + root
    assert flat[k] == r["count"]
    assert np.array_equal(F.reshape(-1, 3, 3)[k], r["F"])
    mask = np.zeros(len(pts), dtype=np.uint8)
    libs.rs.hc_inlier_mask(ptr(cu.c64(r["F"].ravel())), ptr(cu.c64(pts)), len(pts), 1.0, ptr(mask))
    assert np.array_equal(mask.astype(bool), r["mask"])
    assert (cu.ransac_margin(r["F"], pts, 1.0) > 0).all()



def test_fit_sign_convention(libs):
    """The fitted F's sign is fixed (calib_pose::fix_sign): its entry of largest magnitude is positive, so that the
    order of the four motions of E does not depend on how the eigen solver's rounding falls."""
    for seed in range(3):
        x1, x2, _, _, _ = contaminated_pair(seed, 0.2)
        inl = np.ones(len(x1), dtype=bool)
        T = np.r_[cu.hartley(x1, inl), cu.hartley(x2, inl)]
        F = cu.fit_product(libs)(x1, x2, inl, T).ravel()
        assert F[np.argmax(np.abs(F))] > 0
        want = cu.fit_numpy(x1, x2, inl, T).ravel()
        assert np.abs(F - want * np.sign(want[np.argmax(np.abs(want))])).max() < 1e-9

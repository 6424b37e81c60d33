"""The calibration's device kernels against their host model (tests/calib_util.py), stage by stage, through the public
entry points: RANSAC (ctx.fundamental_ransac: k_ransac_hypotheses / k_ransac_score / k_ransac_mask), the adjacent
chain (calibrate_init(method="8point" | "ransac"): k_epipolar_normal_pairs, k_sampson_pairs, k_cheirality) and the
pose graph (calibrate_init(method="graph"): k_epipolar_normal_pairs, k_sampson_pairs, k_pair_cheirality,
k_translation_normal / k_translation_reduce / k_translation_residuals).  The end-quality bars of
test_gpu_calib_ransac.py and test_gpu_calib_graph.py cannot see a kernel that drops a ragged tile, a partial sum or a
point at a tile boundary -- the optimiser absorbs it -- so these compare decisions exactly and values to 1e-9.

A decision (an inlier bit, a Sampson selection, a front flag, a weight at 0.5) may differ from the model's only where
rounding can move it: nvcc contracts to fused multiply-adds, the g++ builds use -ffp-contract=off.  Where one differs,
the model's float64 quantity must lie within FLIP of its threshold; the difference is printed and the comparisons
downstream of it are skipped for that case.  Anything else fails.  Run with ``-m gpu`` on an H100."""
import importlib

import numpy as np
import pytest

from tests import calib_util as cu
from tests.screen_util import contaminated_tracks

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
REL = 1e-9              # F, R, median / residual angles (degrees)
REL_T = 1e-8            # translations, |t_1| = 1
FLIP = 1e-9             # how close to its threshold a decision must be for the device to take it differently

# (C, n_points, frac, hypotheses, seed).  n_points is not a multiple of 16 or 64 (ragged tiles and a ragged last CTA
# in the translation stage); 77 points: one CTA; 1500 points at C = 2: one pair with more than 1024 common observations
# (two shared-memory tiles in k_ransac_score, several CTAs in k_ransac_mask); hypotheses not multiples of 8 or 128.
RANSAC_CASES = [(2, 1500, 0.2, 1000, 31), (2, 1500, 0.0, 2048, 32), (3, 77, 0.2, 129, 33), (3, 77, 0.0, 1, 34),
                (8, 203, 0.2, 1000, 35), (16, 301, 0.2, 2048, 36), (16, 301, 0.0, 129, 37)]
CHAIN_CASES = [(2, 1500, 0.2, 31), (3, 77, 0.0, 34), (3, 77, 0.2, 33), (8, 203, 0.2, 35), (16, 301, 0.0, 37), (16, 301, 0.2, 36)]
# (C, n_points, frac, hypotheses, seed, graph options).  At 16 cameras the 48 x 48 reduced system has 1176 entries: all
# 5 per-thread slots of k_translation_normal, the fifth partial.  36 points with min_common = 8: pairs of 8 to 31 common
# observations (fewer than a warp) and a single CTA in the translation stage.
GRAPH_CASES = [(2, 1500, 0.2, 1000, 31, {}), (3, 301, 0.2, 129, 41, {}), (4, 36, 0.0, 1000, 42, {"min_common": 8, "min_inliers": 8}),
               (8, 203, 0.2, 1000, 35, {}), (16, 301, 0.0, 2048, 37, {}), (16, 301, 0.2, 2048, 36, {})]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


@pytest.fixture(scope="module")
def libs():
    return cu.Libs()


def _ctx(C, K):
    ctx = pkg.MocapContext(C, 640, 480)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    return ctx


def _ids(cases):
    return ["C{}_n{}_f{}_H{}".format(*c[:4]) if len(c) > 4 else "C{}_n{}_f{}".format(*c[:3]) for c in cases]


def close(got, want, rel):
    """max |got - want| <= rel * max |want| (same sign: both sides normalise with the same arithmetic)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    return np.abs(got - want).max() <= rel * max(np.abs(want).max(), 1e-300)


def decisions_agree(what, dev, host, margin):
    """True if the device's decisions equal the model's; a difference where the model's quantity lies within FLIP of
    its threshold is printed and gives False (the comparisons that depend on it are then skipped); any other
    difference fails."""
    dev, host = np.asarray(dev), np.asarray(host)
    if np.array_equal(dev, host):
        return True
    m = float(np.min(margin))
    assert m <= FLIP, f"{what}: device {dev.tolist() if dev.size < 20 else int((dev != host).sum())} differs from the model " \
                      f"{host.tolist() if host.size < 20 else ''}, nearest decision {m:.3g} relative from its threshold"
    print(f"\n{what}: a decision within {m:.3g} of its threshold went the other way on the device (rounding)")
    return False


# ------------------------------------------------------------------------------------------------------------ RANSAC
@pytest.mark.parametrize("C,n,frac,H,seed", RANSAC_CASES, ids=_ids(RANSAC_CASES))
def test_ransac_equals_host_selection(torch, libs, C, n, frac, H, seed):
    """Per adjacent pair: the device's F is the host scan's winner to 1e-9 relative, and its inlier mask (whose size is
    the winner's inlier count) is the host's."""
    obs, mask, _, _, _, K, _ = contaminated_tracks(C, n, frac, seed)
    F_dev, inl_dev = _ctx(C, K).fundamental_ransac(obs, mask, hypotheses=H, seed=seed)
    for p_, (a, b, frames) in enumerate(cu.chain_pairs(mask)):
        r = cu.host_ransac(libs, cu.pair_points(obs, a, b, frames), p_, H, seed, 1.0)
        assert r["ok"]
        assert close(F_dev[p_], r["F"], REL), (p_, F_dev[p_], r["F"])
        dev_mask = inl_dev[frames, p_].astype(bool)
        if decisions_agree(f"RANSAC pair {p_} mask", dev_mask, r["mask"], r["margin"]):
            assert dev_mask.sum() == r["count"]
        assert not inl_dev[np.setdiff1d(np.arange(n), frames), p_].any()


def test_ransac_ties_go_to_the_lowest_hypothesis_and_root(torch, libs):
    """Noise-free tracks of one pair of 12 points: about every hypothesis reaches the full count, across all warps and
    CTAs of k_ransac_score, and the winner -- the lowest (hypothesis, root), here a third root -- is the only model the
    device may return.  The tied models differ from it by far more than the comparison's tolerance, but for the few
    hypotheses that drew the winner's 7 points again (12 points have 792 such sets)."""
    obs, mask, _, K = cu.float_tracks(2, 12, seed=21, missing_frac=0.0)
    a, b, frames = cu.chain_pairs(mask)[0]
    pts = cu.pair_points(obs, a, b, frames)
    H = 2048
    _, counts, F = cu.ransac_models(libs, pts, 0, H, 0, 1.0)
    tied = np.argwhere(counts == counts.max())
    assert counts.max() == 12 and len(tied) > H // 2 and len(np.unique(tied[:, 0] // 8)) > 100
    h0, r0 = tied[0]
    assert r0 > 0                                     # the winner is not a first root: a root-order mistake shows
    win = F[h0, r0]
    others = np.array([np.abs(F[h, r] - win).max() for h, r in tied[1:]]) / np.abs(win).max()
    assert (others <= 10 * REL).sum() <= 5 and np.sort(others)[5] > 10 * REL
    F_dev, inl_dev = _ctx(2, K).fundamental_ransac(obs, mask, hypotheses=H, seed=0)
    assert close(F_dev[0], win, REL), (F_dev[0], win)
    assert inl_dev[:, 0].all()


# ------------------------------------------------------------------------------------------------------------ chain
@pytest.mark.parametrize("method", ["8point", "ransac"])
@pytest.mark.parametrize("C,n,frac,seed", CHAIN_CASES, ids=_ids(CHAIN_CASES))
def test_chain_equals_model(torch, libs, method, C, n, frac, seed):
    """calibrate_init(method): per pair F_used to 1e-9 relative, the cheirality votes exactly, the RANSAC start's
    final Sampson sets exactly, and the chained poses to 1e-9."""
    obs, mask, _, _, _, K, _ = contaminated_tracks(C, n, frac, seed)
    H = 1000
    out = _ctx(C, K).calibrate_init(obs, mask, method=method, hypotheses=H, seed=seed)
    model = cu.chain_model(libs, obs, mask, [K] * C, method=method, H=H, seed=seed)
    poses, F_used, votes = out[:3]
    for c in range(C - 1):
        mg = model["margins"][c]
        if method == "ransac":
            r = model["ransac"][c]
            frames = cu.chain_pairs(mask)[c][2]
            if not decisions_agree(f"{method} pair {c} Sampson set", out[3][frames, c], model["inliers"][frames, c],
                                   [mg["sampson"], r["margin"].min()]):
                return
        assert close(F_used[c], model["F"][c], REL), (c, F_used[c], model["F"][c])
        if not decisions_agree(f"{method} pair {c} votes", votes[c], model["votes"][c], mg["front"]):
            return
    if method == "ransac":
        assert np.array_equal(out[3], model["inliers"])
    for c in range(C):
        assert close(poses[c]["R"], model["R"][c], REL), c
        assert np.abs(poses[c]["t"] - model["t"][c]).max() <= REL * max(1.0, np.abs(model["t"][c]).max()), c


@pytest.mark.parametrize("method", ["8point", "ransac"])
def test_chain_is_reproducible(torch, method):
    """Two calls of calibrate_init(method) on the same tracks return the same bits: F_used, votes, the Sampson sets and
    the poses.  The re-fits' normal matrices and selections are summed in a fixed order, so nothing depends on the
    order in which threads finish."""
    C = 16
    obs, mask, _, _, _, K, _ = contaminated_tracks(C, 301, 0.2, 36)
    ctx = _ctx(C, K)
    a, b = (ctx.calibrate_init(obs, mask, method=method, hypotheses=1000, seed=36) for _ in range(2))
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)
    for p, q in zip(a[0], b[0]):
        assert np.array_equal(p["R"], q["R"]) and np.array_equal(p["t"], q["t"])


def test_chain_launches_do_not_grow_per_pair(torch):
    """calibrate_init(method="8point"): at most three fit and two Sampson launches for all pairs, then one cheirality
    launch per pair, at 4 and 16 cameras."""
    for C, n, seed in ((4, 203, 35), (16, 301, 36)):
        obs, mask, _, _, _, K, _ = contaminated_tracks(C, n, 0.2, seed)
        ctx = _ctx(C, K)
        n0 = ctx.launch_count()
        ctx.calibrate_init(obs, mask, method="8point")
        assert ctx.launch_count() - n0 <= 5 + (C - 1), C


# ------------------------------------------------------------------------------------------------------------ graph
@pytest.mark.parametrize("C,n,frac,H,seed,opts", GRAPH_CASES, ids=_ids(GRAPH_CASES))
def test_graph_equals_model(torch, libs, C, n, frac, H, seed, opts):
    """calibrate_init(method="graph"): the pair report (a, b, common, inliers, candidate, in_front, used exactly; median
    triangulation angle and rotation residual to 1e-9 degrees), R to 1e-9, t to 1e-8 (|t_1| = 1) and the support mask
    exactly."""
    obs, mask, _, _, _, K, _ = contaminated_tracks(C, n, frac, seed)
    poses, pairs, support = _ctx(C, K).calibrate_init(obs, mask, method="graph", hypotheses=H, seed=seed, **opts)
    model = cu.graph_model(libs, obs, mask, [K] * C, H=H, seed=seed, **opts)
    assert len(pairs) == len(model["pairs"])
    if opts.get("min_common") == 8:
        assert min(m["common"] for m in model["pairs"]) < 32
    for p_, (d, h) in enumerate(zip(pairs, model["pairs"])):
        mg = model["margins"][p_]
        assert (d["a"], d["b"], d["common"]) == (h["a"], h["b"], h["common"]), p_
        if not decisions_agree(f"graph pair {p_} inliers", d["inliers"], h["inliers"], [mg["ransac"], mg["sampson"]]):
            return
        if not decisions_agree(f"graph pair {p_} cheirality", [d["candidate"], d["in_front"]], [h["candidate"], h["in_front"]],
                               mg["front"]):
            return
        assert d["used"] == h["used"], p_
        if h["candidate"] >= 0:
            assert abs(d["median_angle_deg"] - h["median_angle_deg"]) <= REL, (p_, d["median_angle_deg"], h["median_angle_deg"])
            assert abs(d["rot_residual_deg"] - h["rot_residual_deg"]) <= REL, (p_, d["rot_residual_deg"], h["rot_residual_deg"])
        else:
            assert np.isnan(d["median_angle_deg"]) and np.isnan(d["rot_residual_deg"])
    for c in range(C):
        assert np.abs(poses[c]["R"] - model["R"][c]).max() <= REL, c
        assert np.abs(poses[c]["t"] - model["t"][c]).max() <= REL_T, (c, poses[c]["t"], model["t"][c])
    decisions_agree("graph support", support, model["support"], model["weight_margin"])

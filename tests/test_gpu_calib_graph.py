"""The pose-graph cold start on the GPU (csrc/calib_graph.cu): start quality on rings and arcs with mismatched views,
including the seeds on which the adjacent chain twists a pair, calculate_camera_poses(init="graph") against the
clean-track bar, reproducibility, refusals and the Python checks.  Run with ``-m gpu`` on an H100."""
import importlib

import numpy as np
import pytest

from tests.screen_util import contaminated_tracks

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
EINVAL = -1
REJECT_PX = 8.0
ROT_BAR_DEG = 2.0
CENTRE_BAR = 0.15
RIGS = [(4, 0.0, 14)] + [(8, f, 108) for f in (0.0, 0.1, 0.2, 0.3)] + \
       [(16, f, s) for f in (0.0, 0.1, 0.2) for s in range(116, 122)]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _ctx(C, K):
    ctx = pkg.MocapContext(C, 640, 480)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    return ctx


def _angle(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(np.asarray(Ra).T @ np.asarray(Rb)) - 1) / 2, -1, 1)))


def start_errors(est, poses):
    """(max rotation error in degrees, max camera-centre error after a similarity fit of the centres to the truth)"""
    rot = max(_angle(e["R"], p["R"]) for e, p in zip(est, poses))
    ce = np.array([-np.asarray(e["R"]).T @ np.asarray(e["t"]).reshape(3) for e in est])
    ct = np.array([-np.asarray(p["R"]).T @ np.asarray(p["t"]).reshape(3) for p in poses])
    A, B = ce - ce.mean(0), ct - ct.mean(0)
    U, S, Vt = np.linalg.svd(A.T @ B)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    Rf = U @ D @ Vt                                   # A @ Rf ~ s B
    s = np.trace(np.diag(S) @ D) / (A ** 2).sum()
    return rot, np.linalg.norm(s * A @ Rf - B, axis=1).max()


def _chain_twisted(ctx, obs, mask, poses):
    chain = ctx.calibrate_init(obs, mask, method="ransac")[0]
    for c in range(len(poses) - 1):
        Rt = np.asarray(poses[c + 1]["R"]) @ np.asarray(poses[c]["R"]).T
        Re = np.asarray(chain[c + 1]["R"]) @ np.asarray(chain[c]["R"]).T
        if _angle(Rt, Re) >= 2.0:
            return True
    return False


@pytest.mark.parametrize("C,frac,seed", RIGS, ids=[f"C{c}_f{f}_s{s}" for c, f, s in RIGS])
def test_start_quality(torch, C, frac, seed):
    """300 points: every rotation within 2 degrees of the truth and every camera centre within 0.15 after a similarity
    fit (ring radius 3), and the pair report is consistent."""
    obs, mask, _, bad, poses, K, _ = contaminated_tracks(C, 300, frac, seed)
    poses_g, pairs, support = _ctx(C, K).calibrate_init(obs, mask, method="graph")
    rot, cen = start_errors(poses_g, poses)
    assert rot < ROT_BAR_DEG and cen < CENTRE_BAR, (rot, cen)
    assert abs(np.linalg.norm(poses_g[1]["t"]) - 1.0) < 1e-12
    assert support.shape == mask.shape and not (support.astype(bool) & ~mask.astype(bool)).any()
    assert ((support.sum(1) == 0) | (support.sum(1) >= 2)).all()
    assert sum(p["used"] for p in pairs) >= C - 1
    for p in pairs:
        assert 0 <= p["a"] < p["b"] < C and p["inliers"] <= p["common"]
    if frac > 0:
        kept = support.astype(bool)
        assert (kept & bad).sum() <= 0.02 * kept.sum(), (kept & bad).sum()


def test_start_quality_recorded_at_40_percent(torch, capsys):
    """8 cameras at 40 % mismatched views: recorded, no bar (DESIGN section 7)."""
    obs, mask, _, _, poses, K, _ = contaminated_tracks(8, 300, 0.4, 108)
    try:
        poses_g, pairs, _ = _ctx(8, K).calibrate_init(obs, mask, method="graph")
        rot, cen = start_errors(poses_g, poses)
        msg = f"max rotation error {rot:.2f} deg, max centre error {cen:.3f}, {sum(p['used'] for p in pairs)} of {len(pairs)} pairs used"
    except pkg.MocapError as e:
        msg = f"refused: {e}"
    with capsys.disabled():
        print(f"\n8 cameras, 40 % mismatched, graph start: {msg}")


def test_twisted_chain_seeds(torch, capsys):
    """Every rig of test_start_quality on which the adjacent RANSAC chain gets an adjacent rotation 2 degrees or more
    wrong: the graph start meets the same bars there."""
    twisted = []
    for C, frac, seed in RIGS:
        obs, mask, _, _, poses, K, _ = contaminated_tracks(C, 300, frac, seed)
        ctx = _ctx(C, K)
        if not _chain_twisted(ctx, obs, mask, poses):
            continue
        rot, cen = start_errors(ctx.calibrate_init(obs, mask, method="graph")[0], poses)
        twisted.append((C, frac, seed, rot, cen))
    with capsys.disabled():
        print(f"\nchain twisted on {len(twisted)} of {len(RIGS)} rigs: " +
              "; ".join(f"C{c} {f:.0%} seed {s}: graph {r:.2f} deg / {e:.3f}" for c, f, s, r, e in twisted))
    for C, frac, seed, rot, cen in twisted:
        assert rot < ROT_BAR_DEG and cen < CENTRE_BAR, (C, frac, seed, rot, cen)


def aligned_error(ctx, obs, clean, pts, rig, K):
    C = obs.shape[1]
    keep = clean.sum(axis=1) >= 2
    ctx.set_cameras([K] * C, rig)
    X, _, valid = ctx.triangulate(obs[keep], clean[keep])
    assert valid.all()
    A = X - X.mean(0); Bm = pts[keep] - pts[keep].mean(0)
    A *= np.linalg.norm(Bm) / np.linalg.norm(A)
    U, _, Vt = np.linalg.svd(A.T @ Bm)
    return np.abs(A @ (U @ Vt) - Bm).max()


@pytest.mark.parametrize("C,frac,seed", [(8, 0.3, 108), (16, 0.2, 116), (16, 0.0, 116)])
def test_calculate_camera_poses_graph_end_to_end(torch, capsys, C, frac, seed):
    """calculate_camera_poses(init="graph", reject_px=8): the points within 0.03 of the truth after a similarity
    alignment (the clean-track bar), on the cases the chain start leaves without a bar and on the clean arc."""
    obs, mask, obs_obj, bad, poses, K, pts = contaminated_tracks(C, 300, frac, seed)
    final = pkg.calculate_camera_poses(obs_obj.tolist(), session=pkg.MocapSession([K] * C), init="graph", reject_px=REJECT_PX)
    clean = (mask.astype(bool) & ~bad).astype(np.uint8)
    err = aligned_error(_ctx(C, K), obs, clean, pts, final, K)
    with capsys.disabled():
        print(f"\n{C} cameras, {frac:.0%} mismatched, seed {seed}, graph start + reject_px={REJECT_PX}: point error {err:.4f}")
    assert err < 0.03, err


def test_reproducible(torch):
    """The same inputs and seed give the same poses, pair report and support, bit for bit."""
    obs, mask, _, _, _, K, _ = contaminated_tracks(16, 300, 0.2, 116)
    ctx = _ctx(16, K)
    a = ctx.calibrate_init(obs, mask, method="graph", seed=3)
    b = _ctx(16, K).calibrate_init(obs, mask, method="graph", seed=3)
    for x, y in zip(a[0], b[0]):
        assert np.array_equal(x["R"], y["R"]) and np.array_equal(x["t"], y["t"])
    assert np.array_equal(a[2], b[2])
    table = lambda rep: np.array([[float(v) for v in p.values()] for p in rep])
    assert np.array_equal(table(a[1]), table(b[1]), equal_nan=True)


def test_refusals_launch_nothing(torch):
    C = 4
    obs, mask, _, _, _, K, _ = contaminated_tracks(C, 200, 0.1, 2)
    ctx = _ctx(C, K)
    n0 = ctx.launch_count()
    cut = mask.copy()
    cut[:, 3] = 0
    cut[:20, 3] = 1                       # camera 3 shares at most 20 observations with any other camera
    bad_calls = [lambda: ctx.calibrate_init(obs, cut, method="graph"),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", min_common=10_000),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", min_common=5),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", min_inliers=0),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", min_angle_deg=-1.0),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", min_angle_deg=float("nan")),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", rot_outlier_deg=0.0),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", irls_rounds=0),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", hypotheses=0),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", threshold=float("inf"))]
    for call in bad_calls:
        with pytest.raises(pkg.MocapError) as e:
            call()
        assert e.value.status == EINVAL
    with pytest.raises(pkg.MocapError) as e:
        ctx.calibrate_init(obs, cut, method="graph")
    assert "3" in str(e.value) and "not connected" in str(e.value)
    for call in (lambda: ctx.calibrate_init(obs, mask, method="graf"),
                 lambda: ctx.calibrate_init(obs, mask, method="graph", min_comon=30),
                 lambda: ctx.calibrate_init(obs, mask, method="ransac", min_common=30),
                 lambda: pkg.calculate_camera_poses([[[1, 2]] * C] * 10, session=pkg.MocapSession([K] * C), init="tree")):
        with pytest.raises(ValueError):
            call()
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0


def test_launches_do_not_grow_with_pairs(torch):
    """3 RANSAC launches, 3 x (fit + Sampson), one cheirality launch and 3 per translation round, at 4 and 16 cameras."""
    for C, seed in ((4, 14), (16, 116)):
        obs, mask, _, _, _, K, _ = contaminated_tracks(C, 300, 0.1, seed)
        ctx = _ctx(C, K)
        n0 = ctx.launch_count()
        ctx.calibrate_init(obs, mask, method="graph", irls_rounds=2)
        assert ctx.launch_count() - n0 == 3 + 6 + 1 + 3 * 2

"""The per-view screen on the GPU (csrc/screen.cu) and the screened bundle adjustment built on it: bit-equal masks and
stats against the host build of screen.cuh, drop rates on contaminated tracks, calculate_camera_poses(robust=True,
reject_px=...) reaching the clean-track bar with mismatched views, launch accounting, the config-3 chain on a side
stream, reproducibility and refusals.  Run with ``-m gpu`` on an H100."""
import importlib

import numpy as np
import pytest

from tests.screen_util import build_screen_host, contaminated_tracks, host_screen, poses_arrays, screen_inputs

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth
EINVAL = -1
REJECT_PX = 8.0          # the value INTEGRATION.md recommends (tools/screen_threshold_probe.py)
INPUTS = list(screen_inputs())


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build_screen_host(tmp_path_factory.mktemp("screen"))


def _ctx(C, K, poses=None):
    ctx = pkg.MocapContext(C, 640, 480)
    ctx.set_cameras([K] * C, poses or [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    return ctx


def _dev(torch, obs, mask, poses):
    R, t = poses_arrays(poses)
    return (torch.from_numpy(np.ascontiguousarray(obs)).cuda(), torch.from_numpy(np.ascontiguousarray(mask)).cuda(),
            torch.from_numpy(R).cuda(), torch.from_numpy(t).cuda())


@pytest.mark.parametrize("case", range(len(INPUTS)), ids=[c[0] for c in INPUTS])
def test_device_equals_host_build(torch, lib, case):
    """Every input of the CPU tier: the device mask and stats equal the host build's, through the device entry point
    (all rows, and n_points read from device memory with the rows past it untouched) and through the host entry point."""
    name, obs, mask, K, poses = INPUTS[case]
    C = mask.shape[1]
    want, want_stats = host_screen(lib, obs, mask, [K] * C, poses, 4.0)
    ctx = _ctx(C, K)
    d_obs, d_mask, R, t = _dev(torch, obs, mask, poses)
    got = ctx.screen_observations_dev(d_obs, d_mask, R, t, 4.0)
    torch.cuda.synchronize()
    assert np.array_equal(got["mask"].cpu().numpy(), want), name
    assert got["stats"].cpu().tolist() == want_stats.tolist()
    n = len(mask) - 7
    part_want, part_stats = host_screen(lib, obs[:n], mask[:n], [K] * C, poses, 4.0)
    out = {"mask": torch.full_like(d_mask, 0xAB), "stats": torch.zeros((4,), dtype=torch.int32, device="cuda")}
    ctx.screen_observations_dev(d_obs, d_mask, R, t, 4.0, n_points=torch.tensor([n], dtype=torch.int32, device="cuda"), out=out)
    torch.cuda.synchronize()
    m = out["mask"].cpu().numpy()
    assert np.array_equal(m[:n], part_want) and (m[n:] == 0xAB).all()
    assert out["stats"].cpu().tolist() == part_stats.tolist()
    h = ctx.screen_observations(obs, mask, poses, 4.0)
    assert np.array_equal(h["mask"], want) and h["stats"].tolist() == want_stats.tolist()


def _rates(torch, C, frac, seed=108, n=300):
    obs, mask, _, bad, poses, K, _ = contaminated_tracks(C, n, frac, seed)
    kept = _ctx(C, K).screen_observations(obs, mask, poses, 4.0)["mask"].astype(bool)
    seen = mask.astype(bool)
    return (~kept & bad).sum() / max(1, bad.sum()), (seen & ~bad & ~kept).sum() / max(1, (seen & ~bad).sum())


@pytest.mark.parametrize("C", [8, 16])
@pytest.mark.parametrize("frac", [0.1, 0.2, 0.3, 0.4])
def test_drop_rates_at_true_poses(torch, C, frac):
    """At the true poses, 4 px: >= 99.5 % of the mismatched views dropped and <= 0.5 % of the good ones at 10-30 %;
    >= 98 % and <= 1 % at 40 %."""
    drop_bad, drop_good = _rates(torch, C, frac)
    lo, hi = (0.98, 0.01) if frac >= 0.4 else (0.995, 0.005)
    assert drop_bad >= lo and drop_good <= hi, (drop_bad, drop_good)


def test_drop_rates_four_cameras_recorded(torch, capsys):
    """Four cameras: most tracks have 2-3 views and two views only test epipolar consistency.  Recorded, no bar."""
    rows = [(frac,) + tuple(_rates(torch, 4, frac)) for frac in (0.1, 0.2, 0.3, 0.4)]
    with capsys.disabled():
        print("\n4 cameras, 4 px, true poses: " + "; ".join(f"{f:.0%} mismatched: {100 * b:.2f} % of them and {100 * g:.2f} % "
                                                            f"of the good views dropped" for f, b, g in rows))
    assert all(b > 0.9 for _, b, _ in rows)


def rel_rot_errors(chain, poses):
    out = []
    for c in range(len(poses) - 1):
        Rt = np.asarray(poses[c + 1]["R"]) @ np.asarray(poses[c]["R"]).T
        Re = np.asarray(chain[c + 1]["R"], dtype=np.float64) @ np.asarray(chain[c]["R"], dtype=np.float64).T
        out.append(np.degrees(np.arccos(np.clip((np.trace(Rt.T @ Re) - 1) / 2, -1, 1))))
    return np.array(out)


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


def _end_to_end(C, frac, seed):
    obs, mask, obs_obj, bad, poses, K, pts = contaminated_tracks(C, 300, frac, seed)
    ctx = _ctx(C, K)
    start = ctx.calibrate_init(obs, mask, method="ransac")[0]
    if not (rel_rot_errors(start, poses) < 2.0).all():
        return None
    final = pkg.calculate_camera_poses(obs_obj.tolist(), session=pkg.MocapSession([K] * C), robust=True, reject_px=REJECT_PX)
    clean = (mask.astype(bool) & ~bad).astype(np.uint8)
    ctx.set_cameras([K] * C, final)
    cost = 0.5 * np.sum(np.log1p(ctx.ba_residuals(obs, clean, final).astype(np.float64) ** 2))
    ctx.set_cameras([K] * C, start)
    _, rep = ctx.bundle_adjust(obs, clean, start)
    return aligned_error(ctx, obs, clean, pts, final, K), cost, rep["cost_final"]


def _first_good_seed(C, frac, seeds):
    """the first seed whose chain the cheirality vote gets right (DESIGN section 7: the vote can twist a pair however
    good F is)"""
    for seed in seeds:
        r = _end_to_end(C, frac, seed)
        if r is not None:
            return r
    raise AssertionError("no seed with a correct chain")


@pytest.mark.parametrize("frac", [0.2, 0.1])
def test_calculate_camera_poses_screened_end_to_end(torch, frac):
    """test_calculate_camera_poses_robust_end_to_end's tracks (8 cameras, 300 points, 20 % mismatched, seed 108), and
    10 %: with reject_px the points lie within 0.03 of the truth after a similarity alignment (the clean-track bar the
    unscreened adjustment misses), and the final robust cost on the good views is within 1.05 x that of an adjustment
    on exactly the good views from the same chain."""
    err, cost, clean_cost = _end_to_end(8, frac, 108)
    assert err < 0.03, err
    assert cost <= 1.05 * clean_cost + 1e-6, (cost, clean_cost)


def test_calculate_camera_poses_screened_four_cameras(torch, capsys):
    """4 cameras, 20 % mismatched: the points meet the 0.03 bar.  Most tracks have 2-3 views there, and a mismatched
    view of a 2-view track that lies near the epipolar line cannot be told from a good one, so the cost on the good views
    is recorded, not held to 1.05 x."""
    err, cost, clean_cost = _first_good_seed(4, 0.2, [104, 105, 106, 107])
    with capsys.disabled():
        print(f"\n4 cameras, 20 % mismatched, reject_px={REJECT_PX}: point error {err:.4f}, cost on the good views "
              f"{cost:.3f} against {clean_cost:.3f} for an adjustment on exactly the good views")
    assert err < 0.03, err


@pytest.mark.parametrize("C,frac,seeds", [(8, 0.3, [108]), (16, 0.2, [116, 117, 118, 119, 120, 121])])
def test_calculate_camera_poses_screened_recorded(torch, capsys, C, frac, seeds):
    """8 cameras at 30 % and the 16-camera arc at 20 %: recorded, no bar.  The first solve (on the views that are RANSAC
    inliers with a neighbour) does not converge there, and the screens that follow cannot repair it (DESIGN section 7)."""
    err, cost, clean_cost = _first_good_seed(C, frac, seeds)
    with capsys.disabled():
        print(f"\n{C} cameras, {frac:.0%} mismatched, reject_px={REJECT_PX}: point error {err:.4f}, cost on the good views "
              f"{cost:.3f} against {clean_cost:.3f}")
    assert np.isfinite(err) and np.isfinite(cost)


def test_clean_tracks_lose_no_view_and_meet_the_8point_bar(torch):
    """On the clean tracks of test_clean_tracks_meet_the_8point_bar the screen drops no view at the poses it sees, and
    calculate_camera_poses(robust=True, reject_px=...) meets that test's bars: a cost within 1.05 x the adjustment
    started from the cv2 chain, and points within 0.03 of the truth."""
    from oracle.ref_port import RefPort
    C = 4
    obs_obj, poses, K, pts = synth.make_tracks(C, 80, seed=14, missing_frac=0.1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    ctx = _ctx(C, K)
    start = ctx.calibrate_init(obs, mask, method="ransac")[0]
    ctx.set_cameras([K] * C, start)
    _, _, kept = ctx.bundle_adjust_screened(obs, mask, start, REJECT_PX, rounds=2)
    assert np.array_equal(kept, mask)
    final = pkg.calculate_camera_poses(obs_obj.tolist(), session=pkg.MocapSession([K] * C), robust=True, reject_px=REJECT_PX)
    ctx.set_cameras([K] * C, final)
    cost_own = 0.5 * np.sum(np.log1p(ctx.ba_residuals(obs, mask, final).astype(np.float64) ** 2))
    ref_chain = RefPort([K] * C).calibrate_init(obs_obj.tolist(), rng_seed=0)
    ref_start = [{"R": np.asarray(p["R"], dtype=np.float64), "t": np.asarray(p["t"], dtype=np.float64).ravel()} for p in ref_chain]
    ctx.set_cameras([K] * C, ref_start)
    _, rep = ctx.bundle_adjust(obs, mask, ref_start)
    assert cost_own <= rep["cost_final"] * 1.05 + 1e-6
    assert aligned_error(ctx, obs, mask, pts, final, K) < 0.03


def test_default_keeps_the_unscreened_path(torch, monkeypatch):
    """reject_px=None is the adjustment of every view: the same poses as bundle_adjust from the same chain, and as
    bundle_adjust_screened with rounds=0 -- bit for bit.  calculate_camera_poses builds its own chain, which agrees with
    another run's to rounding only (calibrate_init's re-fits sum with atomics); on these 20 % mismatched tracks the
    adjustment carries that 1e-13 to several 1e-5 in the final poses, so the API's poses are compared with bundle_adjust
    from the very chain it built, recorded as it goes by."""
    C = 8
    obs, mask, obs_obj, _, _, K, _ = contaminated_tracks(C, 200, 0.2, seed=31)
    ctx = _ctx(C, K)
    start = ctx.calibrate_init(obs, mask, method="ransac")[0]
    ctx.set_cameras([K] * C, start)
    plain, _ = ctx.bundle_adjust(obs, mask, start)
    zero, _, kept = ctx.bundle_adjust_screened(obs, mask, start, REJECT_PX, rounds=0)
    assert np.array_equal(kept, mask)
    for a, b in zip(plain, zero):
        assert np.array_equal(a["R"], b["R"]) and np.array_equal(a["t"], b["t"])
    session = pkg.MocapSession([K] * C)
    inner, chains = session.ctx(C), []
    real = inner.calibrate_init

    def recording(*a, **kw):
        chains.append(real(*a, **kw))
        return chains[-1]
    monkeypatch.setattr(inner, "calibrate_init", recording)
    via_api = pkg.calculate_camera_poses(obs_obj.tolist(), session=session, robust=True)
    assert len(chains) == 1
    own_start = chains[0][0]
    for a, b in zip(start, own_start):
        assert np.abs(np.asarray(a["R"]) - b["R"]).max() < 1e-9 and np.abs(np.ravel(a["t"]) - np.ravel(b["t"])).max() < 1e-9
    ctx.set_cameras([K] * C, own_start)
    same, _ = ctx.bundle_adjust(obs, mask, own_start)
    for a, b in zip(same, via_api):
        assert np.array_equal(a["R"], b["R"]) and np.array_equal(a["t"], b["t"])
    # and from the other chain the adjustment ends at the same rig, to what it makes of the chains' rounding
    for a, b in zip(plain, via_api):
        assert np.abs(a["R"] - b["R"]).max() < 1e-3 and np.abs(a["t"] - b["t"]).max() < 1e-3


@pytest.mark.parametrize("rounds", [0, 1, 2, 3])
def test_launch_accounting(torch, rounds):
    """bundle_adjust_screened with `rounds` = r launches r screen kernels and r + 1 solves (one launch each)."""
    C = 8
    obs, mask, _, _, poses, K, _ = contaminated_tracks(C, 200, 0.2, seed=33)
    ctx = _ctx(C, K, poses)
    d_obs, d_mask, R, t = _dev(torch, obs, mask, poses)
    n0 = ctx.launch_count()
    ctx.screen_observations_dev(d_obs, d_mask, R, t, REJECT_PX)
    assert ctx.launch_count() == n0 + 1
    ctx.bundle_adjust_dev(d_obs, d_mask, R, t)
    assert ctx.launch_count() == n0 + 2
    torch.cuda.synchronize()
    n1 = ctx.launch_count()
    ctx.bundle_adjust_screened(obs, mask, synth.perturb_poses(poses, seed=2, rot_sigma=0.003, t_sigma=0.005), REJECT_PX, rounds=rounds)
    assert ctx.launch_count() - n1 == rounds + (rounds + 1)


def test_config3_chain_with_the_screen_on_a_side_stream(torch, lib):
    """pipeline(want_tracks=True) -> tracks_to_observations_dev -> screen_observations_dev (row count from device
    memory) -> bundle_adjust_dev, enqueued on a side stream without a host synchronisation: the screened mask equals
    the host build's on the rows written, the rows past them are untouched, and the solve equals one on that mask."""
    C = 8
    frames, _, poses, K = synth.make_frame_pool(C, 4, 64, seed=3)
    ctx = pkg.MocapContext(C, 640, 480, max_roots=16)
    ctx.set_cameras([K] * C, poses)
    fr = torch.from_numpy(frames).cuda()
    R0, t0 = (torch.from_numpy(a).cuda() for a in poses_arrays(poses))
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda.set_sync_debug_mode("error")
        try:
            tracks = ctx.pipeline(fr, want_tracks=True)
            o = ctx.tracks_to_observations_dev(tracks)
            out = {"mask": torch.full_like(o["mask"], 0xAB), "stats": torch.empty((4,), dtype=torch.int32, device="cuda")}
            before = ctx.launch_count()
            ctx.screen_observations_dev(o["obs"], o["mask"], R0, t0, REJECT_PX, n_points=o["n"], out=out)
            R, t = R0.clone(), t0.clone()
            rep = ctx.bundle_adjust_dev(o["obs"], out["mask"], R, t, n_points=o["n"])
            assert ctx.launch_count() == before + 2
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    n = int(o["n"].item())
    assert n > 0
    obs, mask, m = o["obs"].cpu().numpy()[:n], o["mask"].cpu().numpy()[:n], out["mask"].cpu().numpy()
    want, stats = host_screen(lib, obs, mask, [K] * C, poses, REJECT_PX)
    assert np.array_equal(m[:n], want) and (m[n:] == 0xAB).all()
    assert out["stats"].cpu().tolist() == stats.tolist()
    R2, t2 = R0.clone(), t0.clone()
    rep2 = ctx.bundle_adjust_dev(o["obs"], out["mask"], R2, t2, n_points=o["n"])
    torch.cuda.synchronize()
    assert torch.equal(R, R2) and torch.equal(t, t2)
    a, b = ctx.decode_ba_report(rep), ctx.decode_ba_report(rep2)
    a.pop("phase_ms"); b.pop("phase_ms")
    assert a == b


def test_reproducible(torch):
    """The screen gives the same bits on every call; bundle_adjust_screened from fixed starting poses gives the same
    poses, report and kept mask for a given CTA budget."""
    C = 8
    obs, mask, _, _, poses, K, _ = contaminated_tracks(C, 300, 0.2, seed=108)
    ctx = _ctx(C, K, poses)
    start = synth.perturb_poses(poses, seed=4, rot_sigma=0.003, t_sigma=0.005)
    d_obs, d_mask, R, t = _dev(torch, obs, mask, start)
    a = ctx.screen_observations_dev(d_obs, d_mask, R, t, REJECT_PX)
    b = ctx.screen_observations_dev(d_obs, d_mask, R, t, REJECT_PX)
    torch.cuda.synchronize()
    assert torch.equal(a["mask"], b["mask"]) and torch.equal(a["stats"], b["stats"])
    for grid in (0, 33):
        ctx.set_ba_grid(grid)
        runs = [ctx.bundle_adjust_screened(obs, mask, start, REJECT_PX, rounds=2) for _ in range(2)]
        (p1, r1, k1), (p2, r2, k2) = runs
        for x, y in zip(p1, p2):
            assert np.array_equal(x["R"], y["R"]) and np.array_equal(x["t"], y["t"])
        r1.pop("phase_ms"); r2.pop("phase_ms")
        assert r1 == r2 and np.array_equal(k1, k2)


def test_refusals_launch_nothing(torch):
    C = 4
    obs, mask, _, _, poses, K, _ = contaminated_tracks(C, 100, 0.1, seed=2)
    ctx = _ctx(C, K, poses)
    d_obs, d_mask, R, t = _dev(torch, obs, mask, poses)
    n0 = ctx.launch_count()
    for thr in (0.0, -1.0, float("nan"), float("inf")):
        for call in (lambda: ctx.screen_observations_dev(d_obs, d_mask, R, t, thr),
                     lambda: ctx.screen_observations(obs, mask, poses, thr),
                     lambda: ctx.bundle_adjust_screened(obs, mask, poses, thr)):
            with pytest.raises(pkg.MocapError) as e:
                call()
            assert e.value.status == EINVAL
    with pytest.raises(pkg.MocapError) as e:
        ctx.screen_observations_dev(d_obs, d_mask, R, t, 4.0, out={"mask": d_mask, "stats": None})
    assert e.value.status == EINVAL
    for rounds in (-1, -3):
        with pytest.raises(ValueError):
            ctx.bundle_adjust_screened(obs, mask, poses, 4.0, rounds=rounds)
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0

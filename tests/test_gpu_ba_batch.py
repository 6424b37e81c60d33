"""mocap_bundle_adjust_batch_dev: several independent bundle adjustments in ONE cooperative launch.  Problem k of K
runs on G // K + (k < G % K) of the context's G CTAs and must give the bits of mocap_bundle_adjust_dev on a context
whose budget is that many CTAs."""
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
synth = importlib.import_module("low-cost-mocap_b200.synth")
_lib = importlib.import_module("low-cost-mocap_b200._lib")

C = 8
SIZES = (18800, 3000, 500, 40)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _ctx(**kw):
    return pkg.MocapContext(C, 640, 480, **kw)


@pytest.fixture(scope="module")
def rig(torch):
    """One rig, four problems of 18 800 / 3000 / 500 / 40 points with their own seeds and perturbed starts."""
    _, poses, K, _ = synth.make_tracks(C, 8, seed=1, missing_frac=0.1)
    probs = []
    for i, F in enumerate(SIZES):
        obs_obj, _, _, _ = synth.make_tracks(C, F, seed=40 + i, missing_frac=0.1)
        obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
        mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
        start = synth.perturb_poses(poses, seed=60 + i)
        R0 = np.stack([np.asarray(p["R"]) for p in start])
        t0 = np.stack([np.asarray(p["t"]).reshape(3) for p in start])
        probs.append((obs, mask, R0, t0))
    return K, poses, probs


def _dev(torch, prob):
    obs, mask, R0, t0 = prob
    return {"obs": torch.from_numpy(obs).cuda(), "mask": torch.from_numpy(mask).cuda(),
            "R": torch.from_numpy(R0).cuda().contiguous(), "t": torch.from_numpy(t0).cuda().contiguous()}


def _result(ctx, d, rep):
    r = ctx.decode_ba_report(rep)
    r.pop("phase_ms")
    return d["R"].cpu().numpy(), d["t"].cpu().numpy(), r


def _single(torch, K, poses, prob, g, **opt):
    """bundle_adjust_dev on a context with budget g (None: the default)"""
    ctx = _ctx()
    ctx.set_cameras([K] * C, poses)
    if g is not None:
        ctx.set_ba_grid(g)
    d = _dev(torch, prob)
    rep = ctx.bundle_adjust_dev(d["obs"], d["mask"], d["R"], d["t"], n_points=d.get("n"), **opt)
    torch.cuda.synchronize()
    return _result(ctx, d, rep)


def _same(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert a[2] == b[2], (a[2], b[2])


def _split(G, K):
    return [G // K + (1 if k < G % K else 0) for k in range(K)]


@pytest.mark.parametrize("opt", [{}, {"prefit": False, "jacobian": 0}], ids=["default", "noprefit_fd32"])
def test_batch_equals_single_solves(torch, rig, opt):
    """K = 4, K = 5 (an uneven split of the SMs) and K = 1: every problem equals its single solve bit for bit."""
    K, poses, probs = rig
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    five = probs + [probs[2]]
    for batch in (probs, five, [probs[0]]):
        ctx = _ctx()
        ctx.set_cameras([K] * C, poses)
        ds = [_dev(torch, p) for p in batch]
        reps = ctx.bundle_adjust_batch_dev(ds, **opt)
        torch.cuda.synchronize()
        got = [_result(ctx, d, r) for d, r in zip(ds, reps)]
        grids = _split(sms, len(batch)) if len(batch) > 1 else [None]
        for prob, g, res in zip(batch, grids, got):
            assert res[2]["status"] in (0, 1, 2, 3, 4) and res[2]["n_launches"] == 1
            _same(res, _single(torch, K, poses, prob, g, **opt))


def test_batch_empty_problem(torch, rig):
    """A device count of 0, and a problem whose points have one view each: status -3, poses untouched; the
    neighbours equal their single solves."""
    K, poses, probs = rig
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = _ctx()
    ctx.set_cameras([K] * C, poses)
    ds = [_dev(torch, p) for p in probs[1:4]]
    ds[0]["n"] = torch.zeros((1,), dtype=torch.int32, device="cuda")
    one = probs[3][1].copy()
    one[:, 1:] = 0
    ds[2] = _dev(torch, (probs[3][0], one, probs[3][2], probs[3][3]))
    reps = ctx.bundle_adjust_batch_dev(ds)
    torch.cuda.synchronize()
    for k in (0, 2):
        R, t, r = _result(ctx, ds[k], reps[k])
        assert r["status"] == -3 and r["n_residuals"] == 0
        src = probs[1 + k]
        assert np.array_equal(R, src[2]) and np.array_equal(t, src[3])
    _same(_result(ctx, ds[1], reps[1]), _single(torch, K, poses, probs[2], _split(sms, 3)[1]))


def test_batch_config3_chain_on_one_stream(torch):
    """pipeline(want_tracks=True) -> tracks_to_observations_dev on four slices -> one batch call, enqueued on a side
    stream without a synchronisation: one launch for the batch, each problem equal to its single solve."""
    frames, _, poses, K = synth.make_frame_pool(C, 4, 64, seed=3)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    start = synth.perturb_poses(poses, seed=10)
    R0 = torch.from_numpy(np.stack([np.asarray(p["R"]) for p in start])).cuda().contiguous()
    t0 = torch.from_numpy(np.stack([np.asarray(p["t"]).reshape(3) for p in start])).cuda().contiguous()
    ctx = _ctx(max_roots=16)
    ctx.set_cameras([K] * C, poses)
    fr = torch.from_numpy(frames).cuda()
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        tracks = ctx.pipeline(fr, want_tracks=True)
        obs = []
        for j in range(4):
            sl = slice(16 * j, 16 * (j + 1))
            obs.append(ctx.tracks_to_observations_dev({k: tracks[k][sl] for k in ("track_xy", "n", "err")}, max_err=5.0))
        ds = [{"obs": o["obs"], "mask": o["mask"], "n": o["n"], "R": R0.clone(), "t": t0.clone()} for o in obs]
        before = ctx.launch_count()
        reps = ctx.bundle_adjust_batch_dev(ds)
        assert ctx.launch_count() == before + 1
    torch.cuda.synchronize()
    grids = _split(sms, 4)
    for j in range(4):
        got = _result(ctx, ds[j], reps[j])
        assert got[2]["n_residuals"] > 0
        single = _ctx(max_roots=16)
        single.set_cameras([K] * C, poses)
        single.set_ba_grid(grids[j])
        R, t = R0.clone(), t0.clone()
        rep = single.bundle_adjust_dev(ds[j]["obs"], ds[j]["mask"], R, t, n_points=ds[j]["n"])
        torch.cuda.synchronize()
        _same(got, _result(single, {"R": R, "t": t}, rep))


def test_batch_is_reproducible(torch, rig):
    K, poses, probs = rig
    runs = []
    for _ in range(2):
        ctx = _ctx()
        ctx.set_cameras([K] * C, poses)
        ds = [_dev(torch, p) for p in probs]
        reps = ctx.bundle_adjust_batch_dev(ds)
        torch.cuda.synchronize()
        runs.append([_result(ctx, d, r) for d, r in zip(ds, reps)])
    for a, b in zip(*runs):
        _same(a, b)


def test_batch_refusals_launch_nothing(torch, rig):
    K, poses, probs = rig
    ctx = _ctx()
    ctx.set_cameras([K] * C, poses)
    d = _dev(torch, probs[3])
    ctx.set_ba_grid(3)
    before = ctx.launch_count()
    bad = [
        [],                                                       # K < 1
        [d] * 4,                                                  # K > G
        [dict(d, obs=None)],                                      # NULL pointers
        [dict(d, mask=None)],
        [dict(d, R=None)],
        [dict(d, t=None)],
        [dict(d, obs=d["obs"][:0])],                              # n_points_max <= 0
    ]
    for problems in bad:
        with pytest.raises(pkg.MocapError):
            ctx.bundle_adjust_batch_dev(problems)
    ctx.set_ba_grid(0)
    with pytest.raises(pkg.MocapError):
        ctx.bundle_adjust_batch_dev([d] * (_lib.MOCAP_BA_MAX_BATCH + 1))
    assert ctx.launch_count() == before
    unset = _ctx()                                                # cameras not set
    with pytest.raises(pkg.MocapError):
        unset.bundle_adjust_batch_dev([d])
    assert unset.launch_count() == 0
    one = pkg.MocapContext(1, 640, 480)                           # fewer than two cameras
    one.set_cameras([K], poses[:1])
    before = one.launch_count()
    with pytest.raises(pkg.MocapError):
        one.bundle_adjust_batch_dev([d])
    assert one.launch_count() == before

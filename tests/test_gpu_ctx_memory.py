"""The context's buffers as they grow: one context runs each family of entry points at a small, then a larger, then
again a small size, and every result must equal, bit for bit, what a fresh context gives at that size.  This covers the
grow-only buffers (detection images, the chunked matcher, host staging and frame-set outputs, the live loop's staging,
the overlay's line counts, the JPEG scratch and output, the bundle adjustment's workspace and barrier words) and the
generic scratch shared by the triangulation, screening, bundle adjustment and calibration entry points."""
import importlib

import numpy as np
import pytest

from tests.live_util import CAPTURE, DIST, IN_H, IN_W, K as LIVE_K, TRIANGULATE, make_scene, render_read

pytestmark = pytest.mark.gpu
api = importlib.import_module("low-cost-mocap_b200.api")
pkg = importlib.import_module("low-cost-mocap_b200")
synth = importlib.import_module("low-cost-mocap_b200.synth")
SIZES = (0, 1, 0)                 # index into each family's (small, large) inputs: small, large, small again


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _leaves(x):
    if isinstance(x, dict):
        return [v for k in sorted(x) for v in _leaves(x[k])]
    if isinstance(x, (list, tuple)):
        return [v for e in x for v in _leaves(e)]
    if hasattr(x, "cpu"):
        return [x.cpu().numpy()]
    return [np.asarray(x)]


def _same(a, b, what):
    la, lb = _leaves(a), _leaves(b)
    assert len(la) == len(lb), what
    for j, (u, v) in enumerate(zip(la, lb)):
        assert u.shape == v.shape and u.dtype == v.dtype and u.tobytes() == v.tobytes(), (what, j, u, v)


def _agree(a, b, what):
    """The calibration chains after RANSAC: their 8-point re-fits sum with floating-point atomics, so two runs agree to
    rounding only (the bar of test_gpu_calib_ransac.py's determinism test)."""
    la, lb = _leaves(a), _leaves(b)
    assert len(la) == len(lb), what
    for j, (u, v) in enumerate(zip(la, lb)):
        assert u.shape == v.shape and u.dtype == v.dtype, (what, j)
        if u.dtype.kind == "f":
            assert np.allclose(u, v, rtol=1e-9, atol=1e-9), (what, j, u, v)
        elif u.dtype == np.uint8 and u.ndim == 2:            # inlier masks
            assert (u == v).mean() >= 0.999, (what, j)
        else:
            assert np.array_equal(u, v), (what, j, u, v)


def _check(make, run, inputs, rounding=()):
    """run(ctx, inputs[i]) on one context for i in SIZES, each against a fresh context's run; run returns a dict of
    named results, bit-identical except those named in `rounding`."""
    shared = make()
    for step, i in enumerate(SIZES):
        got, want = run(shared, inputs[i]), run(make(), inputs[i])
        assert sorted(got) == sorted(want)
        for k in sorted(got):
            (_agree if k in rounding else _same)(got[k], want[k], (step, k))


def _tracks(out, torch):
    """n, flags and the filled rows of obj / err (rows past n are not written)"""
    torch.cuda.synchronize()
    n = out["n"].cpu().numpy()
    obj, err = out["obj"].cpu().numpy(), out["err"].cpu().numpy()
    return [n, out["flags"].cpu().numpy()] + [np.concatenate([obj[b, :n[b]].ravel(), err[b, :n[b]]]) for b in range(len(n))]


def test_pipeline_and_matcher_grow(torch):
    C = 4
    pools = [synth.make_frame_pool(C, 6, B, seed=3 + B)[0] for B in (3, 24)]
    _, _, poses, K = synth.make_frame_pool(C, 6, 1, seed=3)

    def make():
        ctx = pkg.MocapContext(C, 640, 480)
        ctx.set_cameras([K] * C, poses)
        return ctx

    def run(ctx, frames):
        f = torch.from_numpy(frames).cuda()
        det = ctx.detect(f.reshape(-1, 480, 640).contiguous())
        return {"pipeline": _tracks(ctx.pipeline(f), torch), "match": _tracks(ctx.match_triangulate(det["xy"], det["n"]), torch)}

    _check(make, run, pools)


def test_pipeline_host_staging_and_sets_grow(torch):
    C = 4
    pools = [synth.make_frame_pool(C, 6, B, seed=11 + B)[0] for B in (2, 20)]
    _, _, poses, K = synth.make_frame_pool(C, 6, 1, seed=11)

    def make():
        ctx = pkg.MocapContext(C, 640, 480)
        ctx.set_cameras([K] * C, poses)
        return ctx

    _check(make, lambda ctx, frames: {"pipeline_host": _tracks(ctx.pipeline_host(frames), torch)}, pools)


def _live_make(scene, overlay):
    def make():
        C = scene["C"]
        ctx = api.MocapContext(C, 320, 320, **api.MIRROR_LIMITS)
        if overlay:
            ctx.set_overlay(True)
        ctx.set_preprocess(IN_W, IN_H, scene["rotations"], [LIVE_K] * C, [DIST] * C)
        ctx.set_cameras([LIVE_K] * C, scene["poses"])
        return ctx
    return make


def _live_result(out, keys):
    return {k: out[k] for k in keys + ("frames",)}


def test_live_host_with_overlay_grows(torch):
    scene = make_scene(5, np.eye(4))
    reads = [np.stack([render_read(scene, k) for k in range(B)]) for B in (1, 5)]
    mode = CAPTURE | TRIANGULATE

    def run(ctx, raw):
        ctx.set_overlay(True)                  # the session's line counter (so the line colours) starts again at 0
        out = ctx.live_host(raw, mode, want_frames=True)
        n = out["n"]
        return dict(_live_result(out, ("flags", "gate", "blob_n", "first", "n")), obj=[out["obj"][b, :n[b]] for b in range(len(n))])

    _check(_live_make(scene, True), run, reads)


def test_live_host_jpeg_grows(torch):
    scene = make_scene(6, np.eye(4))
    reads = [np.stack([render_read(scene, k) for k in range(B)]) for B in (1, 6)]

    def run(ctx, raw):
        out = ctx.live_host(raw, CAPTURE, want_frames=True, jpeg=True)
        return dict(_live_result(out, ("flags", "gate", "blob_n", "first", "jpeg_len")),
                    jpeg=[out["jpeg"][b, :out["jpeg_len"][b]] for b in range(raw.shape[0])])

    _check(_live_make(scene, False), run, reads)


def _obs_mask(obs_obj):
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    return obs, mask


def test_ba_batch_workspace_grows(torch):
    C = 4
    _, poses, K, _ = synth.make_tracks(C, 8, seed=1, missing_frac=0.1)

    def problems(sizes, seed):
        out = []
        for i, F in enumerate(sizes):
            obs, mask = _obs_mask(synth.make_tracks(C, F, seed=seed + i, missing_frac=0.1)[0])
            start = synth.perturb_poses(poses, seed=seed + 20 + i)
            out.append((obs, mask, np.stack([np.asarray(p["R"]) for p in start]), np.stack([np.asarray(p["t"]).reshape(3) for p in start])))
        return out

    inputs = [problems((60, 40), 40), problems((900, 300, 120), 50)]

    def make():
        ctx = pkg.MocapContext(C, 640, 480)
        ctx.set_cameras([K] * C, poses)
        return ctx

    def run(ctx, probs):
        dev = [{"obs": torch.from_numpy(o).cuda(), "mask": torch.from_numpy(m).cuda(), "R": torch.from_numpy(R).cuda().contiguous(),
                "t": torch.from_numpy(t).cuda().contiguous()} for o, m, R, t in probs]
        reps = ctx.bundle_adjust_batch_dev(dev)
        torch.cuda.synchronize()
        out = {}
        for k, (d, rep) in enumerate(zip(dev, reps)):
            r = ctx.decode_ba_report(rep)
            r.pop("phase_ms")
            out[f"problem {k}"] = [d["R"], d["t"], r]
        return out

    _check(make, run, inputs, rounding=("ransac", "graph"))


def test_scratch_users_share_one_scratch(torch):
    """triangulate, screen_observations, ba_residuals, bundle_adjust and calibrate_init (ransac and graph) in turn on one
    context, small, large, small."""
    C = 4
    _, poses, K, _ = synth.make_tracks(C, 8, seed=2, missing_frac=0.1)
    inputs = []
    for F, seed in ((60, 70), (900, 71)):
        obs, mask = _obs_mask(synth.make_tracks(C, F, seed=seed, missing_frac=0.1)[0])
        inputs.append((obs, mask, synth.perturb_poses(poses, seed=seed + 5)))

    def make():
        ctx = pkg.MocapContext(C, 640, 480)
        ctx.set_cameras([K] * C, poses)
        return ctx

    def outcome(call):
        try:
            return call()
        except api.MocapError as e:          # a refusal must be the same refusal
            return str(e)

    def run(ctx, inp):
        obs, mask, start = inp
        ctx.set_cameras([K] * C, poses)
        out = {"triangulate": ctx.triangulate(obs, mask), "screen": ctx.screen_observations(obs, mask, start, 2.0),
               "ba_residuals": ctx.ba_residuals(obs, mask, start)}
        adj, rep = ctx.bundle_adjust(obs, mask, start)
        rep.pop("phase_ms")
        out["bundle_adjust"] = [adj, rep]
        out["fundamental_ransac"] = ctx.fundamental_ransac(obs, mask, hypotheses=256)
        out["ransac"] = outcome(lambda: ctx.calibrate_init(obs, mask, method="ransac", hypotheses=256))
        out["graph"] = outcome(lambda: ctx.calibrate_init(obs, mask, method="graph", hypotheses=256))
        return out

    _check(make, run, inputs, rounding=("ransac", "graph"))

"""GPU parity tests: the CUDA path (through the C ABI) against the committed golden vectors
written by the real reference, against the oracle port on seeded inputs, and -- at BASELINE
sizes -- through size-independent properties.  Run with ``-m gpu`` on an H100."""
import importlib
import os

import numpy as np
import pytest

from tests.hostbuild import ptr
from tests.util import load_golden, poses_from, obs_from, as3

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth

PIPE_CASES = ["pipe_c2_m1", "pipe_c4_m4", "pipe_c8_m16"]
X_TOL = 1e-7          # pose units; BASELINE north_star: 1e-4 mm with poses in metres
ERR_RTOL = 1e-9       # reprojection errors are float32-quantised upstream; expected bit-equal


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _ctx(C, **kw):
    return pkg.MocapContext(C, 640, 480, **kw)


# ------------------------------------------------------------------------------------------ S1
@pytest.mark.parametrize("name", PIPE_CASES + ["blobs_irregular"])
def test_detect_exact_vs_reference_golden(torch, name):
    z = load_golden(name)
    frames = z["frames"]
    B, C = frames.shape[:2]
    ctx = _ctx(C, max_blobs=64)
    d = ctx.detect(torch.from_numpy(frames).cuda(), want_moments=True)
    n = d["n"].cpu().numpy().reshape(B, C)
    xy = d["xy"].cpu().numpy().reshape(B, C, 64, 2)
    assert (d["flags"].cpu().numpy() == 0).all()
    assert np.array_equal(n, z["blob_n"])                       # exact count
    for b in range(B):
        for c in range(C):
            k = n[b, c]
            assert np.array_equal(xy[b, c, :k], z["blob_xy"][b, c, :k]), (b, c)   # exact centres, exact order


def test_detect_pixel_counts_and_moments_vs_cv2(torch):
    """Auxiliary checksum (SURVEY §8(d)): per-blob pixel count == cv2.connectedComponentsWithStats
    (8-connectivity), and A2/SX6/SY6 == the integers cv.moments accumulates for the contour."""
    import cv2
    z = load_golden("blobs_irregular")
    frames = z["frames"][:, 0]
    ctx = _ctx(1, max_blobs=64)
    d = ctx.detect(torch.from_numpy(frames).cuda(), want_moments=True)
    n = d["n"].cpu().numpy(); mom = d["mom"].cpu().numpy()
    for f in range(len(frames)):
        binary = (frames[f] > 51).astype(np.uint8)
        contours, _ = cv2.findContours(binary * 255, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
        ncc, lab, stats, _ = cv2.connectedComponentsWithStats(binary, connectivity=8)
        kept = []
        for cnt in contours:
            m = cv2.moments(cnt)
            if m["m00"] != 0:
                x0, y0 = cnt[0, 0]
                kept.append((round(m["m00"] * 2), round(m["m10"] * 6), round(m["m01"] * 6), stats[lab[y0, x0], cv2.CC_STAT_AREA]))
        assert n[f] == len(kept)
        for i, ref in enumerate(kept):
            assert tuple(int(v) for v in mom[f, i]) == ref, (f, i)


def test_detect_three_channel_layout_matches_oracle(torch):
    """The drop-in layout (HxWx3, helpers.py:143) incl. cvtColor's fixed-point grey on unequal channels."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(9)
    frames, _, _, _ = synth.make_frame_pool(2, 5, 3, seed=21)
    imgs = []
    for f in frames.reshape(-1, 480, 640):
        img = as3(f)
        img[..., 0] = np.clip(img[..., 0].astype(int) + rng.integers(-30, 30, size=f.shape), 0, 255)
        img[..., 2] = np.clip(img[..., 2].astype(int) + rng.integers(-30, 30, size=f.shape), 0, 255)
        imgs.append(img)
    imgs = np.stack(imgs)
    ctx = _ctx(1, max_blobs=64)
    d = ctx.detect(torch.from_numpy(imgs).cuda())
    port = RefPort([np.eye(3)])
    for i, img in enumerate(imgs):
        ref = [p for p in port.find_dot(img.copy()) if p[0] is not None]
        k = int(d["n"][i])
        assert d["xy"][i, :k].cpu().numpy().tolist() == ref


@pytest.mark.parametrize("threshold", [0, 1, 50, 51, 52, 127, 128, 129, 200, 254, 255])
def test_threshold_is_strictly_greater(torch, threshold):
    """pix > threshold for every byte value (the SWAR compare has two regimes around 128)."""
    img = np.zeros((480, 640), np.uint8)
    for v in range(256):                       # 256 isolated 2x2 squares, one per grey value
        y, x = 8 + 12 * (v // 32), 8 + 12 * (v % 32)
        img[y:y + 2, x:x + 2] = v
    ctx = _ctx(1, max_blobs=64, max_segments=1024)
    d = ctx.detect(torch.from_numpy(img[None]).cuda(), threshold=threshold, want_moments=True)
    expect = 255 - threshold
    n = int(d["n"][0]); flags = int(d["flags"][0])
    assert (n == min(expect, 64)) and ((flags & 2) != 0) == (expect > 64)


@pytest.mark.parametrize("threshold", [0, 51, 127, 128, 129, 254, 255])
def test_three_channel_threshold_regimes(torch, threshold):
    """3-channel stream: the packed "no byte above the threshold" skip must never drop a segment whose grey
    value (cv2's fixed-point RGB2GRAY) passes, in both compare regimes; isolated 2x2 squares of random colours
    plus colours whose grey value sits right at the threshold."""
    import cv2
    rng = np.random.default_rng(threshold + 7)
    img = np.zeros((480, 640, 3), np.uint8)
    cols = rng.integers(0, 256, size=(60, 3), dtype=np.uint8)
    t = min(max(threshold, 1), 254)
    cols[:8] = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [t + 1, t, t], [t, t + 1, t], [t, t, t + 1], [t, t, t], [t + 1] * 3], dtype=np.uint8)
    for v in range(60):
        y, x = 6 + 12 * (v // 20), 6 + 12 * (v % 20)
        img[y:y + 2, x:x + 2] = cols[v]
    grey = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
    expect = int(sum(grey[6 + 12 * (v // 20), 6 + 12 * (v % 20)] > threshold for v in range(60)))
    ctx = _ctx(1, max_blobs=64, max_segments=1024)
    d = ctx.detect(torch.from_numpy(img[None]).cuda(), threshold=threshold)
    assert int(d["n"][0]) == expect and int(d["flags"][0]) == 0


def test_detect_edge_cases(torch):
    ctx = _ctx(1, max_blobs=8, max_segments=64)
    imgs = np.zeros((6, 480, 640), np.uint8)
    imgs[1, 100, 100] = 255                                  # single pixel: zero polygon area -> dropped
    imgs[2, 0:3, 0:3] = 255; imgs[2, 477:480, 637:640] = 255  # blobs touching the image corners
    imgs[3, 10:12, 14:18] = 255                              # blob straddling a 16-px segment boundary
    imgs[4, :, :] = 255                                      # everything set: segment overflow must be flagged
    for k in range(12):                                      # 12 blobs > max_blobs = 8
        imgs[5, 20 + 10 * k: 23 + 10 * k, 50:53] = 255
    d = ctx.detect(torch.from_numpy(imgs).cuda())
    n = d["n"].cpu().numpy(); fl = d["flags"].cpu().numpy(); xy = d["xy"].cpu().numpy()
    assert n[0] == 0 and fl[0] == 0
    assert n[1] == 0 and fl[1] == 0
    assert n[2] == 2 and xy[2, 0].tolist() == [638, 478] and xy[2, 1].tolist() == [1, 1]
    assert n[3] == 1 and xy[3, 0].tolist() == [15, 10]
    assert n[4] == 0 and (fl[4] & 1)
    assert n[5] == 8 and (fl[5] & 2)
    assert xy[5, 0].tolist() == [51, 131]                    # reverse raster order: bottom-most blob first
    # the batch after an overflow must be clean again (segment counters are self-resetting)
    d2 = ctx.detect(torch.from_numpy(imgs[:4]).cuda())
    assert d2["n"].cpu().numpy().tolist() == [0, 0, 2, 1]


# --------------------------------------------------------------------------------------- S2 + S3
@pytest.mark.parametrize("name", PIPE_CASES)
def test_match_triangulate_vs_reference_golden(torch, name):
    z = load_golden(name)
    C = int(z["C"]); B = z["blob_n"].shape[0]
    ctx = _ctx(C, max_blobs=64, max_roots=128)
    ctx.set_cameras([z["K"]] * C, poses_from(z))
    xy = torch.from_numpy(z["blob_xy"].reshape(B * C, 64, 2)).cuda()
    n = torch.from_numpy(z["blob_n"].reshape(B * C)).cuda()
    d = ctx.match_triangulate(xy, n)
    k = d["n"].cpu().numpy()
    assert np.array_equal(k, z["nroot"])                      # same number of kept roots
    assert (d["flags"].cpu().numpy() == 0).all()
    obj = d["obj"].cpu().numpy(); err = d["err"].cpu().numpy()
    worst = 0.0
    for b in range(B):
        worst = max(worst, np.abs(obj[b, :k[b]] - z["obj"][b, :k[b]]).max())
        assert np.allclose(err[b, :k[b]], z["err"][b, :k[b]], rtol=ERR_RTOL, atol=1e-12)
    assert worst <= X_TOL, worst


@pytest.mark.parametrize("name", PIPE_CASES)
def test_full_pipeline_from_pixels_vs_reference_golden(torch, name):
    z = load_golden(name)
    C = int(z["C"]); B = z["blob_n"].shape[0]
    ctx = _ctx(C, max_blobs=64, max_roots=128)
    ctx.set_cameras([z["K"]] * C, poses_from(z))
    out = ctx.pipeline(torch.from_numpy(z["frames"]).cuda())
    k = out["n"].cpu().numpy()
    assert np.array_equal(k, z["nroot"])
    obj = out["obj"].cpu().numpy()
    for b in range(B):
        assert np.abs(obj[b, :k[b]] - z["obj"][b, :k[b]]).max() <= X_TOL
    # host-buffer entry point gives the same bits as the device entry point
    host = ctx.pipeline_host(torch.from_numpy(z["frames"]))
    assert np.array_equal(host["n"].numpy(), k)
    for b in range(B):
        assert np.array_equal(host["obj"].numpy()[b, :k[b]], obj[b, :k[b]])


@pytest.mark.parametrize("name", ["tri_c4", "tri_c8", "tri_c16"])
def test_triangulate_points_vs_reference_golden(torch, name):
    z = load_golden(name)
    C = z["R"].shape[0]
    ctx = _ctx(C)
    ctx.set_cameras([z["K"]] * C, poses_from(z))
    X, err, valid = ctx.triangulate(z["obs"], z["mask"])
    assert valid.all()
    assert np.abs(X - z["X"]).max() <= X_TOL
    assert np.allclose(err, z["err"], rtol=ERR_RTOL, atol=1e-12)
    e2, v2 = ctx.reprojection_errors(z["obs"], z["mask"], z["X"])
    assert np.allclose(e2, z["err"], rtol=ERR_RTOL, atol=1e-12)


def test_matcher_edge_cases_vs_oracle(torch):
    """Empty cameras, camera 0 empty (all roots born later), a lone view, ragged counts."""
    from oracle.ref_port import RefPort
    C = 4
    poses, K = synth.make_rig(C)
    port = RefPort([K] * C)
    ctx = _ctx(C, max_blobs=16, max_roots=32)
    ctx.set_cameras([K] * C, poses)
    rng = np.random.default_rng(3)
    pts3 = rng.uniform(-0.4, 0.4, size=(5, 3)) + np.array([0, 0, 3.0])
    proj = [[list(map(int, synth.project(pts3[i:i + 1], p, K)[0])) for i in range(5)] for p in poses]
    cases = [
        [proj[0], proj[1], proj[2], proj[3]],
        [[], proj[1], proj[2], proj[3]],                      # no roots from camera 0
        [proj[0], [], [], []],                                # single views only -> nothing
        [proj[0][:2], proj[1][:5], [], proj[3][:1]],          # ragged
        [[], [], [], proj[3]],
        [proj[0], proj[1][::-1], proj[2][2:] + proj[2][:2], proj[3]],   # permuted blob order
    ]
    MB = 16
    xy = np.zeros((len(cases), C, MB, 2), np.int32); n = np.zeros((len(cases), C), np.int32)
    for i, case in enumerate(cases):
        for c in range(C):
            n[i, c] = len(case[c])
            if case[c]:
                xy[i, c, :len(case[c])] = case[c]
    d = ctx.match_triangulate(torch.from_numpy(xy.reshape(-1, MB, 2)).cuda(), torch.from_numpy(n.reshape(-1)).cuda(), want_chosen=True)
    for i, case in enumerate(cases):
        e, o, chosen = port.match_and_triangulate([[list(p) for p in cam] for cam in case], poses)
        k = int(d["n"][i])
        assert k == len(e), i
        if k:
            assert np.abs(d["obj"][i, :k].cpu().numpy() - np.asarray(o, dtype=np.float64)).max() <= X_TOL
            assert np.allclose(d["err"][i, :k].cpu().numpy(), e, rtol=ERR_RTOL, atol=1e-12)
            ch = d["chosen"][i, :k].cpu().numpy()
            for r in range(k):                                # identical selected correspondences
                for c in range(C):
                    want = chosen[r][c]
                    got = None if ch[r, c] < 0 else case[c][ch[r, c]]
                    assert (want[0] is None and got is None) or (got is not None and list(want) == list(got))


def test_mirror_functions_match_oracle(torch):
    """The reference-signature layer (api.py) against the oracle port, argument for argument."""
    from oracle.ref_port import RefPort
    C = 3
    obs, poses, K, _ = synth.make_tracks(C, 25, seed=4, missing_frac=0.3)
    port = RefPort([K] * C)
    s = pkg.MocapSession([K] * C)
    X = pkg.triangulate_points(obs, poses, session=s)
    Xr = port.triangulate_many(obs, poses)
    for a, b in zip(X, Xr):
        assert (a[0] is None) == (b[0] is None)
        if a[0] is not None:
            assert np.abs(np.asarray(a, float) - np.asarray(b, float)).max() <= X_TOL
    e = pkg.calculate_reprojection_errors(obs, Xr, poses, session=s)
    assert np.allclose(e, port.reprojection_errors(obs, Xr, poses), rtol=ERR_RTOL)
    assert pkg.triangulate_point([[10, 10], [None, None], [None, None]], poses, session=s) == [None, None, None]
    assert pkg.calculate_reprojection_error([[10, 10], [None, None], [None, None]], [0, 0, 1.0], poses, session=s) is None
    frames, _, poses4, K4 = synth.make_frame_pool(4, 3, 2, seed=8)
    s4 = pkg.MocapSession([K4] * 4)
    port4 = RefPort([K4] * 4)
    for b in range(2):
        pts = []
        for c in range(4):
            img, p = pkg.find_dot(as3(frames[b, c]), session=s4)
            assert p == port4.find_dot(as3(frames[b, c]))
            pts.append(p)
        assert pkg.find_dot(np.zeros((480, 640, 3), np.uint8), session=s4)[1] == [[None, None]]
        e, o, _ = pkg.find_point_correspondance_and_object_points([list(map(list, p)) for p in pts], poses4, [None] * 4, session=s4)
        e2, o2, _ = port4.match_and_triangulate(pts, poses4)
        assert len(e) == len(e2)
        assert np.abs(o - np.asarray(o2, dtype=np.float64)).max() <= X_TOL
        assert np.allclose(e, e2, rtol=ERR_RTOL)


def test_world_transform_epilogue(torch):
    z = load_golden("pipe_c4_m4")
    C = 4; B = z["blob_n"].shape[0]
    ctx = _ctx(C, max_blobs=64, max_roots=128)
    ctx.set_cameras([z["K"]] * C, poses_from(z))
    M = np.array([[0.9, 0.1, 0, 0.3], [-0.1, 0.9, 0.05, -0.2], [0, -0.05, 1.1, 0.7], [0, 0, 0, 1.0]])
    ctx.set_world_transform(M)
    xy = torch.from_numpy(z["blob_xy"].reshape(B * C, 64, 2)).cuda()
    n = torch.from_numpy(z["blob_n"].reshape(B * C)).cuda()
    d = ctx.match_triangulate(xy, n)
    obj = d["obj"].cpu().numpy()
    for b in range(B):
        for r in range(int(z["nroot"][b])):
            p = np.array([[-1, 0, 0], [0, -1, 0], [0, 0, 1]]) @ z["obj"][b, r]      # helpers.py:96-103
            p = M @ np.concatenate((p, [1]))
            p = p[:3] / p[3]
            p[1], p[2] = p[2], p[1]
            assert np.abs(obj[b, r] - p).max() < 1e-9


# ------------------------------------------------------------------- BASELINE-size properties
def test_config2_size_properties(torch):
    """BASELINE config 2 size (4 cameras, 4 markers, 10 000 frame-sets): (i) every replica of a
    frame-set gives bit-identical tracks wherever it sits in the batch, (ii) a permuted batch
    gives the permuted result, (iii) recovered points sit on the ground truth to pixel-quantisation
    accuracy, (iv) the first frame-sets equal the oracle."""
    from oracle.ref_port import RefPort
    C, M, P, B = 4, 4, 50, 10000
    frames, truth, poses, K = synth.make_frame_pool(C, M, P, seed=123)
    ctx = _ctx(C, max_roots=16)
    ctx.set_cameras([K] * C, poses)
    pool = torch.from_numpy(frames).cuda()
    idx = torch.arange(B, device="cuda") % P
    big = pool[idx].contiguous()                                # 12.3 GB resident, >> L2
    out = ctx.pipeline(big)
    torch.cuda.synchronize()
    n = out["n"].cpu().numpy(); obj = out["obj"].cpu().numpy(); err = out["err"].cpu().numpy()
    assert (out["flags"].cpu().numpy() == 0).all()
    for p in range(P):                                          # (i)
        sel = np.arange(p, B, P)
        assert (n[sel] == n[p]).all()
        assert (obj[sel, :n[p]] == obj[p, :n[p]]).all() and (err[sel, :n[p]] == err[p, :n[p]]).all()
    perm = torch.randperm(B, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    out2 = ctx.pipeline(big[perm].contiguous())                 # (ii)
    torch.cuda.synchronize()
    assert torch.equal(out2["n"], out["n"][perm])
    pn = n[perm.cpu().numpy()]
    o2 = out2["obj"].cpu().numpy(); o1 = obj[perm.cpu().numpy()]
    mask = np.arange(obj.shape[1])[None, :] < pn[:, None]
    assert (o2[mask] == o1[mask]).all()
    for p in range(P):                                          # (iii)
        assert n[p] >= M
        for m in range(M):
            dmin = np.linalg.norm(obj[p, :n[p]] - truth[p, m], axis=1).min()
            assert dmin < 0.02, (p, m, dmin)
    port = RefPort([K] * C)                                     # (iv)
    for b in range(3):
        pts = [port.find_dot(as3(frames[b, c])) for c in range(C)]
        e, o, _ = port.match_and_triangulate(pts, poses)
        assert len(e) == n[b]
        assert np.abs(obj[b, :n[b]] - np.asarray(o, dtype=np.float64)).max() <= X_TOL


# ------------------------------------------------------------------------------------------ S4
def _ref_cost(port, poses, obs_obj):
    r = port.ba_residuals(port.poses_to_params(poses), obs_obj)
    return 0.5 * float(np.sum(np.log1p(r.astype(np.float64) ** 2))), r


BA_GOLDEN = ["ba_c4", "ba_c8", "ba_c16"]       # 4 cameras x 40 points, 8 x 60 (config-3 rig), 16 x 96 (config-5 rig)


@pytest.mark.parametrize("name", BA_GOLDEN)
def test_ba_residual_vector_parity(torch, name):
    """SURVEY §7 level (i): the residual vector at identical parameters, after the same float32 cast."""
    z = load_golden(name)
    C = z["mask"].shape[1]
    ctx = _ctx(C)
    start = [{"R": z["R_start"][c], "t": z["t_start"][c]} for c in range(C)]
    ctx.set_cameras([z["K"]] * C, start)
    r = ctx.ba_residuals(z["obs"], z["mask"], start)
    assert r.dtype == np.float32 and r.shape == z["r0"].shape
    assert np.allclose(r, z["r0"], rtol=1e-6, atol=1e-7)
    assert np.mean(r == z["r0"]) > 0.9                       # float32-quantised: almost all bit-equal
    final = [{"R": z["R_final"][c], "t": z["t_final"][c]} for c in range(C)]
    assert np.allclose(ctx.ba_residuals(z["obs"], z["mask"], final), z["rf"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", BA_GOLDEN)
def test_ba_outcome_not_worse_than_reference(torch, name):
    """SURVEY §7 level (ii): final robust cost <= the reference's on the same start (the real reference's
    bundle_adjustment run, golden); the returned cost is re-computed with the oracle; re-triangulated points agree
    with the truth up to the free global scale at least as well as the reference's result; and continuing the
    reference's own iteration from the returned poses does not lower the objective by more than its own stopping
    tolerance (ftol = 1e-2), i.e. the polish was not stopped short."""
    from oracle.ref_port import RefPort
    z = load_golden(name)
    C = z["mask"].shape[1]
    port = RefPort([z["K"]] * C)
    obs_obj = obs_from(z)
    ctx = _ctx(C)
    start = [{"R": z["R_start"][c], "t": z["t_start"][c]} for c in range(C)]
    ctx.set_cameras([z["K"]] * C, start)
    out, rep = ctx.bundle_adjust(z["obs"], z["mask"], start)
    assert abs(rep["cost_initial"] - float(z["cost0"])) < 1e-3 * float(z["cost0"])
    cost_oracle, _ = _ref_cost(port, out, obs_obj)
    assert abs(cost_oracle - rep["cost_final"]) <= 1e-3 * max(1.0, cost_oracle)
    assert cost_oracle <= float(z["costf"])
    assert np.allclose(out[0]["R"], np.eye(3)) and np.allclose(out[0]["t"], 0)        # camera 0 stays pinned
    for p in out:
        assert np.allclose(p["R"] @ p["R"].T, np.eye(3), atol=1e-12)

    truth = np.asarray(port.triangulate_many(obs_obj, [{"R": z["R_true"][c], "t": z["t_true"][c]} for c in range(C)]), dtype=np.float64)

    def scale_free_error(poses):      # camera 0 is pinned, so only the global scale is free
        X = np.asarray(port.triangulate_many(obs_obj, poses), dtype=np.float64)
        s = np.linalg.norm(truth) / np.linalg.norm(X)
        return np.abs(X * s - truth).max()
    ref_final = [{"R": z["R_final"][c], "t": z["t_final"][c]} for c in range(C)]
    assert scale_free_error(out) <= scale_free_error(ref_final) + 1e-9
    assert rep["status"] in (1, 2, 3, 4) and np.isfinite(rep["optimality"])
    # more of the reference's iteration (no prefit) from the result: nothing substantial left to gain
    ctx.set_cameras([z["K"]] * C, out)
    out2, rep2 = ctx.bundle_adjust(z["obs"], z["mask"], out, prefit=False)
    assert rep2["cost_final"] >= rep["cost_final"] * (1.0 - 1e-2) - 1e-9
    assert rep2["cost_final"] <= rep["cost_final"] * (1.0 + 1e-9) + 1e-12      # and it never gets worse


def test_ba_reference_iteration_only(torch):
    """prefit off, float32 finite differences: the reference's own iteration (trajectory is chaotic,
    so only sanity is asserted: cost goes down, scipy-style status, evaluation counts)."""
    z = load_golden("ba_c4")
    C = 4
    ctx = _ctx(C)
    start = [{"R": z["R_start"][c], "t": z["t_start"][c]} for c in range(C)]
    ctx.set_cameras([z["K"]] * C, start)
    lib = ctx.lib
    import ctypes as Ct
    _l = importlib.import_module("low-cost-mocap_b200._lib")
    opt = _l.BAOptions(); lib.mocap_ba_default_options(Ct.byref(opt))
    opt.prefit = 0; opt.jacobian = 0
    rep = _l.BAReport()
    R = np.ascontiguousarray(z["R_start"].copy()); t = np.ascontiguousarray(z["t_start"].copy())
    obs = np.ascontiguousarray(z["obs"]); mask = np.ascontiguousarray(z["mask"])
    st = lib.mocap_bundle_adjust_host(ctx.h, ptr(obs), ptr(mask), obs.shape[0], ptr(R), ptr(t), Ct.byref(opt), Ct.byref(rep))
    assert st == 0
    assert abs(rep.cost_initial - float(z["cost0"])) < 1e-3 * float(z["cost0"])
    assert rep.cost_final < rep.cost_initial and rep.status in (0, 1, 2, 3, 4)
    assert rep.n_fev >= rep.n_iterations + 1 and rep.n_residuals == int(z["r0"].shape[0])


def test_ba_mirror_function(torch):
    z = load_golden("ba_c4")
    C = 4
    s = pkg.MocapSession([z["K"]] * C)
    start = [{"R": z["R_start"][c], "t": z["t_start"][c]} for c in range(C)]

    class Sock:
        def __init__(self): self.events = []
        def emit(self, name, payload): self.events.append((name, payload))
    sock = Sock()
    out = pkg.bundle_adjustment(obs_from(z), start, sock, session=s)
    assert len(out) == C and out[1]["R"].shape == (3, 3) and out[1]["t"].shape == (3,)
    assert sock.events and sock.events[-1][0] == "camera-pose" and len(sock.events[-1][1]["camera_poses"]) == C


def test_ba_config5_size(torch):
    """BASELINE config 5 shape: 16 cameras, 64 markers (x 25 frames = 1600 tracked points, ~10 % views
    missing), cold start from perturbed poses.  Properties: robust cost falls by orders of magnitude and
    the scale-free geometry matches the truth."""
    from oracle.ref_port import RefPort
    C, F = 16, 1600
    obs_obj, poses, K, pts = synth.make_tracks(C, F, seed=77, missing_frac=0.1)
    start = synth.perturb_poses(poses, seed=78)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    ctx = _ctx(C)
    ctx.set_cameras([K] * C, start)
    out, rep = ctx.bundle_adjust(obs, mask, start)
    assert rep["n_residuals"] == F
    assert rep["cost_final"] < 1e-2 * rep["cost_initial"]
    ctx.set_cameras([K] * C, out)
    X, _, valid = ctx.triangulate(obs, mask)
    s = np.linalg.norm(pts - pts.mean(0)) / np.linalg.norm(X - X.mean(0))
    # similarity alignment (scale + rigid) via Procrustes
    A = (X - X.mean(0)) * s; Bm = pts - pts.mean(0)
    U, _, Vt = np.linalg.svd(A.T @ Bm)
    Rm = (U @ Vt)
    assert np.abs(A @ Rm - Bm).max() < 0.02


def test_detect_large_image_wide_accumulators(torch):
    """1024x768: moment sums exceed 32 bits, so the 64-bit accumulator kernels run; irregular blobs far
    from the origin (largest sums), incl. one wider than a warp's segment budget (full-size fallback)."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(12)
    H, W = 768, 1024
    imgs = np.zeros((3, H, W), np.uint8)
    for f in range(3):
        for _ in range(10):
            cx, cy = rng.integers(W - 200, W - 30), rng.integers(H - 200, H - 30)
            yy, xx = np.mgrid[-20:21, -20:21]
            r = rng.uniform(3, 12)
            disc = (xx * xx + yy * yy) <= r * r
            ys, xs = np.nonzero(disc)
            imgs[f, np.clip(cy + ys - 20, 0, H - 1), np.clip(cx + xs - 20, 0, W - 1)] = 255
        imgs[f, 40:120, 30:700] = 200                    # 80 rows x 42 segments: > 128 segments, < max_segments
    ctx = pkg.MocapContext(1, W, H, max_blobs=64, max_segments=4096)
    d = ctx.detect(torch.from_numpy(imgs).cuda())
    port = RefPort([np.eye(3)])
    for f in range(3):
        ref = [p for p in port.find_dot(as3(imgs[f])) if p[0] is not None]
        k = int(d["n"][f])
        assert int(d["flags"][f]) == 0
        assert d["xy"][f, :k].cpu().numpy().tolist() == ref


def test_fused_and_split_pipelines_agree(torch, monkeypatch):
    """The single fused kernel (default) and the three-kernel pipeline give identical bits, including
    frame-sets whose images exceed the warp-level capacities (worklist fallbacks)."""
    z = load_golden("pipe_c4_m4")
    C = 4
    frames = z["frames"][:8].copy()
    frames[1, 2, 100:160, 40:600] = 255          # 60 rows x 36 segments: deferred image -> deferred set
    frames[5, 0, 300:304, 100:400] = 255         # long thin blob, fits a warp
    for b in (2, 6):                             # > 64 blobs in one image: exceeds a warp's accumulators
        for k in range(70):
            y, x = 10 + 6 * (k // 35), 20 + 16 * (k % 35)
            frames[b, 1, y:y + 3, x:x + 3] = 255
    results = {}
    for mode in ("fused", "split"):
        monkeypatch.setenv("MOCAP_PIPELINE", mode)
        ctx = _ctx(C, max_blobs=64, max_roots=128, max_segments=4096)
        ctx.set_cameras([z["K"]] * C, poses_from(z))
        out = ctx.pipeline(torch.from_numpy(frames).cuda())
        torch.cuda.synchronize()
        results[mode] = {k: v.cpu().numpy().copy() for k, v in out.items()}
        # a second pass on the same context must be identical (self-resetting counters / worklists)
        out2 = ctx.pipeline(torch.from_numpy(frames).cuda())
        torch.cuda.synchronize()
        assert np.array_equal(out2["n"].cpu().numpy(), results[mode]["n"])
    a, b = results["fused"], results["split"]
    assert np.array_equal(a["n"], b["n"]) and np.array_equal(a["flags"], b["flags"])
    for s in range(len(frames)):
        k = a["n"][s]
        assert np.array_equal(a["obj"][s, :k], b["obj"][s, :k]) and np.array_equal(a["err"][s, :k], b["err"][s, :k])
    # the untouched frame-sets still match the reference golden
    for s in (0, 3, 4, 7):
        k = int(z["nroot"][s])
        assert a["n"][s] == k and np.abs(a["obj"][s, :k] - z["obj"][s, :k]).max() <= X_TOL


def test_locate_objects_vs_oracle(torch):
    """SURVEY §8(f) #3: marker triplets -> drone records, batched on the GPU, against the oracle port
    (pinned to the live reference in tests/test_oracle_pinned.py): pos and error bit-exact, heading within 4 ulp of
    pi/2.  tests/test_gpu_locate.py owns the locator's edges; this is the well-separated case next to the pipeline."""
    from oracle.ref_port import RefPort
    ctx = _ctx(2, max_roots=32)
    B, R, MO = 60, 32, 6
    obj = np.zeros((B, R, 3)); err = np.zeros((B, R)); n = np.zeros((B,), np.int32)
    scenes = []
    for b in range(B):
        pts, errs = synth.make_drone_points(b % 4, b % 7, seed=100 + b)
        if b == 7:
            pts, errs = pts[:0], errs[:0]                      # empty frame-set
        scenes.append((pts, errs))
        n[b] = len(pts); obj[b, :len(pts)] = pts; err[b, :len(pts)] = errs
    d = ctx.locate_objects(torch.from_numpy(obj).cuda(), torch.from_numpy(err).cuda(), torch.from_numpy(n).cuda(), max_objects=MO)
    cnt = d["n"].cpu().numpy(); rec = d["objects"].cpu().numpy(); di = d["drone_index"].cpu().numpy()
    total = 0
    for b, (pts, errs) in enumerate(scenes):
        ref = RefPort.locate_objects(pts, errs) if len(pts) else []
        assert cnt[b] == len(ref), b
        total += len(ref)
        for k, o in enumerate(ref):
            assert np.array_equal(rec[b, k, :3], o["pos"]) and rec[b, k, 4] == o["error"]
            assert abs(rec[b, k, 3] - o["heading"]) <= 4 * np.spacing(np.pi / 2)
            assert di[b, k] == o["droneIndex"]
    assert total > 60
    s = pkg.MocapSession([np.eye(3)] * 2)
    pts, errs = synth.make_drone_points(2, 3, seed=5)
    got = pkg.locate_objects(pts, errs, session=s)
    ref = RefPort.locate_objects(pts, errs)
    assert len(got) == len(ref) == 2 and all(g["droneIndex"] == r["droneIndex"] for g, r in zip(got, ref))
    assert pkg.locate_objects(np.zeros((0, 3)), np.zeros(0), session=s) == []


def test_config3_shape_pipeline_then_batch_ba(torch):
    """BASELINE config 3 shape (8 cameras, 16 markers; 150 frame-sets here): S1 -> S2+S3 with the
    selected correspondences -> S4 on the batch's tracks from perturbed poses.  The adjusted rig must
    explain the tracks at least as well as the true rig does, under the reference's own objective."""
    C, M, B = 8, 16, 150
    frames, truth, poses, K = synth.make_frame_pool(C, M, B, seed=31)
    ctx = _ctx(C, max_roots=64)
    ctx.set_cameras([K] * C, poses)
    d = ctx.detect(torch.from_numpy(frames).cuda())
    m = ctx.match_triangulate(d["xy"], d["n"], want_chosen=True)
    assert (m["flags"].cpu().numpy() == 0).all() and (d["flags"].cpu().numpy() == 0).all()
    obs, mask = ctx.tracks_to_observations(d["xy"], m["n"], m["chosen"])
    P = int(m["n"].sum())
    assert obs.shape == (P, C, 2) and mask.shape == (P, C) and (mask.sum(1) >= 2).all()
    # the observations really are the blobs the matcher chose: re-triangulating them gives the same points
    X, _, valid = ctx.triangulate(obs, mask)
    Xm = np.concatenate([m["obj"][b, :int(m["n"][b])].cpu().numpy() for b in range(B)])
    assert valid.all() and np.abs(X - Xm).max() < 1e-9
    start = synth.perturb_poses(poses, seed=32)
    ctx.set_cameras([K] * C, start)
    out, rep = ctx.bundle_adjust(obs, mask, start)
    true_cost = 0.5 * np.sum(np.log1p(ctx.ba_residuals(obs, mask, poses).astype(np.float64) ** 2))
    assert rep["cost_final"] <= true_cost * 1.05 + 1e-6 and rep["cost_final"] < 1e-2 * rep["cost_initial"]


def test_preprocess_bit_exact_vs_cv2_chain(torch):
    """SURVEY §8(f) #2: rot90 -> make_square -> undistort -> GaussianBlur 9x9 -> filter2D 5x5 -> RGB2BGR in one
    kernel, bit-exact against the reference's cv2 chain (oracle port) on worst-case random-noise frames and
    on marker-like frames; then S1 on the processed frames equals the reference's _find_dot."""
    import json, os
    from oracle.ref_port import RefPort
    K = np.array([[320.0, 0, 160], [0, 320, 160], [0, 0, 1]])
    dist = [-1.26372388e-01, 2.62661497e-01, 1.21306197e-03, 2.24507008e-04, -2.48534118e-01]   # camera-params.json
    C = 2
    ctx = pkg.MocapContext(C, 320, 320, max_blobs=64)
    ctx.set_preprocess(320, 240, [0, 2], [K, K], [dist, [d * 0.5 for d in dist]])
    port = RefPort([K, K])
    # the fixed-point undistortion map equals cv2's
    import cv2
    for cam, dd in ((0, dist), (1, [d * 0.5 for d in dist])):
        m1, m2 = ctx.undistort_map(cam)
        r1, r2 = cv2.initUndistortRectifyMap(K, np.array(dd), np.eye(3), K, (320, 320), cv2.CV_16SC2)
        assert np.array_equal(m1, r1) and np.array_equal(m2, r2)
    rng = np.random.default_rng(4)
    raw = rng.integers(0, 256, size=(3, C, 240, 320, 3), dtype=np.uint8)
    # marker-like frames: dark clutter + bright Gaussian spots (stay solid through blur + sharpen; hard-edged discs
    # turn into rings, i.e. blobs with holes: tests/test_gpu_holes.py runs those through the raw-frame chain)
    yy, xx = np.mgrid[:240, :320]
    for b in range(1, 3):
        raw[b] = rng.integers(0, 30, size=(C, 240, 320, 3), dtype=np.uint8)
        for c in range(C):
            for _ in range(6):
                cy, cx, sg = rng.uniform(20, 220), rng.uniform(20, 300), rng.uniform(1.5, 4.0)
                spot = (255 * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sg * sg))).astype(np.uint8)
                raw[b, c] = np.maximum(raw[b, c], spot[:, :, None])
    out = ctx.preprocess(torch.from_numpy(raw).cuda())
    got = out.cpu().numpy().reshape(3, C, 320, 320, 3)
    for b in range(3):
        for c, (dd, rot) in enumerate(((dist, 0), ([d * 0.5 for d in dist], 2))):
            ref = port.preprocess(raw[b, c], c, dd, rot)
            assert np.array_equal(got[b, c], ref), (b, c, int((got[b, c] != ref).sum()))
    det = ctx.detect(out)
    for i in range(C, 3 * C):                      # the marker-like frames (the noise frame is all clutter)
        assert int(det["flags"][i]) == 0
        ref_pts = [p for p in port.find_dot(got.reshape(-1, 320, 320, 3)[i].copy()) if p[0] is not None]
        k = int(det["n"][i])
        assert det["xy"][i, :k].cpu().numpy().tolist() == ref_pts


def test_calibrate_init_vs_oracle(torch):
    """SURVEY §8(f) #4.  (i) Given the reference's own fundamental matrices (cv2 RANSAC, seeded) the essential
    decomposition, cheirality vote and pose chain equal the reference's (index.py:247-265).  (ii) With the
    deterministic 8-point estimator the chain is at least as close to the truth, and after bundle adjustment
    the rig explains the tracks as well as the adjusted reference chain does."""
    from oracle.ref_port import RefPort
    C = 4
    obs_obj, poses, K, pts = synth.make_tracks(C, 80, seed=14, missing_frac=0.1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    port = RefPort([K] * C)
    ref_chain, Fs = port.calibrate_init(obs_obj.tolist(), rng_seed=0, return_F=True)
    ctx = _ctx(C)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    chain, F_used, votes = ctx.calibrate_init(obs, mask, F_given=np.stack(Fs))
    assert np.allclose(F_used, np.stack(Fs))
    for a, b in zip(chain, ref_chain):                           # (i)
        assert np.abs(a["R"] - np.asarray(b["R"], dtype=np.float64)).max() < 1e-8
        assert np.abs(a["t"] - np.asarray(b["t"], dtype=np.float64).ravel()).max() < 1e-8
    assert (votes.max(axis=1) > 0).all()

    def rot_err_deg(chain_):
        errs = []
        for c in range(1, C):
            Rt, Re = np.asarray(poses[c]["R"]), np.asarray(chain_[c]["R"], dtype=np.float64)
            errs.append(np.degrees(np.arccos(np.clip((np.trace(Rt.T @ Re) - 1) / 2, -1, 1))))
        return max(errs)
    own, F_own, _ = ctx.calibrate_init(obs, mask)                # (ii)
    assert rot_err_deg(own) <= rot_err_deg(ref_chain) + 0.5
    for c in range(C - 1):                                       # epipolar constraint holds on the tracks
        both = (mask[:, c] & mask[:, c + 1]).astype(bool)
        x1 = np.c_[obs[both, c], np.ones(both.sum())]; x2 = np.c_[obs[both, c + 1], np.ones(both.sum())]
        l = x1 @ F_own[c].T
        d = np.abs(np.sum(x2 * l, axis=1)) / np.sqrt(l[:, 0] ** 2 + l[:, 1] ** 2)
        assert np.median(d) < 1.0
    s = pkg.MocapSession([K] * C)
    final = pkg.calculate_camera_poses(obs_obj.tolist(), session=s)
    ctx.set_cameras([K] * C, final)
    cost_own = 0.5 * np.sum(np.log1p(ctx.ba_residuals(obs, mask, final).astype(np.float64) ** 2))
    ref_start = [{"R": np.asarray(p["R"], dtype=np.float64), "t": np.asarray(p["t"], dtype=np.float64).ravel()} for p in ref_chain]
    ctx.set_cameras([K] * C, ref_start)
    adj_ref, rep = ctx.bundle_adjust(obs, mask, ref_start)
    assert cost_own <= rep["cost_final"] * 1.05 + 1e-6
    ctx.set_cameras([K] * C, final)
    X, _, valid = ctx.triangulate(obs, mask)
    A = X - X.mean(0); Bm = pts - pts.mean(0)
    A *= np.linalg.norm(Bm) / np.linalg.norm(A)
    U, _, Vt = np.linalg.svd(A.T @ Bm)
    assert np.abs(A @ (U @ Vt) - Bm).max() < 0.03


def test_plain_c_example_runs(torch, tmp_path):
    """examples/pipeline_host.c (what a cgo / JNI binding would call) through the host entry point."""
    import os, subprocess
    from tests.util import ROOT
    lib_dir = os.path.join(ROOT, "low-cost-mocap_b200")
    exe = tmp_path / "pipeline_host"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "pipeline_host.c"),
                           "-L", lib_dir, "-lmocap_b200", "-Wl,-rpath," + lib_dir, "-o", str(exe)])
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    lines = [l for l in r.stdout.splitlines() if l.startswith("frame-set")]
    assert len(lines) == 4
    for l in lines:
        x, y, z = [float(v) for v in l.split(":")[1].split()[:3]]
        assert abs(x - 0.1) < 0.01 and abs(y - 0.05) < 0.01 and abs(z - 3.0) < 0.05


def test_raw_frames_to_tracks_vs_oracle_chain(torch):
    """helpers.py:70-103 end to end on raw camera frames: preprocess -> _find_dot -> matcher, one C-ABI call,
    against the same chain of the oracle port."""
    from oracle.ref_port import RefPort
    C = 2
    K = np.array([[320.0, 0, 160], [0, 320, 160], [0, 0, 1]])
    dist = [-1.26372388e-01, 2.62661497e-01, 1.21306197e-03, 2.24507008e-04, -2.48534118e-01]
    poses = [{"R": np.eye(3), "t": np.zeros(3)}, {"R": np.eye(3), "t": np.array([-0.4, 0.0, 0.0])}]
    rng = np.random.default_rng(8)
    B = 3
    raw = rng.integers(0, 25, size=(B, C, 240, 320, 3), dtype=np.uint8)
    yy, xx = np.mgrid[:240, :320]
    for b in range(B):
        for m in range(3):
            X = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.25, 0.25), rng.uniform(2.0, 3.0)])
            for c in range(C):
                pc = poses[c]["R"] @ X + poses[c]["t"]
                u, v = 320 * pc[0] / pc[2] + 160, 320 * pc[1] / pc[2] + 160 - 40      # row offset of make_square
                spot = (255 * np.exp(-((yy - v) ** 2 + (xx - u) ** 2) / (2 * 2.0 ** 2))).astype(np.uint8)
                raw[b, c] = np.maximum(raw[b, c], spot[:, :, None])
    ctx = pkg.MocapContext(C, 320, 320, max_blobs=32, max_roots=32)
    ctx.set_preprocess(320, 240, [0, 0], [K, K], [dist, dist])
    ctx.set_cameras([K, K], poses)
    out = ctx.pipeline_raw(torch.from_numpy(raw).cuda(), want_frames=True)
    port = RefPort([K, K])
    n = out["n"].cpu().numpy(); obj = out["obj"].cpu().numpy(); frames = out["frames"].cpu().numpy()
    total = 0
    for b in range(B):
        pts = []
        for c in range(C):
            f = port.preprocess(raw[b, c], c, dist, 0)
            assert np.array_equal(frames[b, c], f)
            pts.append(port.find_dot(f.copy()))
        e, o, _ = port.match_and_triangulate(pts, poses)
        assert n[b] == len(e)
        total += len(e)
        if len(e):
            assert np.abs(obj[b, :n[b]] - np.asarray(o, dtype=np.float64)).max() <= X_TOL
    assert total >= B
    out2 = ctx.pipeline_raw(torch.from_numpy(raw).cuda())              # without keeping the frames
    assert np.array_equal(out2["n"].cpu().numpy(), n)
    assert np.array_equal(out2["obj"].cpu().numpy()[:, :n.max()], obj[:, :n.max()])
    # other entry points grow and reuse the context's scratch memory; the preprocessing tables must survive that
    # (they were once freed with it), and a much larger batch (several launch groups) must agree with the small one
    big = 200000
    ctx.triangulate(np.full((big, C, 2), 100.0), np.ones((big, C), dtype=np.uint8))
    reps = 700
    out3 = ctx.pipeline_raw(torch.from_numpy(np.tile(raw, (reps, 1, 1, 1, 1))).cuda())
    assert np.array_equal(out3["n"].cpu().numpy(), np.tile(n, reps))
    assert np.array_equal(out3["obj"].cpu().numpy()[:B, :n.max()], obj[:, :n.max()])


@pytest.mark.parametrize("shape", [(320, 320, 3), (1024, 768, 1), (640, 480, 6), (48, 32, 2)])
def test_fused_pipeline_other_geometries(torch, monkeypatch, shape):
    """The fused kernel on image sizes whose segment count is not a multiple of a warp iteration (ragged
    slices), on the 64-bit-accumulator variant, on tiny frames and on other camera counts: identical to the
    three-kernel pipeline, and S1 identical to the oracle."""
    from oracle.ref_port import RefPort
    W, H, C = shape
    rng = np.random.default_rng(W + H + C)
    B = 5
    frames = rng.integers(0, 40, size=(B, C, H, W), dtype=np.uint8)
    yy, xx = np.mgrid[:H, :W]
    for b in range(B):
        for c in range(C):
            for _ in range(4):
                cy, cx, sg = rng.uniform(4, H - 4), rng.uniform(4, W - 4), rng.uniform(1.0, 2.5)
                spot = (255 * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sg * sg))).astype(np.uint8)
                frames[b, c] = np.maximum(frames[b, c], spot)
    poses = [{"R": np.eye(3), "t": np.array([-0.3 * c, 0.0, 0.0])} for c in range(C)]
    K = np.array([[W * 0.9, 0, W / 2], [0, W * 0.9, H / 2], [0, 0, 1.0]])
    res = {}
    for mode in ("fused", "split"):
        monkeypatch.setenv("MOCAP_PIPELINE", mode)
        ctx = pkg.MocapContext(C, W, H, max_blobs=32, max_roots=64)
        ctx.set_cameras([K] * C, poses)
        out = ctx.pipeline(torch.from_numpy(frames).cuda())
        torch.cuda.synchronize()
        res[mode] = {k: v.cpu().numpy().copy() for k, v in out.items()}
        if mode == "split":
            d = ctx.detect(torch.from_numpy(frames).cuda())
            port = RefPort([K] * C)
            for i in range(B * C):
                ref = [p for p in port.find_dot(as3(frames.reshape(-1, H, W)[i])) if p[0] is not None]
                k = int(d["n"][i])
                assert d["xy"][i, :k].cpu().numpy().tolist() == ref
    a, b = res["fused"], res["split"]
    assert np.array_equal(a["n"], b["n"]) and np.array_equal(a["flags"], b["flags"])
    for s in range(B):
        k = a["n"][s]
        assert np.array_equal(a["obj"][s, :k], b["obj"][s, :k]) and np.array_equal(a["err"][s, :k], b["err"][s, :k])


def _random_solid_frame(rng, H, W, n_shapes):
    import cv2
    img = np.zeros((H, W), np.uint8)
    for _ in range(n_shapes):
        cx, cy = int(rng.integers(3, W - 3)), int(rng.integers(3, H - 3))
        kind = int(rng.integers(0, 4))
        val = int(rng.integers(52, 256))
        if kind == 0:
            cv2.ellipse(img, (cx, cy), (int(rng.integers(1, 9)), int(rng.integers(1, 9))), float(rng.uniform(0, 180)), 0, 360, val, -1)
        elif kind == 1:
            x = y = 0
            for _ in range(int(rng.integers(3, 40))):
                px, py = np.clip(cx + x, 0, W - 1), np.clip(cy + y, 0, H - 1)
                img[py, px] = val
                x += int(rng.integers(-1, 2)); y += int(rng.integers(-1, 2))
        elif kind == 2:
            pts = (np.array([[cx, cy]]) + rng.integers(-8, 9, size=(int(rng.integers(3, 7)), 2))).astype(np.int32)
            cv2.fillPoly(img, [pts], val)
        else:
            img[cy:cy + int(rng.integers(1, 6)), cx:cx + int(rng.integers(1, 20))] = val
    binary = (img > 51).astype(np.uint8)                 # fill holes: this fuzz is of solid blobs (holed ones: test_gpu_holes.py)
    ff = binary.copy()
    cv2.floodFill(ff, np.zeros((H + 2, W + 2), np.uint8), (0, 0), 1)
    if binary[0, 0]:
        return None
    img[ff == 0] = 255
    return np.maximum(img, rng.integers(0, 52, size=(H, W), dtype=np.uint8))


def test_blob_detector_fuzz_vs_cv2(torch):
    """400 random frames of random solid shapes (ellipses, random walks, polygons, bars; touching, nested in
    concavities, on the border, 1 px wide): centres, count and order identical to cv2's findContours + moments."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(2024)
    H, W = 96, 160
    frames = []
    while len(frames) < 400:
        f = _random_solid_frame(rng, H, W, int(rng.integers(1, 14)))
        if f is not None:
            frames.append(f)
    frames = np.stack(frames)
    ctx = pkg.MocapContext(1, W, H, max_blobs=64, max_segments=1024)
    d = ctx.detect(torch.from_numpy(frames).cuda())
    n = d["n"].cpu().numpy(); xy = d["xy"].cpu().numpy(); fl = d["flags"].cpu().numpy()
    port = RefPort([np.eye(3)])
    blobs = 0
    for i, f in enumerate(frames):
        ref = [p for p in port.find_dot(as3(f)) if p[0] is not None]
        assert fl[i] == 0
        assert xy[i, :n[i]].tolist() == ref, i
        blobs += len(ref)
    assert blobs > 1500


def test_matcher_fuzz_vs_oracle(torch):
    """Random blob constellations that do not come from any scene (many wrong correspondences, ragged counts,
    near-threshold distances to epipolar lines): the kept roots, their order and the chosen points equal the oracle's."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(77)
    for C in (3, 5):
        poses, K = synth.make_rig(C)
        port = RefPort([K] * C)
        ctx = _ctx(C, max_blobs=16, max_roots=64, max_cands=16)
        ctx.set_cameras([K] * C, poses)
        B, MB = 60, 16
        xy = np.zeros((B, C, MB, 2), np.int32); n = np.zeros((B, C), np.int32)
        for b in range(B):
            # half consistent (a few real 3D points), half clutter
            pts3 = rng.uniform(-0.5, 0.5, size=(int(rng.integers(0, 5)), 3)) + np.array([0, 0, 3.0])
            for c in range(C):
                lst = [list(map(int, synth.project(p[None], poses[c], K)[0])) for p in pts3 if rng.uniform() < 0.85]
                lst += [[int(rng.integers(100, 540)), int(rng.integers(100, 380))] for _ in range(int(rng.integers(0, 4)))]
                seen, uniq = set(), []
                for p in lst:
                    if tuple(p) not in seen:
                        seen.add(tuple(p)); uniq.append(p)
                order = rng.permutation(len(uniq))
                uniq = [uniq[i] for i in order][:MB]
                n[b, c] = len(uniq)
                if uniq:
                    xy[b, c, :len(uniq)] = uniq
        d = ctx.match_triangulate(torch.from_numpy(xy.reshape(-1, MB, 2)).cuda(), torch.from_numpy(n.reshape(-1)).cuda())
        cnt = d["n"].cpu().numpy(); obj = d["obj"].cpu().numpy(); err = d["err"].cpu().numpy()
        assert (d["flags"].cpu().numpy() == 0).all()
        for b in range(B):
            lists = [[list(map(int, xy[b, c, i])) for i in range(n[b, c])] for c in range(C)]
            e, o, _ = port.match_and_triangulate(lists, poses)
            assert cnt[b] == len(e), (C, b)
            if len(e):
                # wrong correspondences give ill-conditioned triangulations: compare with a relative bar there
                ref = np.asarray(o, dtype=np.float64)
                scale = np.maximum(1.0, np.abs(ref).max(axis=1, keepdims=True))
                assert (np.abs(obj[b, :cnt[b]] - ref) / scale).max() <= 1e-6, (C, b)
                assert np.allclose(err[b, :cnt[b]], e, rtol=1e-6, atol=1e-9)


def test_matcher_heavy_fuzz_8_cameras(torch):
    """The heavy regime of BASELINE configs 3/4: 8 cameras, 16-24 blobs per camera (16 markers seen by most cameras
    plus clutter), candidate lists of up to 16 per epipolar line, hundreds of candidate groups per frame-set.  Kept
    roots, their order, the chosen points and errors equal the oracle's; no capacity flag at max_cands = 16."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(99)
    C, B, MB = 8, 24, 32
    poses, K = synth.make_rig(C)
    port = RefPort([K] * C)
    ctx = _ctx(C, max_blobs=MB, max_roots=128, max_cands=16, max_groups=1 << 16)
    ctx.set_cameras([K] * C, poses)
    xy = np.zeros((B, C, MB, 2), np.int32); n = np.zeros((B, C), np.int32)
    for b in range(B):
        pts3 = rng.uniform(-0.5, 0.5, size=(16, 3)) + np.array([0, 0, 3.0])
        for c in range(C):
            lst = [list(map(int, synth.project(p[None], poses[c], K)[0])) for p in pts3 if rng.uniform() < 0.9]
            lst += [[int(rng.integers(100, 540)), int(rng.integers(100, 380))] for _ in range(int(rng.integers(2, 9)))]
            seen, uniq = set(), []
            for p in lst:
                if tuple(p) not in seen and 0 <= p[0] < 640 and 0 <= p[1] < 480:
                    seen.add(tuple(p)); uniq.append(p)
            order = rng.permutation(len(uniq))
            uniq = [uniq[i] for i in order][:MB]
            n[b, c] = len(uniq)
            xy[b, c, :len(uniq)] = uniq
    assert n.mean() >= 16
    d = ctx.match_triangulate(torch.from_numpy(xy.reshape(-1, MB, 2)).cuda(), torch.from_numpy(n.reshape(-1)).cuda())
    cnt = d["n"].cpu().numpy(); obj = d["obj"].cpu().numpy(); err = d["err"].cpu().numpy()
    assert (d["flags"].cpu().numpy() == 0).all()
    for b in range(B):
        lists = [[list(map(int, xy[b, c, i])) for i in range(n[b, c])] for c in range(C)]
        e, o, _ = port.match_and_triangulate(lists, poses)
        assert cnt[b] == len(e), b
        ref = np.asarray(o, dtype=np.float64)
        scale = np.maximum(1.0, np.abs(ref).max(axis=1, keepdims=True))
        assert (np.abs(obj[b, :cnt[b]] - ref) / scale).max() <= 1e-6, b
        assert np.allclose(err[b, :cnt[b]], e, rtol=1e-6, atol=1e-9)


def test_install_into_patches_a_helpers_like_module(torch):
    """install_into() on a stand-in for the reference's helpers module (same attribute surface: the Cameras
    singleton with camera_params, and the module-level hot-path functions): afterwards the module's own names
    run on the CUDA path with the reference's argument and return conventions."""
    import types
    from oracle.ref_port import RefPort
    C = 4
    frames, truth, poses, K = synth.make_frame_pool(C, 3, 1, seed=17)

    class _Cams:
        camera_params = [{"intrinsic_matrix": K.tolist(), "distortion_coef": [0] * 5, "rotation": 0} for _ in range(C)]

    class Cameras:
        _inst = _Cams()

        @classmethod
        def instance(cls):
            return cls._inst

        def _find_dot(self, img):
            raise AssertionError("not patched")
    helpers = types.ModuleType("helpers_standin")
    helpers.Cameras = Cameras
    for name in ("triangulate_point", "triangulate_points", "calculate_reprojection_error", "calculate_reprojection_errors",
                 "find_point_correspondance_and_object_points", "bundle_adjustment", "locate_objects"):
        setattr(helpers, name, None)
    pkg.install_into(helpers)
    port = RefPort([K] * C)
    image_points = []
    for c in range(C):
        img, pts = helpers.Cameras.instance()._find_dot(as3(frames[0, c]))
        assert img.shape == (480, 640, 3) and pts == port.find_dot(as3(frames[0, c]))
        image_points.append(pts)
    errors, object_points, fr = helpers.find_point_correspondance_and_object_points([list(map(list, p)) for p in image_points], poses, [None] * C)
    e2, o2, _ = port.match_and_triangulate(image_points, poses)
    assert isinstance(errors, np.ndarray) and object_points.shape == (len(e2), 3)
    assert np.abs(object_points - np.asarray(o2, dtype=np.float64)).max() <= X_TOL
    X = helpers.triangulate_points([[p[0] for p in image_points]], poses)
    assert X.shape == (1, 3)
    assert helpers.calculate_reprojection_errors([[p[0] for p in image_points]], X, poses).shape == (1,)
    assert helpers.locate_objects(object_points, errors) == []


def test_error_behaviour(torch):
    """C-ABI status codes surface as MocapError with the library's message; nothing falls back silently."""
    with pytest.raises(pkg.MocapError):
        pkg.MocapContext(0)                                    # invalid configuration
    with pytest.raises(pkg.MocapError):
        pkg.MocapContext(4, 641, 480)                          # width must be a multiple of 16
    ctx = _ctx(2)
    frames = torch.zeros((1, 2, 480, 640), dtype=torch.uint8, device="cuda")
    with pytest.raises(pkg.MocapError) as ei:
        ctx.pipeline(frames)                                   # cameras not set
    assert "mocap_set_cameras" in str(ei.value)
    with pytest.raises(pkg.MocapError):
        ctx.preprocess(torch.zeros((2, 240, 320, 3), dtype=torch.uint8, device="cuda"))   # preprocessing not set
    with pytest.raises(pkg.MocapError):
        ctx.set_preprocess(320, 240, [0, 0], [np.eye(3)] * 2, [[0] * 5] * 2)              # context is not square
    ctx.set_cameras([np.eye(3)] * 2, [{"R": np.eye(3), "t": np.zeros(3)}] * 2)
    out = ctx.pipeline(frames)                                 # empty frames: zero points, no error
    assert int(out["n"][0]) == 0 and int(out["flags"][0]) == 0


def test_heavy_batches_take_the_three_kernel_pipeline(torch, monkeypatch):
    """With MOCAP_PIPELINE unset the context picks the pipeline per batch from the blob count of the previous
    batch (mapped host memory, no synchronisation): light frame-sets stay on the single-pass kernel (3 launches
    per batch), heavy ones (8 cameras x 16 markers) move to the three-kernel pipeline (5 launches: pixel stream, warp-level and
    full-size blob reduction, matcher, the matcher's items of heavy frame-sets) from the second batch on -- with
    identical results."""
    monkeypatch.delenv("MOCAP_PIPELINE", raising=False)
    for C, M, heavy in ((8, 16, True), (4, 4, False)):
        frames, truth, poses, K = synth.make_frame_pool(C, M, 6, seed=3)
        ctx = pkg.MocapContext(C, 640, 480, max_roots=64)
        ctx.set_cameras([K] * C, poses)
        batch = torch.from_numpy(frames).cuda()
        outs, launches = [], []
        for _ in range(3):
            before = ctx.launch_count()
            o = ctx.pipeline(batch)
            torch.cuda.synchronize()
            launches.append(ctx.launch_count() - before)
            outs.append({k: v.cpu().numpy() for k, v in o.items()})
        split = 5 if os.environ.get("MOCAP_MATCH_CHUNK", "") != "0" else 4
        assert launches[0] == 3 and launches[1] == launches[2] == (split if heavy else 3), launches
        n = outs[0]["n"]
        assert n.sum() > 0
        for o in outs[1:]:
            assert np.array_equal(o["n"], n) and np.array_equal(o["flags"], outs[0]["flags"])
            for b in range(len(n)):
                assert np.array_equal(o["obj"][b, :n[b]], outs[0]["obj"][b, :n[b]])
                assert np.array_equal(o["err"][b, :n[b]], outs[0]["err"][b, :n[b]])


# ---------------------------------------------------------------------------------------------------------------
# S4 wholly on the device: k_ba_solve (one cooperative launch) behind mocap_bundle_adjust_dev / _host
# ---------------------------------------------------------------------------------------------------------------
def _tracks_case(C, F, seed):
    obs_obj, poses, K, pts = synth.make_tracks(C, F, seed=seed, missing_frac=0.1)
    start = synth.perturb_poses(poses, seed=seed + 1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    return obs, mask, poses, start, K, pts


@pytest.mark.parametrize("C,F,prefit", [(4, 40, True), (4, 40, False), (8, 1500, True), (16, 800, True), (2, 64, True), (3, 200, True)])
def test_ba_device_engine_agrees_with_host_stepped(torch, C, F, prefit):
    """The persistent grid-synchronous solve (engine 0) against the host-stepped solve (engine 1: optimiser control
    of trf_core.h on the host, one launch per phase): same algorithm, so the same iteration counts, the same final
    cost and the same poses up to the rounding of differently ordered sums."""
    if C == 4:
        z = load_golden("ba_c4")
        obs, mask, K = z["obs"], z["mask"], z["K"]
        start = [{"R": z["R_start"][c], "t": z["t_start"][c]} for c in range(C)]
    else:
        obs, mask, _, start, K, _ = _tracks_case(C, F, seed=100 + C)
    ctx = _ctx(C)
    ctx.set_cameras([K] * C, start)
    out0, rep0 = ctx.bundle_adjust(obs, mask, start, engine=0, prefit=prefit)
    out1, rep1 = ctx.bundle_adjust(obs, mask, start, engine=1, prefit=prefit)
    assert rep0["n_launches"] == 1 and rep1["n_launches"] > 5
    assert rep0["n_residuals"] == rep1["n_residuals"]
    assert abs(rep0["cost_initial"] - rep1["cost_initial"]) <= 1e-9 * rep1["cost_initial"]
    assert rep0["prefit_iterations"] == rep1["prefit_iterations"]
    assert abs(rep0["prefit_cost_final"] - rep1["prefit_cost_final"]) <= 1e-6 * max(1.0, rep1["prefit_cost_final"])
    assert (rep0["n_iterations"], rep0["n_fev"], rep0["status"]) == (rep1["n_iterations"], rep1["n_fev"], rep1["status"])
    assert abs(rep0["cost_final"] - rep1["cost_final"]) <= 1e-6 * max(1.0, rep1["cost_final"])
    for a, b in zip(out0, out1):
        assert np.abs(a["R"] - b["R"]).max() < 1e-7 and np.abs(a["t"] - b["t"]).max() < 1e-7
    assert np.allclose(out0[0]["R"], np.eye(3)) and np.allclose(out0[0]["t"], 0)


def test_ba_device_engine_is_reproducible(torch):
    """No atomics in the solve: two runs give the same bits."""
    obs, mask, _, start, K, _ = _tracks_case(8, 3000, seed=5)
    ctx = _ctx(8)
    ctx.set_cameras([K] * 8, start)
    a, ra = ctx.bundle_adjust(obs, mask, start)
    b, rb = ctx.bundle_adjust(obs, mask, start)
    ra.pop("phase_ms"); rb.pop("phase_ms")
    assert ra == rb
    for p, q in zip(a, b):
        assert np.array_equal(p["R"], q["R"]) and np.array_equal(p["t"], q["t"])


def test_ba_grid_setter_and_solves_side_by_side(torch):
    """mocap_set_ba_grid: the result of a solve does not depend on the number of CTAs, two contexts with half of the SMs
    each run their solves on two streams side by side with the same result, and values outside 0 .. SMs are refused."""
    obs, mask, _, start, K, _ = _tracks_case(8, 3000, seed=5)
    ctx = _ctx(8)
    ctx.set_cameras([K] * 8, start)
    ref, rep = ctx.bundle_adjust(obs, mask, start)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for n in (1, 37, sms // 2, 0):
        ctx.set_ba_grid(n)
        out, r = ctx.bundle_adjust(obs, mask, start)
        assert r["status"] == rep["status"] and r["n_fev"] == rep["n_fev"] and abs(r["cost_final"] - rep["cost_final"]) <= 1e-9 * rep["cost_final"]
        for a, b in zip(out, ref):
            assert np.abs(a["R"] - b["R"]).max() < 1e-10 and np.abs(a["t"] - b["t"]).max() < 1e-10
    for bad in (-1, sms + 1):
        with pytest.raises(pkg.MocapError):
            ctx.set_ba_grid(bad)
    d_obs, d_mask = torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda()
    R0 = torch.from_numpy(np.stack([np.asarray(p["R"]) for p in start])).cuda().contiguous()
    t0 = torch.from_numpy(np.stack([np.asarray(p["t"]).reshape(3) for p in start])).cuda().contiguous()
    pair = [_ctx(8), _ctx(8)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    Rs, ts = [R0.clone() for _ in range(4)], [t0.clone() for _ in range(4)]
    for c in pair:
        c.set_cameras([K] * 8, start)
        c.set_ba_grid(sms // 2)
    torch.cuda.synchronize()
    for i in range(4):
        with torch.cuda.stream(streams[i % 2]):
            pair[i % 2].bundle_adjust_dev(d_obs, d_mask, Rs[i], ts[i])
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.equal(Rs[i], Rs[0]) and torch.equal(ts[i], ts[0])
        assert np.abs(Rs[i].cpu().numpy() - np.stack([p["R"] for p in ref])).max() < 1e-10


def test_pipeline_tracks_equal_chosen_correspondences(torch):
    """mocap_pipeline_tracks_dev leaves the pixel of the winning correspondence per camera; it must be the blob the
    `chosen` indices of the separate matcher name, and the device compaction must equal the torch one."""
    z = load_golden("pipe_c8_m16")
    C = 8
    ctx = _ctx(C, max_roots=64)
    ctx.set_cameras([z["K"]] * C, poses_from(z))
    frames = torch.from_numpy(z["frames"]).cuda()
    B = frames.shape[0]
    for mode in ("fused", "split"):
        os.environ["MOCAP_PIPELINE"] = mode
        try:
            c2 = _ctx(C, max_roots=64)
        finally:
            os.environ.pop("MOCAP_PIPELINE", None)
        c2.set_cameras([z["K"]] * C, poses_from(z))
        tr = c2.pipeline(frames, want_tracks=True)
        d = c2.detect(frames.view(-1, 480, 640))
        m = c2.match_triangulate(d["xy"], d["n"], want_chosen=True)
        assert torch.equal(tr["n"], m["n"])
        obs_ref, mask_ref = c2.tracks_to_observations(d["xy"], m["n"], m["chosen"])
        o = c2.tracks_to_observations_dev(tr)
        torch.cuda.synchronize()
        n = int(o["n"].item())
        assert n == obs_ref.shape[0] == int(m["n"].sum().item())
        assert np.array_equal(o["mask"][:n].cpu().numpy(), mask_ref)
        assert np.array_equal(o["obs"][:n].cpu().numpy(), obs_ref)
        # error filter: keeps exactly the tracks at or below the bound, in order
        bound = float(np.median(m["err"][0, :int(m["n"][0])].cpu().numpy()))
        of = c2.tracks_to_observations_dev(tr, max_err=bound)
        keep = np.concatenate([(m["err"][b, :int(m["n"][b])] <= bound).cpu().numpy() for b in range(B)])
        nf = int(of["n"].item())
        assert nf == int(keep.sum()) and np.array_equal(of["obs"][:nf].cpu().numpy(), obs_ref[keep])


def test_config3_chain_on_the_device(torch):
    """BASELINE config 3's step without the host: frames -> S1-S3 (+ winners' pixels) -> observations -> S4 from
    perturbed poses, all enqueued on one stream with no synchronisation in between; the refined poses reproduce the
    true rig up to the free global scale."""
    C, M, B = 8, 16, 120
    frames, truth, poses, K = synth.make_frame_pool(C, M, B, seed=21)
    ctx = _ctx(C, max_roots=64)
    ctx.set_cameras([K] * C, poses)
    tr = ctx.pipeline(torch.from_numpy(frames).cuda(), want_tracks=True)
    o = ctx.tracks_to_observations_dev(tr, max_err=2.0)
    start = synth.perturb_poses(poses, seed=22)
    R = torch.from_numpy(np.stack([p["R"] for p in start])).cuda().contiguous()
    t = torch.from_numpy(np.stack([np.asarray(p["t"]).reshape(3) for p in start])).cuda().contiguous()
    rep = ctx.bundle_adjust_dev(o["obs"], o["mask"], R, t, n_points=o["n"])
    torch.cuda.synchronize()
    rep = ctx.decode_ba_report(rep)
    assert int((tr["flags"] != 0).sum().item()) == 0
    assert rep["n_residuals"] == int(o["n"].item()) and rep["n_residuals"] >= B * M * 0.9
    assert rep["status"] in (1, 2, 3, 4) and rep["cost_final"] < 1e-3 * rep["cost_initial"]
    Rn, tn = R.cpu().numpy(), t.cpu().numpy()
    s = np.linalg.norm(np.stack([p["t"] for p in poses])) / np.linalg.norm(tn)       # camera 0 pinned: only the scale is free
    for c in range(C):
        assert np.abs(Rn[c] - np.asarray(poses[c]["R"])).max() < 5e-3
        assert np.abs(tn[c] * s - np.asarray(poses[c]["t"]).reshape(3)).max() < 2e-2


def test_detect_reproduces_retr_tree_on_blobs_with_holes(torch):
    """Blobs with holes (golden blobs_rings: rings, frames, porous patches, nested blobs through the REAL _find_dot):
    cv.findContours(RETR_TREE) emits an extra contour per hole, fills the outer one and orders along its hierarchy.
    Through mocap_detect_dev and through both pipelines the points -- count, values, order -- equal the real
    reference's on every frame, with and without holes, and no flag is left; the mirror returns the reference's list.
    A holed blob too large for the slow path's window is flagged (and the mirror raises)."""
    z = load_golden("blobs_rings")
    frames = z["frames"]                                   # [F, 1, H, W]
    F = frames.shape[0]
    assert int(z["has_hole"].sum()) >= 5 and int((1 - z["has_hole"]).sum()) >= 5
    ctx = _ctx(1, max_blobs=64)
    d = ctx.detect(torch.from_numpy(frames).cuda(), want_moments=True)
    flags = d["flags"].cpu().numpy(); n = d["n"].cpu().numpy(); xy = d["xy"].cpu().numpy()
    fits = z["blob_n"][:, 0] <= 64                         # the library keeps at most 64 points per image (MOCAP_F_BLOBS beyond)
    assert fits.sum() >= F - 4 and (z["has_hole"].astype(bool) & fits).sum() >= 5
    for f in range(F):
        k = min(int(z["blob_n"][f, 0]), 64)
        if not fits[f] and flags[f] == 32:
            continue                                       # more than 64 holes in one image: left flagged (frame 14 of the golden: 68 holes)
        assert flags[f] == (0 if fits[f] else 2) and n[f] == k and np.array_equal(xy[f, :k], z["blob_xy"][f, 0, :k]), f
    assert int((flags == 32).sum()) <= 1
    K1 = np.array([[600.0, 0, 320], [0, 600, 240], [0, 0, 1]])
    for mode in ("fused", "split"):
        os.environ["MOCAP_PIPELINE"] = mode
        try:
            c2 = _ctx(1, max_blobs=64)
        finally:
            os.environ.pop("MOCAP_PIPELINE", None)
        c2.set_cameras([K1], [{"R": np.eye(3), "t": np.zeros(3)}])
        for rep in range(2):                               # twice: the deferral path re-arms its worklists
            out = c2.pipeline(torch.from_numpy(frames).cuda())
            assert np.array_equal(out["flags"].cpu().numpy(), flags), mode
        d2 = c2.detect(torch.from_numpy(frames).cuda())
        live = torch.arange(d["xy"].shape[1], device="cuda")[None, :] < d["n"][:, None]      # rows past the count are unspecified
        assert torch.equal(d2["n"], d["n"]) and torch.equal(d2["xy"][live], d["xy"][live])
    s = pkg.MocapSession([np.eye(3)])
    for f in (int(np.argmax(z["has_hole"].astype(bool) & fits)), int(np.argmax(~z["has_hole"].astype(bool) & fits))):
        _, pts = pkg.find_dot(as3(frames[f, 0]), session=s)
        assert pts == z["blob_xy"][f, 0, :int(z["blob_n"][f, 0])].tolist()
    import cv2
    big = np.zeros((480, 640), np.uint8)
    cv2.circle(big, (300, 200), 60, 255, 3)                # a 120-px ring: does not fit the 62-px window
    db = ctx.detect(torch.from_numpy(big[None]).cuda())
    assert int(db["flags"][0].item()) == 32 and int(db["n"][0].item()) == 1
    with pytest.raises(pkg.MocapError):
        pkg.find_dot(as3(big), session=s)

"""GPU tests of the batch paths the parity tests do not reach: the 3-channel single-pass kernel, batches that span
several launch groups, the host entry point's staging over several chunks, capacity flags raised on the device, the
chunked matcher at several chunk sizes, and the DLT null vector at near-degenerate geometry.  Run with ``-m gpu`` on
an H100."""
import importlib

import numpy as np
import pytest

from tests.util import load_golden, poses_from, as3

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
api = importlib.import_module("low-cost-mocap_b200.api")
synth = pkg.synth

X_TOL = 1e-7          # pose units; BASELINE north_star: 1e-4 mm with poses in metres
ERR_RTOL = 1e-9       # reprojection errors are float32-quantised upstream; expected bit-equal
ROOMY = dict(max_blobs=64, max_roots=128, max_cands=16, max_groups=1 << 16)      # nothing the tests feed overflows


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _ctx(C, W=640, H=480, **kw):
    return pkg.MocapContext(C, W, H, **kw)


def _pinned_ctx(monkeypatch, C, pipeline=None, chunk=None, W=640, H=480, **kw):
    """A context with the pipeline / matcher chunk pinned (both are read when the context is created)."""
    if pipeline is None:
        monkeypatch.delenv("MOCAP_PIPELINE", raising=False)
    else:
        monkeypatch.setenv("MOCAP_PIPELINE", pipeline)
    if chunk is None:
        monkeypatch.delenv("MOCAP_MATCH_CHUNK", raising=False)
    else:
        monkeypatch.setenv("MOCAP_MATCH_CHUNK", str(chunk))
    return _ctx(C, W, H, **kw)


def _host(out):
    return {k: v.cpu().numpy().copy() for k, v in out.items()}


def _assert_same_tracks(a, b, sets=None, what=""):
    """n and flags equal; obj / err (and track_xy / chosen where both have them) equal bit for bit in the live rows."""
    sets = range(len(a["n"])) if sets is None else sets
    for s in sets:
        k = int(a["n"][s])
        assert int(b["n"][s]) == k and int(a["flags"][s]) == int(b["flags"][s]), (what, s)
        assert np.array_equal(a["obj"][s, :k], b["obj"][s, :k]) and np.array_equal(a["err"][s, :k], b["err"][s, :k]), (what, s)
        for key in ("track_xy", "chosen"):
            if key in a and key in b:
                assert np.array_equal(a[key][s, :k], b[key][s, :k]), (what, key, s)


def _find_dot_at(port, img3, threshold):
    """The reference's _find_dot (helpers.py:143-163) on an HxWx3 image, at another threshold than 255 * 0.2."""
    import cv2
    if threshold == 51:
        return port.find_dot(img3.copy())
    grey = cv2.cvtColor(img3, cv2.COLOR_RGB2GRAY)
    binary = cv2.threshold(grey, threshold, 255, cv2.THRESH_BINARY)[1]
    contours, _ = cv2.findContours(binary, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
    out = []
    for cnt in contours:
        mo = cv2.moments(cnt)
        if mo["m00"] != 0:
            out.append([int(mo["m10"] / mo["m00"]), int(mo["m01"] / mo["m00"])])
    return out if out else [[None, None]]


def _render_spots(rng, H, W, uv, bg=0):
    yy, xx = np.mgrid[:H, :W]
    img = rng.integers(0, bg + 1, size=(H, W), dtype=np.uint8) if bg else np.zeros((H, W), np.uint8)
    for u, v in uv:
        s = rng.uniform(1.0, 1.8)
        img = np.maximum(img, np.floor(255.0 * np.exp(-((xx - u) ** 2 + (yy - v) ** 2) / (2 * s * s))).astype(np.uint8))
    return img


# ------------------------------------------------------------------------------------------------------------- T1
@pytest.mark.parametrize("name", ["pipe_c4_m4", "pipe_c8_m16"])
def test_three_channel_golden_frames_through_both_pipelines(torch, monkeypatch, name):
    """H x W x 3 frame-sets with equal channels (the layout _find_dot receives) through the single-pass kernel and the
    three-kernel pipeline, device and host entry points: the real reference's kept roots, points and errors."""
    z = load_golden(name, n=40 if name == "pipe_c4_m4" else 16)
    C = int(z["C"]); B = z["frames"].shape[0]
    frames = np.ascontiguousarray(np.repeat(z["frames"][..., None], 3, axis=-1))
    for mode in ("fused", "split"):
        ctx = _pinned_ctx(monkeypatch, C, mode, max_blobs=64, max_roots=128)
        ctx.set_cameras([z["K"]] * C, poses_from(z))
        dev = _host(ctx.pipeline(torch.from_numpy(frames).cuda()))
        host = _host(ctx.pipeline_host(torch.from_numpy(frames).pin_memory()))
        for out in (dev, host):
            assert np.array_equal(out["n"], z["nroot"]) and (out["flags"] == 0).all(), mode
            for b in range(B):
                k = int(z["nroot"][b])
                assert np.abs(out["obj"][b, :k] - z["obj"][b, :k]).max() <= X_TOL, (mode, b)
                assert np.allclose(out["err"][b, :k], z["err"][b, :k], rtol=ERR_RTOL, atol=1e-12), (mode, b)
        _assert_same_tracks(dev, host, what=mode)


def _patch_colours(t):
    """Colours whose cv2 grey (fixed point, rounded) sits at, just above and just below the threshold."""
    lo, c = max(t - 1, 0), lambda *v: [min(x, 255) for x in v]
    return [c(t + 1, t, t), c(t, t + 1, t), c(t, t, t + 1), c(t, t, t), c(t + 1, t + 1, t + 1), c(lo, lo, lo),
            c(t + 2, t, t), c(t, t + 1, t + 1), c(t + 1, t + 1, t), c(t, t + 2, t)]


def _plant_threshold_patches(img, t, free_rows):
    """2x2 patches in the top `free_rows` rows (no markers there), 3 x 16 bytes per 16-pixel segment: pixels 2-3 have
    every byte in word 0, 6-7 in word 1, 12-13 in word 2, 4-5 straddle words 0 and 1.  Plus segments where word 0 (a
    lone [t+1, t, t] pixel, grey t) and word 2 (or word 1) pass the byte test but only the later word's pixels pass
    the grey threshold."""
    W = img.shape[1]
    spr = W // 16
    slots = []
    for col in _patch_colours(t):
        for p in (2, 6, 12, 4):
            slots.append([(p, col), (p + 1, col)])
    t1, t2 = [min(t + 1, 255), t, t], [t, min(t + 1, 255), t]
    slots.append([(1, t1), (12, t2), (13, t2)])
    slots.append([(1, t1), (7, t2), (8, t2)])
    slots.append([(0, t1), (14, t2), (15, t2)])
    for k, pixels in enumerate(slots):
        seg, band = k % spr, k // spr
        y = 1 + 3 * band
        assert y + 2 <= free_rows, "patch bands must stay above the markers"
        for p, col in pixels:
            img[y:y + 2, 16 * seg + p] = col


def _threshold_case(geometry):
    """(frames uint8 [B, C, H, W, 3] with unequal channels, K, poses)"""
    rng = np.random.default_rng(17)
    if geometry == "c4_640x480":
        z = load_golden("pipe_c4_m4", n=6)
        grey = z["frames_clean"]                       # zero background: low thresholds must not flood the image
        K, poses = z["K"], poses_from(z)
    else:                                              # 336 x 200: the stream's slices end ragged (not whole warp iterations)
        W, H, C = 336, 200, 2
        K = np.array([[300.0, 0, 168], [0, 300.0, 100], [0, 0, 1]])
        poses = [{"R": np.eye(3), "t": np.zeros(3)}, {"R": np.eye(3), "t": np.array([-0.3, 0.0, 0.0])}]
        grey = np.zeros((6, C, H, W), np.uint8)
        for b in range(6):
            X = rng.uniform([-0.4, -0.15, 2.0], [0.4, 0.2, 3.0], size=(4, 3))
            for c in range(C):
                uv = np.stack([synth.project(X[i:i + 1], poses[c], K)[0] for i in range(4)])
                grey[b, c] = _render_spots(rng, H, W, uv)
    frames = np.repeat(grey[..., None], 3, axis=-1).astype(np.int32)
    lit = grey > 0
    for ch in (0, 2):                                  # unequal channels where there is light
        frames[..., ch] = np.where(lit, np.clip(frames[..., ch] + rng.integers(-30, 31, size=grey.shape), 0, 255), 0)
    return frames.astype(np.uint8), K, poses


@pytest.mark.parametrize("geometry", ["c4_640x480", "c2_336x200"])
@pytest.mark.parametrize("threshold", [0, 51, 127, 128, 200, 254])
def test_three_channel_frames_at_threshold_edges(torch, monkeypatch, geometry, threshold):
    """Unequal channels and colour patches whose grey sits at the threshold, placed so that the only byte above the
    threshold lies in word 0, 1 or 2 of its segment (and segments where an earlier word passes the byte test but only a
    later word's pixels pass the grey test), in both compare regimes of the single-pass kernel (thresholds below and
    from 128 on).  Oracle: _find_dot + the matcher of the reference on every H x W x 3 image; second oracle: the
    1-channel pipeline on cv2's grey frames, bit for bit (points, errors, counts, flags, winners' pixels)."""
    import cv2
    from oracle.ref_port import RefPort
    frames, K, poses = _threshold_case(geometry)
    B, C, H, W = frames.shape[:4]
    for b in range(B):                                 # golden markers keep 7 rows clear of the top; the 336 x 200 ones 70
        _plant_threshold_patches(frames[b, b % C], threshold, 6 if W == 640 else 60)
    grey = np.stack([[cv2.cvtColor(frames[b, c], cv2.COLOR_RGB2GRAY) for c in range(C)] for b in range(B)])
    port = RefPort([K] * C)
    ref, n_blobs = [], 0
    for b in range(B):
        pts = [_find_dot_at(port, frames[b, c], threshold) for c in range(C)]
        n_blobs += sum(p[0] is not None for cam in pts for p in cam)
        ref.append(port.match_and_triangulate(pts, poses))
    assert n_blobs >= B * 10 and (threshold == 254 or sum(len(r[0]) for r in ref) > 0)    # at 254 only the patches pass
    for mode in ("fused", "split"):
        ctx = _pinned_ctx(monkeypatch, C, mode, W=W, H=H, **ROOMY)
        ctx.set_cameras([K] * C, poses)
        d3 = _host(ctx.pipeline(torch.from_numpy(frames).cuda(), threshold=threshold, want_tracks=True))
        d1 = _host(ctx.pipeline(torch.from_numpy(grey).cuda(), threshold=threshold, want_tracks=True))
        h3 = _host(ctx.pipeline_host(torch.from_numpy(frames).pin_memory(), threshold=threshold))
        assert (d3["flags"] == 0).all(), (mode, d3["flags"])
        for b, (e, o, _) in enumerate(ref):
            k = int(d3["n"][b])
            assert k == len(e), (mode, b, k, len(e))
            if k:
                assert np.abs(d3["obj"][b, :k] - np.asarray(o, dtype=np.float64)).max() <= X_TOL, (mode, b)
                assert np.allclose(d3["err"][b, :k], e, rtol=ERR_RTOL, atol=1e-12), (mode, b)
        _assert_same_tracks(d3, d1, what=mode + " 3-channel vs grey")
        _assert_same_tracks(d3, h3, what=mode + " device vs host")


# ------------------------------------------------------------------------------------------------------------- T2
def _small_pool(rng, P, C, H, W, K, poses):
    """P frame-sets of Gaussian spots over clutter; set 0 has an image of 70 blobs (more than a warp accumulates),
    set 1 an image with one blob of more segments than a warp's slab: both take the deferral paths."""
    pool = np.zeros((P, C, H, W), np.uint8)
    for b in range(P):
        X = rng.uniform([-0.5, -0.3, 2.0], [0.5, 0.3, 3.0], size=(int(rng.integers(1, 5)), 3))
        for c in range(C):
            uv = np.stack([synth.project(X[i:i + 1], poses[c], K)[0] for i in range(len(X))])
            pool[b, c] = _render_spots(rng, H, W, uv, bg=40)
    for k in range(70):
        y, x = 2 + 4 * (k // (W // 4)), 2 + 4 * (k % (W // 4))
        pool[0, 1, y:y + 2, x:x + 2] = 255
    pool[1, 0, 4:44, :] = 200                         # 40 rows x 7 segments = 280 segments > 256 of a warp's slab
    return pool


def test_batches_across_launch_groups(torch, monkeypatch):
    """A batch of 2 * 65536 / C + 5 frame-sets (three launch groups of the single-pass kernel, seventeen of the
    three-kernel pipeline) tiled from a pool of distinct frame-sets, the deferred ones placed on both sides of every
    group boundary and last: every frame-set equals the pool's own one-group result -- points, errors, counts, flags,
    winners' pixels -- in both pipelines, the two pipelines agree, and the device compaction of the whole batch's tracks
    equals the concatenation of the per-set tracks.  The host entry point on a host copy of the batch (three staging
    chunks of 24 966 frame-sets, each cut into seven launch groups by the three-kernel pipeline) equals it too."""
    C, H, W, P = 2, 48, 112, 40
    K = np.array([[100.0, 0, 56], [0, 100.0, 24], [0, 0, 1]])
    poses = [{"R": np.eye(3), "t": np.zeros(3)}, {"R": np.eye(3), "t": np.array([-0.2, 0.0, 0.0])}]
    rng = np.random.default_rng(5)
    pool = _small_pool(rng, P, C, H, W, K, poses)
    B = 2 * (65536 // C) + 5
    idx = rng.integers(2, P, size=B)
    for i, d in zip((4095, 4096, 32767, 32768, 65535, 65536, B - 1), (0, 1, 1, 0, 0, 1, 0)):
        idx[i] = d
    idx_d = torch.from_numpy(idx).cuda()
    pool_d = torch.from_numpy(pool).cuda()
    per_mode = {}
    for mode in ("fused", "split"):
        ctx = _pinned_ctx(monkeypatch, C, mode, W=W, H=H, max_blobs=64, max_roots=16, max_segments=512)
        ctx.set_cameras([K] * C, poses)
        ref = ctx.pipeline(pool_d, want_tracks=True)
        assert int(ref["flags"][0]) != 0 and int((ref["n"] > 0).sum()) > P // 2      # the 70-blob set overflows max_blobs
        big_in = pool_d[idx_d].contiguous()                                           # ~700 MB
        big = ctx.pipeline(big_in, want_tracks=True)
        host = ctx.pipeline_host(big_in.cpu())
        del big_in
        torch.cuda.synchronize()
        R = ctx.cfg.max_roots
        live = torch.arange(R, device="cuda")[None, :] < big["n"][:, None]
        assert torch.equal(big["n"], ref["n"][idx_d]) and torch.equal(big["flags"], ref["flags"][idx_d]), mode
        for key in ("obj", "err", "track_xy"):
            assert torch.equal(big[key][live], ref[key][idx_d][live]), (mode, key)
        assert torch.equal(host["n"], ref["n"][idx_d].cpu()) and torch.equal(host["flags"], ref["flags"][idx_d].cpu()), mode
        for key in ("obj", "err"):
            assert torch.equal(host[key][live.cpu()], ref[key][idx_d][live].cpu()), (mode, "host", key)
        obs = ctx.tracks_to_observations_dev(big)
        rows = ref["track_xy"][idx_d][live]                                           # [points, C, 2] in frame order
        mask = rows[..., 0] >= 0
        n_pts = int(obs["n"].item())
        assert n_pts == rows.shape[0] > B // 2
        assert torch.equal(obs["mask"][:n_pts], mask.to(torch.uint8))
        assert torch.equal(obs["obs"][:n_pts], torch.where(mask[..., None], rows.double(), torch.zeros((), dtype=torch.float64, device="cuda")))
        per_mode[mode] = _host({k: ref[k] for k in ("obj", "err", "n", "flags", "track_xy")})
        del big, obs, ref, ctx
        torch.cuda.empty_cache()
    _assert_same_tracks(per_mode["fused"], per_mode["split"], what="fused vs split")


# ------------------------------------------------------------------------------------------------------------- T3
def test_host_entry_point_over_several_staging_chunks(torch, monkeypatch):
    """mocap_pipeline_host stages ~256 MB per chunk on two copy streams and, from the third chunk on, waits for the
    buffer's previous kernel: a batch of 890 frame-sets of 640 x 480 x 4 cameras (five chunks of 218), light and heavy
    frame-sets mixed at random, from a pinned tensor and from a plain numpy array, equals the device entry point on the
    same batch bit for bit in both pipelines; so do a batch of exactly two chunks and a batch of one frame-set."""
    z = load_golden("pipe_c4_m4")
    C = 4
    heavy, _, _, _ = synth.make_frame_pool(C, 16, 12, seed=41)                       # 16 markers: hundreds of groups
    pool = np.concatenate([z["frames"], heavy])
    for k in range(70):                                                              # and one set past max_blobs
        y, x = 10 + 6 * (k // 35), 20 + 16 * (k % 35)
        pool[-1, 2, y:y + 3, x:x + 3] = 255
    rng = np.random.default_rng(11)
    B = 890
    batch = pool[rng.integers(0, len(pool), size=B)]                                 # 1.09 GB, plain pageable memory
    assert batch.nbytes // (C * 640 * 480) == B and B > 4 * ((256 << 20) // (C * 640 * 480))
    pinned = torch.from_numpy(batch).pin_memory()
    res = {}
    for mode in ("fused", "split"):
        ctx = _pinned_ctx(monkeypatch, C, mode, max_blobs=64, max_roots=64)
        ctx.set_cameras([z["K"]] * C, poses_from(z))
        dev_in = pinned.cuda()
        dev = _host(ctx.pipeline(dev_in))
        del dev_in
        torch.cuda.empty_cache()
        assert (dev["flags"] != 0).any() and (dev["n"] > 8).any() and (dev["n"] <= 8).any()
        _assert_same_tracks(dev, _host(ctx.pipeline_host(pinned)), what=mode + " pinned")
        _assert_same_tracks(dev, _host(ctx.pipeline_host(batch)), what=mode + " numpy")
        two = 2 * ((256 << 20) // (C * 640 * 480))
        _assert_same_tracks(dev, _host(ctx.pipeline_host(pinned[:two])), sets=range(two), what=mode + " two chunks")
        _assert_same_tracks(dev, _host(ctx.pipeline_host(batch[:1])), sets=range(1), what=mode + " one set")
        res[mode] = dev
        ctx.close()
        torch.cuda.empty_cache()
    _assert_same_tracks(res["fused"], res["split"], what="fused vs split")


# ------------------------------------------------------------------------------------------------------------- T4
F_SEGMENTS, F_BLOBS, F_ROOTS, F_CANDS, F_GROUPS = api.F_SEGMENTS, api.F_BLOBS, api.F_ROOTS, api.F_CANDS, api.F_GROUPS
TIGHT = dict(max_blobs=64, max_segments=1024, max_roots=24, max_cands=4, max_groups=32)
# 64 kept blobs of the BLOBS offender all become roots: its batch needs room in the matcher
ROOMY_MATCH = dict(max_blobs=64, max_segments=1024, max_roots=128, max_cands=16, max_groups=1 << 16)


def _epipolar_points(K, poses, xy0, cam, avoid, n, step=11.0):
    """n integer pixels of camera `cam` on the epipolar line of camera 0's pixel xy0 (the projections of two points of
    its ray), inside the image and at least 10 px from every pixel of `avoid` and from each other."""
    ray = np.linalg.solve(K, np.array([xy0[0], xy0[1], 1.0]))
    p1, p2 = (synth.project((d * ray)[None], poses[cam], K)[0] for d in (2.0, 4.0))
    u = (p2 - p1) / np.linalg.norm(p2 - p1)
    out, taken = [], [np.asarray(a, float) for a in avoid]
    for s in sorted(np.arange(-60, 61) * step, key=abs):
        q = np.round(p1 + s * u)
        if not (8 <= q[0] < 632 and 8 <= q[1] < 472) or any(np.abs(q - a).max() < 10 for a in taken):
            continue
        out.append([int(q[0]), int(q[1])]); taken.append(q)
        if len(out) == n:
            return out
    raise AssertionError("no room on the epipolar line")


def _free_grid(avoid, n, x0=20, y0=20, dx=24, dy=24):
    out = []
    for y in range(y0, 470, dy):
        for x in range(x0, 630, dx):
            if all(abs(x - a[0]) >= 12 or abs(y - a[1]) >= 12 for a in avoid):
                out.append([x, y])
                if len(out) == n:
                    return out
    raise AssertionError("no room")


def _offender_lists(z, b, kind):
    """The golden blob lists of frame-set b plus the blobs that make it overflow exactly one matcher capacity of TIGHT."""
    C = int(z["C"])
    K, poses = z["K"], poses_from(z)
    lists = [z["blob_xy"][b, c, :int(z["blob_n"][b, c])].tolist() for c in range(C)]
    root = lists[0][0]
    if kind == F_ROOTS:                                 # 28 camera-0 blobs > max_roots = 24
        lists[0] += _free_grid(lists[0], 28 - len(lists[0]))
    elif kind == F_CANDS:                               # max_cands + 1 blobs near the root's line in camera 1
        lists[1] += _epipolar_points(K, poses, root, 1, lists[1], TIGHT["max_cands"] + 1)
    elif kind == F_GROUPS:                              # 3 x 3 x 4 = 36 candidate groups > max_groups = 32, 4 per line at most
        for c, extra in ((1, 2), (2, 2), (3, 3)):
            lists[c] += _epipolar_points(K, poses, root, c, lists[c], extra)
    return lists


def _frames_from_lists(z, b, lists):
    """The golden frames of set b with a 3x3 square (centre = the listed pixel) for every blob beyond the golden list."""
    f = z["frames"][b].copy()
    for c, lst in enumerate(lists):
        for x, y in lst[int(z["blob_n"][b, c]):]:
            f[c, y - 1:y + 2, x - 1:x + 2] = 255
    return f


def _pack(lists_per_set, C, MB=64):
    B = len(lists_per_set)
    xy = np.zeros((B, C, MB, 2), np.int32); n = np.zeros((B, C), np.int32)
    for s, lists in enumerate(lists_per_set):
        for c, lst in enumerate(lists):
            n[s, c] = len(lst)
            if lst:
                xy[s, c, :len(lst)] = lst
    return xy.reshape(B * C, MB, 2), n.reshape(B * C)


def test_capacity_flags_on_the_device(torch, monkeypatch):
    """One offender per capacity among clean frame-sets: SEGMENTS (a large bright rectangle), BLOBS (70 blobs), ROOTS
    (more camera-0 blobs than max_roots), CANDS (max_cands + 1 blobs near one root's epipolar line), GROUPS (candidate
    products above max_groups).  Each offender carries exactly its bit, every other frame-set none; clean frame-sets are
    bit-identical to a batch without the offenders; flags and outputs (truncated ones included) agree between the
    single-pass kernel and the three-kernel pipeline and between matcher chunks of 0 and 32 groups, from blob lists and
    from frames.  The drop-in mirrors raise instead of returning truncated results."""
    z = load_golden("pipe_c4_m4", n=12)
    C = 4
    K, poses = z["K"], poses_from(z)
    clean = [0, 1, 3, 5, 7, 9, 11]
    offenders = {2: F_ROOTS, 4: F_CANDS, 6: F_GROUPS}
    golden = [z["blob_xy"][b, c, :int(z["blob_n"][b, c])].tolist() for b in range(12) for c in range(C)]
    sets = [_offender_lists(z, b, offenders[b]) if b in offenders else golden[b * C:(b + 1) * C] for b in range(12)]
    frames = np.stack([_frames_from_lists(z, b, sets[b]) for b in range(12)])
    frames[8, 2, 100:300, 100:500] = 255                # 200 rows x 25 segments > max_segments = 1024
    for k in range(70):                                 # 70 blobs > max_blobs = 64, a column down the left edge of the last camera
        frames[10, 3, 10 + 6 * k:13 + 6 * k, 2:5] = 255
    expect = np.zeros(12, np.int32)
    for b, f in offenders.items():
        expect[b] = f
    expect[8] = F_SEGMENTS
    roomy_expect = np.zeros(12, np.int32); roomy_expect[8] = F_SEGMENTS; roomy_expect[10] = F_BLOBS
    xy, n = _pack(sets, C)
    xy_c, n_c = _pack([sets[b] for b in clean], C)
    frames_d = torch.from_numpy(frames).cuda()
    runs = {}
    for pipe in ("fused", "split"):
        for chunk in (0, 32):
            tag = f"{pipe}/chunk {chunk}"
            ctx = _pinned_ctx(monkeypatch, C, pipe, chunk, **TIGHT)
            ctx.set_cameras([K] * C, poses)
            lists = _host(ctx.match_triangulate(torch.from_numpy(xy).cuda(), torch.from_numpy(n).cuda(), want_chosen=True))
            pix = _host(ctx.pipeline(frames_d, want_tracks=True))
            only_clean = _host(ctx.pipeline(frames_d[clean].contiguous(), want_tracks=True))
            lists_clean = _host(ctx.match_triangulate(torch.from_numpy(xy_c).cuda(), torch.from_numpy(n_c).cuda(), want_chosen=True))
            lexp = expect.copy(); lexp[8] = 0; lexp[10] = 0      # the blob lists carry no S1 overflow
            assert lists["flags"].tolist() == lexp.tolist(), (tag, lists["flags"])
            assert pix["flags"][[b for b in range(12) if b != 10]].tolist() == [int(expect[b]) for b in range(12) if b != 10], (tag, pix["flags"])
            assert pix["flags"][10] & F_BLOBS, tag       # at TIGHT its 64 kept blobs also overflow the matcher
            for i, b in enumerate(clean):
                _assert_same_tracks({k: v[[b]] for k, v in pix.items()}, {k: v[[i]] for k, v in only_clean.items()}, what=tag)
                _assert_same_tracks({k: v[[b]] for k, v in lists.items()}, {k: v[[i]] for k, v in lists_clean.items()}, what=tag)
                assert int(lists["n"][b]) == int(z["nroot"][b]), (tag, b)
            ctx2 = _pinned_ctx(monkeypatch, C, pipe, chunk, **ROOMY_MATCH)
            ctx2.set_cameras([K] * C, poses)
            roomy = _host(ctx2.pipeline(frames_d, want_tracks=True))
            assert roomy["flags"].tolist() == roomy_expect.tolist(), (tag, roomy["flags"])
            runs[tag] = (lists, pix, roomy)
    first = runs["fused/chunk 0"]
    for tag, r in runs.items():
        if "fused" not in tag:
            _assert_same_tracks(first[0], r[0], what="lists " + tag)
        _assert_same_tracks(first[1], r[1], what="frames " + tag)
        _assert_same_tracks(first[2], r[2], what="frames, roomy matcher " + tag)
    # the drop-in mirrors raise
    s = pkg.MocapSession([K] * C)
    with pytest.raises(pkg.MocapError):
        pkg.find_dot(as3(frames[10, 3]), session=s)
    cand = [list(p) for p in golden[4 * C:5 * C]]
    cand[1] += _epipolar_points(K, poses, cand[0][0], 1, cand[1], api.MIRROR_LIMITS["max_cands"] + 1, step=6.0)
    with pytest.raises(pkg.MocapError):
        pkg.find_point_correspondance_and_object_points(cand, poses, [None] * C, session=s)


# ------------------------------------------------------------------------------------------------------------- T5
def test_chunked_matcher_on_the_device(torch, monkeypatch):
    """The matcher with frame-sets cut into items of 32 or 96 candidate groups, at the default chunk and with one warp
    per frame-set: 400 heavy frame-sets (8 cameras x 16 markers; ~22 items each at 32 groups, so the item list fills and
    claiming warps finish the rest) plus frame-sets with a blob duplicated in cameras 2 and 5 (equal groups in
    different items: the earliest must win, as np.argmin).  Points, errors, counts, flags, chosen blobs and winners'
    pixels are bit-identical across chunk sizes; untouched frame-sets equal the real reference."""
    z = load_golden("pipe_c8_m16", n=100)
    C, G = 8, 100
    reps = 4
    xy = np.tile(z["blob_xy"], (reps, 1, 1, 1)); nb = np.tile(z["blob_n"], (reps, 1))
    tied = []
    for s in range(0, G, 5):                          # 20 frame-sets of the last tile: camera 2 and 5 see one blob twice
        t = (reps - 1) * G + s
        for c in (2, 5):
            k = int(nb[t, c])
            if k < 64:
                xy[t, c, k] = xy[t, c, s % k]; nb[t, c] = k + 1
        tied.append(t)
    B = len(nb)
    xy_d = torch.from_numpy(np.ascontiguousarray(xy.reshape(B * C, 64, 2))).cuda()
    n_d = torch.from_numpy(np.ascontiguousarray(nb.reshape(B * C))).cuda()
    frames_d = torch.from_numpy(z["frames"]).cuda()
    res, pix = {}, {}
    for chunk in (0, 32, 96, None):
        ctx = _pinned_ctx(monkeypatch, C, "split", chunk, max_blobs=64, max_roots=128)
        ctx.set_cameras([z["K"]] * C, poses_from(z))
        before = ctx.launch_count()
        m = ctx.match_triangulate(xy_d, n_d, want_chosen=True)
        torch.cuda.synchronize()
        assert ctx.launch_count() - before == (1 if chunk == 0 else 2), chunk
        m = _host(m)
        m["track_xy"] = np.full(m["chosen"].shape + (2,), -1, np.int32)                # the chosen blobs' pixels, live rows only
        for b in range(B):
            for r in range(int(m["n"][b])):
                for c in np.flatnonzero(m["chosen"][b, r] >= 0):
                    m["track_xy"][b, r, c] = xy[b, c, m["chosen"][b, r, c]]
        res[chunk] = m
        pix[chunk] = _host(ctx.pipeline(frames_d, want_tracks=True))
    one = res[0]
    assert (one["flags"] == 0).all()
    for chunk in (32, 96, None):
        _assert_same_tracks(one, res[chunk], what=f"blob lists, chunk {chunk}")
        _assert_same_tracks(pix[0], pix[chunk], what=f"frames, chunk {chunk}")
    for b in range(B):
        if b in tied:
            continue
        g = b % G
        k = int(z["nroot"][g])
        assert int(one["n"][b]) == k and np.abs(one["obj"][b, :k] - z["obj"][g, :k]).max() <= X_TOL, b
        assert np.allclose(one["err"][b, :k], z["err"][g, :k], rtol=ERR_RTOL, atol=1e-12), b
    # the winners' pixels of the pipeline are the pixels the chosen indices name
    _assert_same_tracks({k: v[:G] for k, v in one.items()}, pix[0], what="lists vs frames")


# ------------------------------------------------------------------------------------------------------------- T6
def test_dlt_at_near_degenerate_geometry_vs_60_digit_reference(torch):
    """ctx.triangulate (the approximate-reciprocal inverse iteration on the device, Jacobi where it does not settle) on
    near-degenerate geometry: within 1e-11 relative of the exact null vector of A^T A (60-digit arithmetic, A from the
    float64 entries numpy forms).  Reprojection errors equal the reference's wherever the reference's point is within
    1e-9 of the exact one and rounds to the same float32 point."""
    pytest.importorskip("mpmath")
    from oracle.ref_port import RefPort
    from tests.util import dlt_cases, dlt_matrix, exact_dlt_point
    for name, Ks, poses, obs, mask in dlt_cases():
        n, C = mask.shape
        ctx = _ctx(C)
        ctx.set_cameras(Ks, poses)
        X, err, valid = ctx.triangulate(obs, mask)
        assert valid.all(), name
        port = RefPort(Ks)
        same_err = 0
        for f in range(n):
            A = dlt_matrix(Ks, poses, obs[f], mask[f])
            Xe = exact_dlt_point(A)
            if Xe is None:
                continue
            scale = max(1.0, np.abs(Xe).max())
            assert np.abs(X[f] - Xe).max() <= 1e-11 * scale, (name, f, X[f], Xe)
            views = [[obs[f, c, 0], obs[f, c, 1]] if mask[f, c] else [None, None] for c in range(C)]
            Xr = np.asarray(port.triangulate_one(views, poses), dtype=np.float64)
            if np.abs(Xr - Xe).max() <= 1e-9 * scale and np.array_equal(Xr.astype(np.float32), X[f].astype(np.float32)):
                assert err[f] == port.reprojection_error(views, Xr, poses), (name, f)
                same_err += 1
        assert same_err >= n // 2, (name, same_err)
        ctx.close()

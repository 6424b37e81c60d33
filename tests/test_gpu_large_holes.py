"""S1's RETR_TREE slow path with the whole-image window (mocap_set_large_holes) on the device, held to cv2 itself:
holed blobs of 40-400 px at three image sizes and in the H x W x 3 layout, bit-equality with the default wherever the
64 x 64 window suffices, large rings in multi-camera frame-sets through every pipeline, the raw-frame chain with
markers that become rings over 62 px, and the drop-in find_dot.  Run with ``-m gpu``."""
import importlib
import os

import numpy as np
import pytest

from tests.large_holes_util import large_holes_fuzz, nested_frames, spiral, wide_porous
from tests.test_gpu_holes import (DIST, _assert_equals_oracle, _first_diff, _same_bits, device_items, raw_marker_frames)
from tests.util import retr_tree_blobs, set_pixel_blobs

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth
F_BLOBS, F_HOLES = 2, 32


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def expected(binary, max_blobs=64):
    """cv2's list with the window on: only more than 64 holes leaves MOCAP_F_HOLES (and the set-pixel list)"""
    items, _, _, holes = retr_tree_blobs(binary)
    flags = 0
    if holes > 64:
        items, flags = set_pixel_blobs(binary), F_HOLES
    if len(items) > max_blobs:
        flags |= F_BLOBS
    return items[:max_blobs], flags


@pytest.mark.parametrize("W,H,n,channels", [(640, 480, 300, 1), (1024, 768, 50, 1), (336, 200, 100, 1), (640, 480, 100, 3)])
def test_large_holed_blob_fuzz_vs_cv2(torch, W, H, n, channels):
    """Random frames with holed blobs of 40-400 px (rings, frames with blobs inside, ellipse rings, nested rings, porous
    bands, cut by the borders) beside small ones, through mocap_detect_dev with the window on: count, centres, order,
    A2 / SX6 / SY6 and pixel counts equal cv2's for every contour, no flag.  The same frames on a context with the window
    switched on and off again, and on one that never had it, give the default's bits; on frames the 64 x 64 window takes,
    the window changes nothing."""
    rng = np.random.default_rng(7 * W + H + channels)
    frames, refs = large_holes_fuzz(rng, n, H, W, channels)
    batch = torch.from_numpy(frames).cuda()
    ctx = pkg.MocapContext(1, W, H, max_blobs=64, max_segments=4096)
    ctx.set_large_holes(True)
    d = ctx.detect(batch, want_moments=True)
    fl = d["flags"].cpu().numpy()
    large = 0
    for i, (items, kept, side) in enumerate(refs):
        got = device_items(d, i)
        assert fl[i] == 0 and got == items, (i, int(fl[i]), _first_diff(got, items))
        large += side > 62
    print(f"{W}x{H}x{channels}: {n} frames, {large} with a holed blob over 62 px")
    assert large >= n // 3
    never = pkg.MocapContext(1, W, H, max_blobs=64, max_segments=4096)
    d_never = never.detect(batch, want_moments=True)
    ctx.set_large_holes(False)
    d_off = ctx.detect(batch, want_moments=True)
    assert torch.equal(d_off["n"], d_never["n"]) and torch.equal(d_off["flags"], d_never["flags"])
    for i in range(n):
        assert device_items(d_off, i) == device_items(d_never, i), i
    fits = [i for i, r in enumerate(refs) if r[2] <= 62]
    for i in fits:
        assert device_items(d_never, i) == device_items(d, i) and int(d_never["flags"][i]) == 0, i
    for i in range(n):
        if refs[i][2] > 62:
            assert int(d_never["flags"][i]) & F_HOLES, i


def named_images(H=480, W=640):
    import cv2

    def new():
        return np.zeros((H, W), np.uint8)
    out = []
    img = new(); cv2.circle(img, (320, 240), 50, 255, 2); out.append(("ring100", img))
    img = new(); cv2.rectangle(img, (0, 0), (W - 1, H - 1), 255, 1); cv2.circle(img, (320, 240), 7, 255, 2)
    img[100:104, 500:510] = 255; out.append(("around_image", img))
    img = new(); spiral(img, 300, 200, 429, 329); out.append(("spiral", img))          # 130 px, 84 turns, 3024 runs
    img = new(); nested_frames(img, 200, 100, 16, gap=4); out.append(("nested16", img))
    img = new(); nested_frames(img, 200, 100, 28, gap=2); out.append(("nested28", img))
    img = new(); wide_porous(img, 200, 100, 64, w=300); out.append(("porous64", img))
    img = new(); wide_porous(img, 200, 100, 65, w=300); out.append(("porous65", img))
    img = new(); cv2.circle(img, (320, 240), 200, 255, 3); cv2.circle(img, (320, 240), 120, 255, 3)
    cv2.circle(img, (320, 240), 5, 255, -1); cv2.circle(img, (250, 200), 20, 255, 2); out.append(("holed_in_hole", img))
    return out


def test_named_large_images(torch):
    """A 100-px ring, a frame around the image, a 130-px spiral (as many turns as 4096 runs allow), 16 and 28 nested frames (up to 56
    contours 56 deep), 64- and 65-hole bands 300 px wide, large holed blobs in large holes: cv2's list, or MOCAP_F_HOLES
    with the set-pixel list at 65 holes; the same on a second call."""
    cases = named_images()
    imgs = torch.from_numpy(np.stack([c[1] for c in cases])).cuda()
    ctx = pkg.MocapContext(1, 640, 480, max_blobs=64, max_segments=4096)
    ctx.set_large_holes(True)
    d = ctx.detect(imgs, want_moments=True)
    for i, (name, img) in enumerate(cases):
        items, flags = expected(img > 0)
        got = device_items(d, i)
        assert int(d["flags"][i]) == flags and got == items, (name, int(d["flags"][i]), flags, _first_diff(got, items))
    assert int(d["flags"][6]) == F_HOLES and len(retr_tree_blobs(cases[4][1] > 0)[0]) == 56
    d2 = ctx.detect(imgs, want_moments=True)
    assert torch.equal(d2["n"], d["n"]) and torch.equal(d2["flags"], d["flags"])
    assert all(device_items(d2, i) == device_items(d, i) for i in range(len(cases)))


def _large_ring_sets(rng, C, B, poses, K):
    """B frame-sets of C 640 x 480 images: ring markers of radius 3-14 at the projections of random points, and in half
    of the frame-sets a ring of radius 35-120 (70-240 px) somewhere in some cameras."""
    import cv2
    frames = np.zeros((B, C, 480, 640), np.uint8)
    for b in range(B):
        while True:
            pts3 = rng.uniform(-0.5, 0.5, size=(int(rng.integers(1, 5 if C == 8 else 7)), 3)) + np.array([0, 0, 3.0])
            look = [(int(rng.integers(3, 15)), int(rng.integers(1, 4))) for _ in pts3]
            imgs = np.zeros((C, 480, 640), np.uint8)
            for c in range(C):
                for p, (r, th) in zip(pts3, look):
                    u, v = synth.project(p[None], poses[c], K)[0]
                    cv2.circle(imgs[c], (int(round(u)), int(round(v))), r, 255, th)
                if b % 2 == 0 and rng.uniform() < 0.7:
                    r = int(rng.integers(35, 121))
                    cv2.circle(imgs[c], (int(rng.integers(r, 640 - r)), int(rng.integers(r, 480 - r))), r, 255, int(rng.integers(1, 4)))
            if all(expected(imgs[c] > 0)[1] == 0 for c in range(C)):
                break
        frames[b] = np.maximum(imgs, rng.integers(0, 52, size=imgs.shape, dtype=np.uint8))
    return frames


@pytest.mark.parametrize("C,B", [(2, 16), (4, 10), (8, 8)])
def test_large_rings_through_every_pipeline(torch, C, B):
    """Frame-sets with rings of 70-240 px beside ring markers, with the window on, through the single-pass kernel and the
    three-kernel pipeline, with the winners' pixels, and through the host entry point:
    equal to the oracle's find_dot + match_and_triangulate per frame-set (cv2's lists), bit-equal across pipelines."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(140 + C)
    poses, K = synth.make_rig(C)
    frames = _large_ring_sets(rng, C, B, poses, K)
    port = RefPort([K] * C)
    ref, large = [], 0
    for fs in frames:
        lists = []
        for img in fs:
            items, _ = expected(img > 51)
            large += retr_tree_blobs(img > 51)[2] > 62
            lists.append([list(it[4:]) for it in items])
        e, o, ch = port.match_and_triangulate(lists, poses)
        ref.append((e, np.asarray(o, dtype=np.float64).reshape(-1, 3), ch, 0))
    assert large >= B // 3
    batch = torch.from_numpy(frames).cuda()
    results = {}
    for mode in ("fused", "split"):
        os.environ["MOCAP_PIPELINE"] = mode
        try:
            ctx = pkg.MocapContext(C, 640, 480, max_blobs=64, max_roots=128, max_cands=16, max_groups=1 << 16, max_segments=4096)
        finally:
            os.environ.pop("MOCAP_PIPELINE", None)
        ctx.set_large_holes(True)
        ctx.set_cameras([K] * C, poses)
        out = ctx.pipeline(batch, want_tracks=True)
        torch.cuda.synchronize()
        run = {k: v.cpu().numpy().copy() for k, v in out.items()}
        _assert_equals_oracle(out, ref, C)
        host = ctx.pipeline_host(frames)
        assert _same_bits({k: v.numpy() for k, v in host.items()}, run), mode
        results[mode] = run
    assert _same_bits(results["fused"], results["split"])


def test_raw_frames_with_large_ring_markers_vs_oracle_chain(torch):
    """pipeline_raw with the window on, hard-edged disc markers of radius 2-14 px and, in every frame-set, one of 40-60 px
    that the reference's blur and sharpen turn into a ring over 62 px: equal to the oracle's preprocess -> find_dot ->
    match_and_triangulate."""
    import cv2
    from oracle.ref_port import RefPort
    rotations, in_w, in_h, B = (0, 2), 320, 240, 6
    C, S = len(rotations), in_w
    rng = np.random.default_rng(77)
    raw, K, poses = raw_marker_frames(rng, B, in_w, in_h, rotations)
    for b in range(B):
        for c in range(C):
            cv2.circle(raw[b, c], (int(rng.integers(70, 250)), int(rng.integers(70, 170))), int(rng.integers(40, 61)), (255, 255, 255), -1)
    ctx = pkg.MocapContext(C, S, S, max_blobs=64, max_roots=64, max_cands=16, max_segments=4096)
    ctx.set_large_holes(True)
    ctx.set_preprocess(in_w, in_h, list(rotations), [K] * C, [DIST] * C)
    ctx.set_cameras([K] * C, poses)
    out = ctx.pipeline_raw(torch.from_numpy(raw).cuda())
    port = RefPort([K] * C)
    n = out["n"].cpu().numpy(); obj = out["obj"].cpu().numpy(); err = out["err"].cpu().numpy(); fl = out["flags"].cpu().numpy()
    large = 0
    for b in range(B):
        pts = []
        for c in range(C):
            f = port.preprocess(raw[b, c], c, DIST, rotations[c])
            _, _, side, holes = retr_tree_blobs(cv2.cvtColor(f, cv2.COLOR_RGB2GRAY) > 51)
            large += side > 62
            pts.append(port.find_dot(f.copy()))
        e, o, _ = port.match_and_triangulate(pts, poses)
        assert n[b] == len(e) and fl[b] == 0, (b, int(n[b]), len(e), int(fl[b]))
        if len(e):
            o = np.asarray(o, dtype=np.float64)
            scale = np.maximum(1.0, np.abs(o).max(axis=1, keepdims=True))
            assert (np.abs(obj[b, :n[b]] - o) / scale).max() <= 1e-7, b
            assert np.allclose(err[b, :n[b]], e, rtol=1e-9, atol=1e-12), b
    print(f"raw: {large} of {B * C} frames with a holed blob over 62 px")
    assert large >= B * C // 2


def test_drop_in_find_dot(torch):
    """find_dot through a MocapSession(large_holes=True) returns cv2's list on a 100-px ring (two contours, the hole's
    centre included); the default session raises, as before."""
    import cv2
    from oracle.ref_port import RefPort
    img = np.zeros((480, 640, 3), np.uint8)
    cv2.circle(img, (300, 200), 50, (255, 255, 255), 3)
    cv2.circle(img, (500, 400), 6, (255, 255, 255), -1)
    K = np.eye(3)
    want = RefPort([K]).find_dot(img.copy())
    s = pkg.MocapSession([K], large_holes=True)
    _, got = pkg.find_dot(img.copy(), s)
    assert got == [list(p) for p in want] and len(got) == 3
    with pytest.raises(pkg.MocapError):
        pkg.find_dot(img.copy(), pkg.MocapSession([K]))

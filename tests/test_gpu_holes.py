"""S1's blobs with holes on the device, held to cv2 itself: cv.findContours(RETR_TREE) + cv.moments reproduced by the
RETR_TREE slow path (csrc/blob_holes.cuh, blob_holes_cta in csrc/blob_device.cuh) -- a random fuzz at three image sizes
and in the H x W x 3 layout, both sides of every limit of that path, holed images inside multi-camera frame-sets
through every pipeline, and the raw-frame chain in which hard-edged markers become rings.  Run with ``-m gpu``."""
import importlib
import os

import numpy as np
import pytest

from tests.util import porous_patch, retr_tree_blobs, set_pixel_blobs

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth

X_TOL = 1e-7          # pose units, as tests/test_parity_gpu.py
ERR_RTOL = 1e-9
F_BLOBS, F_HOLES = 2, 32
WINDOW = 62           # widest / tallest holed blob the slow path takes
HOLE_CAP = 64         # holes per image it takes


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def expected_blobs(binary, max_blobs):
    """What S1 must report for a binary image: (items (A2, SX6, SY6, npix, x, y) truncated to max_blobs, flags).
    Within the slow path's limits that is cv2's RETR_TREE list; beyond them the set-pixel list and MOCAP_F_HOLES."""
    items, _, side, holes = retr_tree_blobs(binary)
    flags = 0
    if side > WINDOW or holes > HOLE_CAP:
        items, flags = set_pixel_blobs(binary), F_HOLES
    if len(items) > max_blobs:
        flags |= F_BLOBS
    return items[:max_blobs], flags


def device_items(d, i):
    n = int(d["n"][i])
    mom, xy = d["mom"][i, :n].cpu().numpy(), d["xy"][i, :n].cpu().numpy()
    return [tuple(int(v) for v in mom[k]) + tuple(int(v) for v in xy[k]) for k in range(n)]


def _first_diff(got, want):
    """(index, device item, expected item) of the first difference of two item lists, for failure messages"""
    for k in range(max(len(got), len(want))):
        a = got[k] if k < len(got) else None
        b = want[k] if k < len(want) else None
        if a != b:
            return k, a, b
    return None


# ------------------------------------------------------------------------------------------------ fuzz
def _draw_shapes(rng, img, colour, solid_only):
    """Random holed and solid shapes: rings, rectangular frames (some with a blob inside), porous patches, rings in
    rings, 1-px holes, holes that touch diagonally, lopsided ellipse rings; near 16-px segment borders and cut by the
    four image borders."""
    import cv2
    H, W = img.shape[:2]
    for _ in range(int(rng.integers(2, 10))):
        kind = int(rng.integers(7, 10)) if solid_only else int(rng.integers(0, 10))
        cx, cy = int(rng.integers(-4, W + 4)), int(rng.integers(-4, H + 4))
        if rng.uniform() < 0.3:
            cx = 16 * (cx // 16) + int(rng.integers(-1, 2))                  # on a segment border
        v = colour()
        if kind == 0:
            cv2.circle(img, (cx, cy), int(rng.integers(2, 15)), v, int(rng.integers(1, 4)))
        elif kind == 1:
            w, h = int(rng.integers(3, 40)), int(rng.integers(3, 30))
            if rng.uniform() < 0.3:                                          # a wall on an image border
                side = int(rng.integers(0, 4))
                cx, cy = [(0, cy), (W - 1 - w, cy), (cx, 0), (cx, H - 1 - h)][side]
            cv2.rectangle(img, (cx, cy), (cx + w, cy + h), v, int(rng.integers(1, 3)))
            if rng.uniform() < 0.5:
                cv2.circle(img, (cx + w // 2, cy + h // 2), int(rng.integers(0, 2)), colour(), -1)     # a blob inside
        elif kind == 2:
            h, w = int(rng.integers(5, 17)), int(rng.integers(5, 25))
            m = rng.uniform(size=(h, w)) < rng.uniform(0.6, 0.85)
            y0, x0 = min(max(cy, 0), H - h), min(max(cx, 0), W - w)
            img[y0:y0 + h, x0:x0 + w][m] = v
        elif kind == 3:
            cv2.circle(img, (cx, cy), int(rng.integers(8, 15)), v, 1)
            cv2.circle(img, (cx, cy), int(rng.integers(2, 6)), colour(), int(rng.integers(1, 3)))
        elif kind == 4:
            y0, x0 = min(max(cy, 0), H - 5), min(max(cx, 0), W - 5)
            img[y0:y0 + 5, x0:x0 + 5] = v
            img[y0 + 2, x0 + 2] = 0                                          # 1-px hole (1-px walls around it)
        elif kind == 5:
            y0, x0 = min(max(cy, 0), H - 6), min(max(cx, 0), W - 6)
            img[y0:y0 + 6, x0:x0 + 6] = v
            img[y0 + 2, x0 + 2] = 0                                          # two holes touching diagonally
            img[y0 + 3, x0 + 3] = 0
        elif kind == 6:
            cv2.ellipse(img, (cx, cy), (int(rng.integers(3, 20)), int(rng.integers(2, 12))), float(rng.uniform(0, 180)),
                        0, 360, v, 1)
        elif kind == 7:
            cv2.circle(img, (cx, cy), int(rng.integers(1, 9)), v, -1)
        elif kind == 8:
            img[max(cy, 0):cy + int(rng.integers(1, 6)), max(cx, 0):cx + int(rng.integers(1, 24))] = v
        else:
            pts = (np.array([[cx, cy]]) + rng.integers(-8, 9, size=(int(rng.integers(3, 7)), 2))).astype(np.int32)
            cv2.fillPoly(img, [pts], v)


def fuzz_frames(rng, n, H, W, max_blobs, channels=1):
    """n random frames within the slow path's limits (and max_blobs), each with its expected items; frames beyond the
    limits are drawn again.  channels == 3: unequal channels, the grey image is cv2's RGB2GRAY."""
    import cv2
    frames, refs = [], []
    while len(frames) < n:
        if channels == 1:
            img = np.zeros((H, W), np.uint8)
            _draw_shapes(rng, img, lambda: int(rng.integers(52, 256)), rng.uniform() < 0.15)
            img = np.maximum(img, rng.integers(0, 52, size=(H, W), dtype=np.uint8))
            grey = img
        else:
            img = np.zeros((H, W, 3), np.uint8)

            def colour():
                c = rng.integers(0, 256, size=3)
                if rng.uniform() < 0.2:                  # one bright channel; grey just above / at the threshold
                    c = [(0, 0, 255), (255, 0, 0), (52, 52, 52), (51, 51, 51)][int(rng.integers(0, 4))]
                return tuple(int(v) for v in c)
            _draw_shapes(rng, img, colour, rng.uniform() < 0.15)
            img = np.maximum(img, rng.integers(0, 46, size=(H, W, 3), dtype=np.uint8))
            grey = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
        items, holes_kept, side, holes = retr_tree_blobs(grey > 51)
        if side > WINDOW or holes > HOLE_CAP or len(items) > max_blobs:
            continue
        frames.append(img)
        refs.append((items, holes_kept))
    return np.stack(frames), refs


@pytest.mark.parametrize("W,H,n,channels", [(640, 480, 400, 1), (1024, 768, 60, 1), (336, 200, 150, 1), (640, 480, 100, 3)])
def test_holed_blob_fuzz_vs_cv2(torch, W, H, n, channels):
    """Random frames of holed and solid blobs through mocap_detect_dev: count, centres and order equal cv2's RETR_TREE
    list; A2, SX6, SY6 equal round(2 m00), round(6 m10), round(6 m01) of every kept contour, hole contours included; the
    pixel count is a blob's 8-connected area, or the size of the region a hole encloses; no flag.  1024 x 768 runs the
    64-bit-accumulator build, 336 x 200 a ragged segment count, and the 3-channel layout cv2's RGB2GRAY."""
    rng = np.random.default_rng(W + H + channels)
    frames, refs = fuzz_frames(rng, n, H, W, 64, channels)
    ctx = pkg.MocapContext(1, W, H, max_blobs=64, max_segments=4096)
    d = ctx.detect(torch.from_numpy(frames).cuda(), want_moments=True)
    fl = d["flags"].cpu().numpy()
    holed_frames = contours = hole_contours = 0
    for i, (items, holes_kept) in enumerate(refs):
        assert fl[i] == 0, (i, int(fl[i]))
        got = device_items(d, i)
        assert got == items, (i, _first_diff(got, items))
        holed_frames += holes_kept > 0
        contours += len(items)
        hole_contours += holes_kept
    print(f"{W}x{H}x{channels}: {n} frames, {holed_frames} with holes, {contours} contours, {hole_contours} of them holes")
    assert holed_frames >= (150 if n >= 400 else n // 3) and hole_contours >= 2 * holed_frames


# ------------------------------------------------------------------------------------------------ limits
def _lopsided_frame(img, x, y, w, h):
    """A 1-px rectangular frame w x h with a lump in one corner: its filled and set-pixel centres differ."""
    import cv2
    cv2.rectangle(img, (x, y), (x + w - 1, y + h - 1), 255, 1)
    img[y + 1:y + 4, x + 1:x + 5] = 255


def _porous(img, y, x, n_holes):
    img[y:y + 17, x:x + 21] = porous_patch(n_holes)


def limit_images(H=480, W=640):
    """(name, image, flagged) on both sides of every limit of the slow path."""
    import cv2
    cases = []

    def new():
        return np.zeros((H, W), np.uint8)
    for side in (WINDOW, WINDOW + 1):
        img = new(); _lopsided_frame(img, 100, 50, side, 20); cv2.circle(img, (400, 300), 6, 255, 1)
        cases.append((f"wide{side}", img, side > WINDOW))
        img = new(); _lopsided_frame(img, 300, 200, 20, side); cv2.circle(img, (40, 40), 6, 255, 1)     # ring filled first
        cases.append((f"tall{side}", img, side > WINDOW))
    img = new(); _lopsided_frame(img, 0, 0, W, H); cv2.circle(img, (320, 240), 7, 255, 2); img[100:104, 500:510] = 255
    cases.append(("around_image", img, True))
    for first, second in ((40, 24), (40, 25), (40, 40), (0, 64), (0, 65)):
        img = new()
        if first:
            _porous(img, 40, 60, first)
        _porous(img, 300, 90, second)                         # across the segment border at x = 96
        cases.append((f"holes{first}+{second}", img, first + second > HOLE_CAP))
    img = new()                                               # 15 concentric frames, 61 px: 30 nested contours
    for k in range(15):
        cv2.rectangle(img, (200 + 2 * k, 100 + 2 * k), (260 - 2 * k, 160 - 2 * k), 255, 1)
    img[130, 230] = 255                                       # and a one-pixel blob (no area: dropped) in the middle
    cases.append(("nested15", img, False))
    return cases


def test_slow_path_limits_on_both_sides(torch):
    """At each limit of the slow path -- a holed blob 62 / 63 px wide or tall, a frame around the whole image, 64 / 65
    holes (the cap met in the second of two blobs, or inside one), 15 nested frames -- the image is reproduced exactly
    on the near side; on the far side it keeps MOCAP_F_HOLES and reports the set-pixel polygon of every blob in reverse
    raster order, including the blobs filled before the limit was met.  max_blobs = 64 leaves MOCAP_F_BLOBS and cv2's
    first 64 contours where an image has more."""
    cases = limit_images()
    imgs = np.stack([c[1] for c in cases])
    ctx = pkg.MocapContext(1, 640, 480, max_blobs=64, max_segments=4096)
    d = ctx.detect(torch.from_numpy(imgs).cuda(), want_moments=True)
    fl = d["flags"].cpu().numpy()
    from scipy import ndimage
    for i, (name, img, flagged) in enumerate(cases):
        items, flags = expected_blobs(img > 0, 64)
        assert bool(flags & F_HOLES) == flagged, name
        if flagged:                                          # the set-pixel and the filled centres differ
            filled = set_pixel_blobs(ndimage.binary_fill_holes(img > 0))
            assert [it[4:] for it in items] != [it[4:] for it in filled], name
        got = device_items(d, i)
        assert int(fl[i]) == flags and got == items, (name, int(fl[i]), flags, _first_diff(got, items))
    assert len(retr_tree_blobs(cases[-1][1] > 0)[0]) == 30
    # twice on the same context: the full-size reduction's scratch re-arms
    d2 = ctx.detect(torch.from_numpy(imgs).cuda(), want_moments=True)
    assert torch.equal(d2["n"], d["n"]) and torch.equal(d2["flags"], d["flags"])
    for i in range(len(cases)):
        assert device_items(d2, i) == device_items(d, i)


def test_more_contours_than_max_blobs(torch):
    """More contours than max_blobs: MOCAP_F_BLOBS and the first max_blobs of cv2's list (holes counted as contours);
    on a flagged image the first max_blobs of the set-pixel list beside MOCAP_F_HOLES."""
    import cv2
    imgs = np.zeros((3, 480, 640), np.uint8)
    for k in range(12):
        cv2.circle(imgs[0], (30 + 50 * k, 100 + 7 * k), 5 + (k % 3), 255, 1)          # 12 rings: 24 contours
        cv2.circle(imgs[1], (30 + 50 * k, 300), 4, 255, -1)                             # 12 discs
        cv2.circle(imgs[2], (30 + 50 * k, 400), 5, 255, 2)                             # (a 1-px ring has no set-pixel area)
    cv2.circle(imgs[1], (320, 150), 6, 255, 1)                                         # 14 contours in all
    cv2.circle(imgs[2], (320, 150), 70, 255, 2)                                        # 140 px: flagged, 13 blobs
    ctx = pkg.MocapContext(1, 640, 480, max_blobs=10, max_segments=4096)
    d = ctx.detect(torch.from_numpy(imgs).cuda(), want_moments=True)
    for i, want in enumerate((F_BLOBS, F_BLOBS, F_BLOBS | F_HOLES)):
        items, flags = expected_blobs(imgs[i] > 0, 10)
        assert flags == want and len(items) == 10
        assert int(d["flags"][i]) == want and device_items(d, i) == items, i


# ---------------------------------------------------------------------------------------- frame-sets
def _ring_frame_sets(rng, C, B, poses, K):
    """B frame-sets of C 640 x 480 images: ring markers (radius 3-14, thickness 1-3) at the projections of random 3D
    points; every third frame-set solid discs; the frame-set B // 2 also holds a ring too large for the slow path."""
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
                    if b % 3 == 2:
                        cv2.circle(imgs[c], (int(round(u)), int(round(v))), max(2, r // 3), 255, -1)
                    else:
                        cv2.circle(imgs[c], (int(round(u)), int(round(v))), r, 255, th)
            if b == B // 2:
                cv2.circle(imgs[C - 1], (90, 90), 40, 255, 2)
            ok = True
            for c in range(C):
                _, fl = expected_blobs(imgs[c] > 0, 64)
                ok &= fl == (F_HOLES if (b == B // 2 and c == C - 1) else 0)
            if ok:
                break
        frames[b] = np.maximum(imgs, rng.integers(0, 52, size=imgs.shape, dtype=np.uint8))
    return frames


def _oracle_sets(port, poses, frames):
    """Per frame-set: (errors, points, chosen groups, flags) of the oracle's matcher on what S1 must report."""
    out = []
    for fs in frames:
        lists, flags = [], 0
        for img in fs:
            items, fl = expected_blobs(img > 51, 64)
            lists.append([list(it[4:]) for it in items])
            flags |= fl
        e, o, ch = port.match_and_triangulate(lists, poses)
        out.append((e, np.asarray(o, dtype=np.float64).reshape(-1, 3), ch, flags))
    return out


def _assert_equals_oracle(out, ref, C, tracks=True):
    n = out["n"].cpu().numpy(); obj = out["obj"].cpu().numpy(); err = out["err"].cpu().numpy(); fl = out["flags"].cpu().numpy()
    txy = out["track_xy"].cpu().numpy() if tracks else None
    for b, (e, o, ch, flags) in enumerate(ref):
        assert n[b] == len(e) and fl[b] == flags, (b, int(n[b]), len(e), int(fl[b]), flags)
        k = len(e)
        if not k:
            continue
        scale = np.maximum(1.0, np.abs(o).max(axis=1, keepdims=True))      # a wrong correspondence is ill-conditioned
        assert (np.abs(obj[b, :k] - o) / scale).max() <= X_TOL, b
        assert np.allclose(err[b, :k], e, rtol=ERR_RTOL, atol=1e-12), b
        if tracks:
            want = np.array([[[-1, -1] if p[0] is None else p for p in g] for g in ch], np.int32).reshape(k, C, 2)
            assert np.array_equal(txy[b, :k], want), b


def _same_bits(a, b):
    """two pipeline results (host arrays) agree bit for bit on every output both carry"""
    n = a["n"]
    if not (np.array_equal(n, b["n"]) and np.array_equal(a["flags"], b["flags"])):
        return False
    keys = [k for k in ("obj", "err", "track_xy") if k in a and k in b]
    return all(np.array_equal(a[k][s, :n[s]], b[k][s, :n[s]]) for s in range(len(n)) for k in keys)


@pytest.mark.parametrize("C,B", [(2, 18), (4, 12), (8, 9)])
def test_holed_frame_sets_through_every_pipeline(torch, C, B):
    """Frame-sets whose images hold ring markers (an outer and a hole contour, often with the same centre: the matcher's
    epipolar distances tie exactly), solid frame-sets and one flagged frame-set, through the single-pass kernel, the
    three-kernel pipeline and the phase-synchronous variant (MOCAP_PIPELINE = fused | split | phased), with the winners'
    pixels, and through the host entry point: counts, points, errors, flags and winners' pixels equal the oracle's
    find_dot + match_and_triangulate per frame-set; the pipelines agree bit for bit, and so does a second call."""
    from oracle.ref_port import RefPort
    rng = np.random.default_rng(40 + C)
    poses, K = synth.make_rig(C)
    frames = _ring_frame_sets(rng, C, B, poses, K)
    ref = _oracle_sets(RefPort([K] * C), poses, frames)
    assert sum(len(r[0]) for r in ref) >= B and ref[B // 2][3] == F_HOLES
    batch = torch.from_numpy(frames).cuda()
    results = {}
    for mode in ("fused", "split", "phased"):
        os.environ["MOCAP_PIPELINE"] = mode
        try:
            ctx = pkg.MocapContext(C, 640, 480, max_blobs=64, max_roots=128, max_cands=16, max_groups=1 << 16, max_segments=4096)
        finally:
            os.environ.pop("MOCAP_PIPELINE", None)
        ctx.set_cameras([K] * C, poses)
        runs = []
        for _ in range(2):                                   # the deferral worklists re-arm
            out = ctx.pipeline(batch, want_tracks=True)
            torch.cuda.synchronize()
            runs.append({k: v.cpu().numpy().copy() for k, v in out.items()})
        _assert_equals_oracle(out, ref, C)
        assert _same_bits(runs[0], runs[1]), mode
        host = ctx.pipeline_host(frames)
        assert _same_bits({k: v.numpy() for k, v in host.items()}, runs[0]), mode
        results[mode] = runs[0]
    assert _same_bits(results["fused"], results["split"]) and _same_bits(results["fused"], results["phased"])


# ---------------------------------------------------------------------------------------- raw frames
DIST = [-1.26372388e-01, 2.62661497e-01, 1.21306197e-03, 2.24507008e-04, -2.48534118e-01]


def raw_marker_frames(rng, B, in_w, in_h, rotations):
    """B frame-sets of raw in_h x in_w x 3 frames (dark clutter) with 2-4 hard-edged white discs of radius 2-14 px at
    the projections of random 3D points on cameras along x; the output square is S = in_w.  Returns (raw, K, poses)."""
    import cv2
    C, S = len(rotations), in_w
    ay = (S - in_h) // 2                                      # make_square's row offset
    K = np.array([[S * 1.0, 0, S / 2], [0, S * 1.0, S / 2], [0, 0, 1]])
    poses = [{"R": np.eye(3), "t": np.array([-0.3 * c, 0.0, 0.0])} for c in range(C)]
    raw = rng.integers(0, 25, size=(B, C, in_h, in_w, 3), dtype=np.uint8)
    for b in range(B):
        for _ in range(int(rng.integers(2, 5))):
            X = np.array([rng.uniform(-0.35, 0.35), rng.uniform(-0.2, 0.2), rng.uniform(2.0, 3.0)])
            r = int(rng.integers(2, 15))
            for c in range(C):
                pc = poses[c]["R"] @ X + poses[c]["t"]
                u, v = S * pc[0] / pc[2] + S / 2, S * pc[1] / pc[2] + S / 2 - ay
                if rotations[c] == 2:                         # the frame is turned by 180 degrees before make_square
                    u, v = in_w - 1 - u, in_h - 1 - v
                cv2.circle(raw[b, c], (int(round(u)), int(round(v))), r, (255, 255, 255), -1)
    return raw, K, poses


@pytest.mark.parametrize("in_w,in_h,rotations", [(320, 240, (0, 2)), (320, 240, (2, 0, 2)), (208, 160, (0, 2))])
def test_raw_frames_with_ring_markers_vs_oracle_chain(torch, in_w, in_h, rotations):
    """Hard-edged disc markers of radius 2-14 px on raw frames: from about 8 px on, the reference's blur and sharpen
    make them rings.  pipeline_raw(want_frames=True) against the oracle's preprocess -> find_dot -> match_and_triangulate:
    the processed frames bit for bit, then counts, points and errors; a quarter of the marker frames at least has a
    hole.  208 x 160 raw frames give 208 x 208 output, not a multiple of the 64-px preprocessing tile."""
    import cv2
    from oracle.ref_port import RefPort
    C, S, B = len(rotations), in_w, 8
    raw, K, poses = raw_marker_frames(np.random.default_rng(in_h + C), B, in_w, in_h, rotations)
    ctx = pkg.MocapContext(C, S, S, max_blobs=64, max_roots=64, max_cands=16, max_segments=4096)
    ctx.set_preprocess(in_w, in_h, list(rotations), [K] * C, [DIST] * C)
    ctx.set_cameras([K] * C, poses)
    out = ctx.pipeline_raw(torch.from_numpy(raw).cuda(), want_frames=True)
    port = RefPort([K] * C)
    n = out["n"].cpu().numpy(); obj = out["obj"].cpu().numpy(); err = out["err"].cpu().numpy()
    fl = out["flags"].cpu().numpy(); got_frames = out["frames"].cpu().numpy()
    holed = total = 0
    for b in range(B):
        pts = []
        for c in range(C):
            f = port.preprocess(raw[b, c], c, DIST, rotations[c])
            assert np.array_equal(got_frames[b, c], f), (b, c)
            grey = cv2.cvtColor(f, cv2.COLOR_RGB2GRAY) > 51
            _, kept_holes, side, holes = retr_tree_blobs(grey)
            assert side <= WINDOW and holes <= HOLE_CAP
            holed += holes > 0
            pts.append(port.find_dot(f.copy()))
        e, o, _ = port.match_and_triangulate(pts, poses)
        assert n[b] == len(e) and fl[b] == 0, (b, int(n[b]), len(e), int(fl[b]))
        total += len(e)
        if len(e):
            o = np.asarray(o, dtype=np.float64)
            scale = np.maximum(1.0, np.abs(o).max(axis=1, keepdims=True))
            assert (np.abs(obj[b, :n[b]] - o) / scale).max() <= X_TOL, b
            assert np.allclose(err[b, :n[b]], e, rtol=ERR_RTOL, atol=1e-12), b
    print(f"raw {in_w}x{in_h} C={C}: {holed} of {B * C} frames with a hole, {total} points")
    assert 4 * holed >= B * C and total >= B
    again = ctx.pipeline_raw(torch.from_numpy(raw).cuda())
    assert np.array_equal(again["n"].cpu().numpy(), n) and np.array_equal(again["flags"].cpu().numpy(), fl)
    for b in range(B):
        assert np.array_equal(again["obj"].cpu().numpy()[b, :n[b]], obj[b, :n[b]])

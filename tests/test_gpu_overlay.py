"""The detection overlay on the H100 (mocap_set_overlay, mocap_overlay_dev, find_dot and install_into(overlay=True)):
the golden live session's frames and stream JPEG against cv2's drawing of the oracle chain's frames -- _find_dot's
contours, labels and pluses, and in triangulate mode the matcher's epipolar lines in the seeded palette's colours --
the batched entry and both mirrors on random scenes, a line counter that carries across calls and wraps, a batch that
splits into launch groups, and the overlay off leaving every output as a context that never drew it."""
import importlib

import numpy as np
import pytest

from tests.live_util import (CAPTURE, DIST, IN_H, IN_W, K, LOCATE, TRIANGULATE, golden_scene, load_golden, make_scene,
                             render_read, timestamp)
from tests.overlay_util import epilines_drawn, find_dot_drawn, palette_of, sparse_scene

pytestmark = pytest.mark.gpu
api = importlib.import_module("low-cost-mocap_b200.api")
pkg = importlib.import_module("low-cost-mocap_b200")
FULL = CAPTURE | TRIANGULATE | LOCATE
KEYS = ("flags", "gate", "blob_n", "first", "n", "n_objects", "called", "pos", "vel", "heading", "present", "chosen")


def _ctx(scene, overlay, world=None):
    C = scene["C"]
    ctx = api.MocapContext(C, 320, 320, **api.MIRROR_LIMITS)
    if overlay:
        ctx.set_overlay(True)
    ctx.set_preprocess(IN_W, IN_H, scene["rotations"], [K] * C, [DIST] * C)
    ctx.set_cameras([K] * C, scene["poses"])
    ctx.set_world_transform(world)
    return ctx


def _drawn(port, scene, raw, mode, palette=None, n=0):
    """The oracle of one read's returned frames: RefPort preprocessing, _find_dot's drawing when capturing, then the
    epipolar lines when triangulating, line n of the session in palette[n % L].  Returns (frames, the session's line
    count after the read)."""
    frames = np.stack([port.preprocess(raw[c], c, DIST, scene["rotations"][c]) for c in range(scene["C"])])
    if mode & CAPTURE:
        pts = [find_dot_drawn(frames[c])[1] for c in range(scene["C"])]
        if mode & TRIANGULATE:
            n = epilines_drawn(port, frames, pts, scene["poses"], palette, n)
    return frames, n


def test_golden_session_through_live_dev():
    """Every read of the golden session through ctx.live(want_frames=True) with the overlay on: the frames equal cv2's
    drawing of the oracle's processed frames byte for byte, in capture, triangulate and locate mode."""
    import torch
    from oracle.ref_port import RefPort
    g = load_golden()
    scene = golden_scene(g)
    ctx = _ctx(scene, True, g["worlds"][0])
    ctx.set_overlay(True, seed=3)
    palette = palette_of(3)
    tr = ctx.tracker(int(g["num_objects"]))
    port = RefPort([K] * 4)
    dev = ctx.torch_device
    n = 0
    for k in range(len(g["mode"])):
        mode = int(g["mode"][k])
        raw = render_read(scene, k, bool(g["dark"][k]))
        ts = torch.tensor([timestamp(k)], dtype=torch.float64, device=dev) if mode & LOCATE else None
        out = ctx.live(torch.from_numpy(raw[None]).to(dev), mode, ts, tr if mode & LOCATE else None, want_frames=True)
        want, n = _drawn(port, scene, raw, mode, palette, n)
        assert np.array_equal(out["frames"][0].cpu().numpy(), want), k
    assert n > 300


def test_golden_session_through_the_stream_drop_in(monkeypatch):
    """install_into(live=True, stream=True, overlay=True) over the golden session: get_frames() is np.hstack of the drawn
    oracle frames and index.cv.imencode('.jpg', get_frames()) returns cv2.imencode's bytes of them; _find_dot draws as
    the reference's does."""
    import cv2
    from oracle.ref_port import RefPort
    from tests.test_gpu_jpeg import _standin_modules
    g = load_golden()
    scene = golden_scene(g)
    monkeypatch.setattr(api.MocapSession, "_default", None)
    k_now = [0]
    plain_read = api.camera_read
    monkeypatch.setattr(api, "camera_read", lambda cams, s=None, clock=None, jpeg=None:
                        plain_read(cams, s, clock=lambda: timestamp(k_now[0]), jpeg=jpeg))
    cams, helpers, index = _standin_modules(g, scene)
    pkg.install_into(helpers, index, live=True, stream=True, overlay=True, overlay_seed=8)
    palette = palette_of(8)
    port = RefPort([K] * 4)
    n = 0
    for k in range(len(g["mode"])):
        k_now[0] = k
        cams.set_read(k)
        want, n = _drawn(port, scene, render_read(scene, k, bool(g["dark"][k])), int(g["mode"][k]), palette, n)
        want = np.hstack(list(want))
        got = cams.get_frames()
        assert np.array_equal(np.asarray(got), want), k
        ok, buf = index.cv.imencode(".jpg", got)
        assert ok and np.array_equal(buf, cv2.imencode(".jpg", want)[1]), k
    frame = port.preprocess(render_read(scene, 3)[1], 1, DIST, scene["rotations"][1])
    want, pts = find_dot_drawn(frame.copy())
    got, got_pts = cams._find_dot(frame.copy())
    assert np.array_equal(got, want) and got_pts == pts


@pytest.mark.parametrize("W,H", [(208, 144), (320, 320), (640, 480)])
def test_batched_entry_and_find_dot_on_random_scenes(W, H):
    """mocap_overlay_dev on a batch of random scenes (blobs on the edges, holed blobs, rings, 1-px dots) with detect's blob lists,
    and find_dot on a session with overlay=True, frame by frame: both equal cv2's drawing of _find_dot."""
    import torch
    rng = np.random.default_rng(W + H)
    imgs = np.stack([sparse_scene(rng, H, W, int(rng.integers(0, 24))) for _ in range(40)])
    ctx = api.MocapContext(1, W, H, **api.MIRROR_LIMITS)
    frames = torch.from_numpy(imgs).to(ctx.torch_device)
    d = ctx.detect(frames)
    ctx.overlay(frames, d["xy"], d["n"])
    got = frames.cpu().numpy()
    flags = d["flags"].cpu().numpy()
    session = api.MocapSession([K], W, H, overlay=True)
    compared = labels = 0
    for i in range(len(imgs)):
        if flags[i]:
            continue
        want, pts = find_dot_drawn(imgs[i].copy())
        assert np.array_equal(got[i], want), i
        img, mp = api.find_dot(imgs[i].copy(), session)
        assert np.array_equal(img, want) and mp == (pts if pts else [[None, None]]), i
        compared += 1
        labels += len(pts)
    assert compared >= 36 and labels > 200


def test_a_batch_across_launch_groups():
    """520 reads of 8 cameras (launch groups of 512 reads) in one ctx.live call with the overlay on: every read's frames
    equal the drawn oracle frames of its raw frames, across the group boundary."""
    import torch
    from oracle.ref_port import RefPort
    g = load_golden()
    scene = make_scene(12, g["worlds"][0], C=8, rotations=[0, 2, 2, 0, 0, 2, 2, 0])
    ctx = _ctx(scene, True)
    distinct = np.stack([render_read(scene, k) for k in range(6)])
    port = RefPort([K] * 8)
    want = torch.from_numpy(np.stack([_drawn(port, scene, distinct[k], CAPTURE)[0] for k in range(6)])).to(ctx.torch_device)
    B = 520
    raw = torch.from_numpy(distinct).to(ctx.torch_device)[torch.arange(B) % 6].contiguous()
    n0 = ctx.launch_count()
    out = ctx.live(raw, CAPTURE, want_frames=True)
    torch.cuda.synchronize()
    frames = out["frames"]
    for r in range(B):
        assert torch.equal(frames[r], want[r % 6]), r
    del out, frames, raw
    assert ctx.launch_count() - n0 == 2 * (5 + 2)          # per group: preprocessing, S1 (3), k_live_blobs, the overlay (2)


def test_off_is_bit_identical_to_a_context_that_never_drew():
    """set_overlay(True) then set_overlay(False): results, frames and JPEG equal those of a context that never drew the
    overlay, bit for bit; with it on, every output but the frames and the JPEG stays the same too."""
    g = load_golden()
    scene = make_scene(6, g["worlds"][0])
    raw = np.stack([render_read(scene, k, dark=k == 3) for k in range(6)])
    ts = np.array([timestamp(k) for k in range(6)])
    never, off, on = (_ctx(scene, False, g["worlds"][0]) for _ in range(3))
    off.set_overlay(True)
    off.set_overlay(False)
    on.set_overlay(True)
    outs = [c.live_host(raw, FULL, ts, c.tracker(2), want_frames=True, jpeg=True) for c in (never, off, on)]
    a, b, c = outs
    for key in KEYS + ("frames", "jpeg_len"):
        assert np.array_equal(a[key], b[key]), key
    for r in range(6):
        assert np.array_equal(a["jpeg"][r, :a["jpeg_len"][r]], b["jpeg"][r, :b["jpeg_len"][r]]), r
        n, m = int(a["n"][r]), int(a["n_objects"][r])
        for key, cnt in (("obj", n), ("err", n), ("objects", m), ("drone_index", m)):
            assert np.array_equal(a[key][r, :cnt], b[key][r, :cnt]) and np.array_equal(a[key][r, :cnt], c[key][r, :cnt]), (r, key)
    for key in KEYS:
        assert np.array_equal(a[key], c[key]), key
    assert not np.array_equal(a["frames"], c["frames"])
    # mode 0 draws nothing, on or off
    z_off, z_on = never.live_host(raw[:2], 0, want_frames=True), on.live_host(raw[:2], 0, want_frames=True)
    assert np.array_equal(z_off["frames"], z_on["frames"])


def test_line_counter_carries_across_calls_and_wraps():
    """A palette of 7 colours, live calls of 1, 4 and 9 reads in triangulate mode: every read's lines take the colours
    the session's running line count gives, across reads of a batch, across calls and around the palette; set_overlay
    starts the count again."""
    import torch
    from oracle.ref_port import RefPort
    g = load_golden()
    scene = make_scene(6, g["worlds"][0])
    ctx = _ctx(scene, True, g["worlds"][0])
    port = RefPort([K] * 4)
    dev = ctx.torch_device
    for rounds in range(2):
        ctx.set_overlay(True, seed=5, palette_len=7)
        palette = palette_of(5, 7)
        n, k = 0, 0
        for B in (1, 4, 9):
            raw = np.stack([render_read(scene, k + r, dark=(k + r) % 6 == 2) for r in range(B)])
            out = ctx.live(torch.from_numpy(raw).to(dev), CAPTURE | TRIANGULATE, want_frames=True)
            got = out["frames"].cpu().numpy()
            for r in range(B):
                want, n = _drawn(port, scene, raw[r], CAPTURE | TRIANGULATE, palette, n)
                assert np.array_equal(got[r], want), (rounds, k + r)
            k += B
        assert n > 7 * 5


def test_matcher_mirror_draws_the_lines():
    """find_point_correspondance_and_object_points on a session with overlay=True draws the epipolar lines into the
    frames it returns, in place, with the session's line counter running from call to call (mocap_overlay_dev in
    triangulate mode); errors and points are those of the session without the overlay."""
    from oracle.ref_port import RefPort
    g = load_golden()
    scene = make_scene(9, g["worlds"][0])
    port = RefPort([K] * 4)
    drawn = api.MocapSession([K] * 4, 320, 320, overlay=True, overlay_seed=4)
    plain = api.MocapSession([K] * 4, 320, 320)
    palette = palette_of(4)
    n = 0
    for k in range(6):
        raw = render_read(scene, k)
        frames = [port.preprocess(raw[c], c, DIST, scene["rotations"][c]) for c in range(4)]
        pts = [port.find_dot(f) for f in frames]
        want = [f.copy() for f in frames]
        n = epilines_drawn(port, want, pts, scene["poses"], palette, n)
        got = [f.copy() for f in frames]
        e1, o1, out = api.find_point_correspondance_and_object_points([list(p) for p in pts], scene["poses"], got, drawn)
        e0, o0, _ = api.find_point_correspondance_and_object_points([list(p) for p in pts], scene["poses"], [f.copy() for f in frames], plain)
        assert out is got and all(np.array_equal(a, b) for a, b in zip(got, want)), k
        assert np.array_equal(e0, e1) and np.array_equal(o0, o1), k
    assert n > 40

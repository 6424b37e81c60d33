"""The JPEG encoder on the H100 (mocap_encode_jpeg_dev, mocap_live_jpeg_host, install_into(stream=True)): batches of
every size, content and quality against cv2.imencode byte for byte and against tests/golden/jpeg_cv2.npz, tiled input
against np.hstack, the golden live session through the stream drop-in, batched replay against single reads, overflow
and refusals."""
import ctypes
import importlib
import json
import types

import numpy as np
import pytest

from tests import jpeg_util as J
from tests.live_util import (CAPTURE, DIST, IN_H, IN_W, K, LOCATE, TRIANGULATE, StandinCameras, golden_scene, load_golden,
                             render_read, timestamp)

pytestmark = pytest.mark.gpu
api = importlib.import_module("low-cost-mocap_b200.api")
pkg = importlib.import_module("low-cost-mocap_b200")
FULL = CAPTURE | TRIANGULATE | LOCATE


@pytest.fixture(scope="module")
def ctx():
    return api.MocapContext(1, 64, 64)


def _host(res, i):
    n = int(res["len"][i])
    return res["jpeg"][i, :n].cpu().numpy() if n >= 0 else None


def _encode(ctx, imgs, quality, tiles=1, stride=None):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(imgs)).to(ctx.torch_device)
    res = ctx.encode_jpeg(d, tiles=tiles, quality=quality, stride=stride)
    torch.cuda.synchronize()
    return res


@pytest.mark.parametrize("h,w", J.SIZES)
def test_batches_equal_cv2(ctx, h, w):
    """Each size: a batch of every content at every quality, the bytes cv2.imencode gives, one by one."""
    imgs = np.stack([J.make_image(c, h, w, seed=1) for c in J.CONTENTS])
    bad = []
    for q in J.QUALITIES:
        res = _encode(ctx, imgs, q)
        for i, c in enumerate(J.CONTENTS):
            want = J.cv2_encode(imgs[i], q)
            got = _host(res, i)
            if got is None or not np.array_equal(got, want):
                bad.append((c, q, None if got is None else len(got), len(want)))
    assert not bad, bad


def test_golden_bytes(ctx):
    """The recorded cv2 4.13 / libjpeg-turbo 3.1.2 bytes, whatever cv2 this machine has."""
    for name, img, q, want in J.load_golden():
        got = _host(_encode(ctx, img[None], q), 0)
        assert got is not None and np.array_equal(got, want), name


@pytest.mark.parametrize("tiles", [2, 4, 8])
@pytest.mark.parametrize("th,tw", [(320, 320), (37, 29)])
def test_tiles_equal_hstack(ctx, tiles, th, tw):
    """images [n][tiles][th][tw][3] encode as cv2 encodes np.hstack of each image's frames."""
    rng = np.random.default_rng(tiles * 1000 + th)
    n = 3
    frames = np.stack([np.stack([J.make_image(J.CONTENTS[(i + t) % 5], th, tw, seed=int(rng.integers(1 << 20))) for t in range(tiles)])
                       for i in range(n)])
    for q in (75, 95):
        res = _encode(ctx, frames, q, tiles=tiles)
        for i in range(n):
            assert np.array_equal(_host(res, i), J.cv2_encode(np.hstack(list(frames[i])), q)), (i, q)


def _standin_modules(g, scene):
    """helpers / index stand-ins around a StandinCameras: Cameras is a Singleton-style wrapper (the replacements go to
    the class of its instance), index holds cv as index.py does (import cv2 as cv)."""
    import cv2

    class _Cams(StandinCameras):
        pass

    cams = _Cams(g, scene)
    helpers = types.ModuleType("helpers_standin")
    helpers.Cameras = types.SimpleNamespace(instance=lambda: cams)
    for name in api.PATCHED_NAMES:
        setattr(helpers, name, lambda *a: None)
    index = types.ModuleType("index_standin")
    index.cv = cv2
    return cams, helpers, index


def test_golden_session_through_the_stream_drop_in(monkeypatch):
    """install_into(live=True, stream=True) over the golden session, every read: get_frames() is np.hstack of the
    frames the live=True path returns, index.cv.imencode('.jpg', get_frames()) returns cv2's bytes of that array, and
    the events and serial bytes are those of the run without stream."""
    import cv2
    g = load_golden()
    scene = golden_scene(g)
    monkeypatch.setattr(api.MocapSession, "_default", None)
    k_now = [0]
    plain_read = api.camera_read
    monkeypatch.setattr(api, "camera_read", lambda cams, s=None, clock=None, jpeg=None:
                        plain_read(cams, s, clock=lambda: timestamp(k_now[0]), jpeg=jpeg))
    cams, helpers, index = _standin_modules(g, scene)
    pkg.install_into(helpers, index, live=True, stream=True)
    assert isinstance(index.cv, api.StreamCv) and index.cv.findFundamentalMat is cv2.findFundamentalMat
    ref = StandinCameras(g, scene)
    ref_session = api.MocapSession([K] * 4, 320, 320)
    sizes = []
    for k in range(len(g["mode"])):
        k_now[0] = k
        cams.set_read(k)
        ref.set_read(k)
        got = cams.get_frames()
        want_frames = plain_read(ref, ref_session, clock=lambda: timestamp(k))
        assert isinstance(got, api.StreamFrames) and np.array_equal(np.asarray(got), np.hstack(want_frames)), k
        ok, buf = index.cv.imencode(".jpg", got)
        assert ok and buf.dtype == np.uint8 and buf.ndim == 1
        assert np.array_equal(buf, cv2.imencode(".jpg", np.hstack(want_frames))[1]), k
        ok2, buf2 = index.cv.imencode(".jpg", got, [cv2.IMWRITE_JPEG_QUALITY, 95])
        assert np.array_equal(buf2, buf), k
        assert json.dumps(cams.events) == json.dumps(ref.events) and cams.lines == ref.lines, k
        sizes.append(len(buf))
    assert min(sizes) > 1000


def test_batched_live_then_encode_equals_per_read_jpegs():
    """live(..., want_frames=True) over a batch, then encode_jpeg(tiles=C), equals live_host(jpeg=True) read by read."""
    import torch
    g = load_golden()
    scene = golden_scene(g)
    B = 12

    def make():
        c = api.MocapContext(4, 320, 320, **api.MIRROR_LIMITS)
        c.set_preprocess(IN_W, IN_H, scene["rotations"], [K] * 4, [DIST] * 4)
        c.set_cameras([K] * 4, scene["poses"])
        c.set_world_transform(g["worlds"][0])
        return c
    a, b = make(), make()
    ta, tb = a.tracker(2), b.tracker(2)
    raw = np.stack([render_read(scene, k, dark=k == 5) for k in range(B)])
    ts = np.array([timestamp(k) for k in range(B)])
    dev = a.torch_device
    whole = a.live(torch.from_numpy(raw).to(dev), FULL, torch.from_numpy(ts).to(dev), ta, want_frames=True)
    enc = a.encode_jpeg(whole["frames"], tiles=4)
    torch.cuda.synchronize()
    for k in range(B):
        one = b.live_host(raw[k:k + 1], FULL, ts[k:k + 1], tb, want_frames=True, jpeg=True)
        want = one["jpeg"][0, :one["jpeg_len"][0]]
        assert np.array_equal(_host(enc, k), want), k
        assert np.array_equal(want, J.cv2_encode(np.hstack(list(one["frames"][0])), 95)), k


def test_overflow_and_refusals(ctx):
    """A stride below an image's length: len -1 and its row untouched (canary), its neighbours encoded; the host entry
    and Python raise; invalid quality, tiles or sizes: MOCAP_EINVAL before any launch."""
    import torch
    imgs = np.stack([J.make_image("noise", 64, 64, seed=2), J.make_image("constant", 64, 64, seed=2)])
    want = [J.cv2_encode(im, 95) for im in imgs]
    stride = (len(want[0]) + len(want[1])) // 2
    assert len(want[1]) <= stride < len(want[0])
    d = torch.from_numpy(imgs).to(ctx.torch_device)
    big = len(want[0]) + 64
    out = torch.full((2, big), 0xAB, dtype=torch.uint8, device=ctx.torch_device)
    ln = torch.full((2,), 7, dtype=torch.int32, device=ctx.torch_device)
    lib = ctx.lib
    st = lib.mocap_encode_jpeg_dev(ctx.h, ctypes.c_void_p(d.data_ptr()), 2, 1, 64, 64, 95, ctypes.c_void_p(out.data_ptr()),
                                   big, ctypes.c_void_p(ln.data_ptr()))
    torch.cuda.synchronize()
    assert st == 0 and int(ln[0]) == len(want[0]) and int(ln[1]) == len(want[1])
    out.fill_(0xAB)
    ln.fill_(7)
    st = lib.mocap_encode_jpeg_dev(ctx.h, ctypes.c_void_p(d.data_ptr()), 2, 1, 64, 64, 95, ctypes.c_void_p(out.data_ptr()),
                                   stride, ctypes.c_void_p(ln.data_ptr()))
    torch.cuda.synchronize()
    o = out.cpu().numpy().reshape(-1)
    assert st == 0 and int(ln[0]) == -1 and int(ln[1]) == len(want[1])
    assert (o[:stride] == 0xAB).all(), "the image that did not fit wrote into its row"
    assert np.array_equal(o[stride:stride + len(want[1])], want[1]) and (o[stride + len(want[1]):] == 0xAB).all()
    for q, tiles, tw, th, n in ((0, 1, 64, 64, 1), (101, 1, 64, 64, 1), (95, 0, 64, 64, 1), (95, 1, 0, 64, 1), (95, 1, 64, 0, 1),
                                (95, 1, 64, 64, -1), (95, 1, 65501, 1, 1), (95, 2, 40000, 1, 1)):
        n0 = ctx.launch_count()
        st = lib.mocap_encode_jpeg_dev(ctx.h, ctypes.c_void_p(d.data_ptr()), n, tiles, tw, th, q, ctypes.c_void_p(out.data_ptr()),
                                       stride, ctypes.c_void_p(ln.data_ptr()))
        assert st == -1 and ctx.launch_count() == n0, (q, tiles, tw, th, n)
    assert lib.mocap_jpeg_bound(0, 5) == 0 and lib.mocap_jpeg_bound(16, 16) > 623
    with pytest.raises(pkg.MocapError):
        ctx.encode_jpeg(d, quality=0)
    # the host entry
    g = load_golden()
    scene = golden_scene(g)
    c = api.MocapContext(4, 320, 320, **api.MIRROR_LIMITS)
    c.set_preprocess(IN_W, IN_H, scene["rotations"], [K] * 4, [DIST] * 4)
    raw = render_read(scene, 0)[None]
    ok = c.live_host(raw, CAPTURE, jpeg=True, quality=90)
    n = int(ok["jpeg_len"][0])
    with pytest.raises(pkg.MocapError, match="does not fit"):
        c.live_host(raw, CAPTURE, jpeg=True, quality=90, jpeg_stride=n - 1)
    exact = c.live_host(raw, CAPTURE, jpeg=True, quality=90, jpeg_stride=n)
    assert np.array_equal(exact["jpeg"][0], ok["jpeg"][0, :n])
    for q in (0, 101):
        n0 = c.launch_count()
        with pytest.raises(pkg.MocapError) as e:
            c.live_host(raw, CAPTURE, jpeg=True, quality=q)
        assert e.value.status == -1 and c.launch_count() == n0


def test_launches_per_read():
    """mocap_live_jpeg_host adds the encoder's four launches to the read's chain."""
    g = load_golden()
    scene = golden_scene(g)
    c = api.MocapContext(4, 320, 320, **api.MIRROR_LIMITS)
    c.set_preprocess(IN_W, IN_H, scene["rotations"], [K] * 4, [DIST] * 4)
    raw = render_read(scene, 0)[None]
    c.live_host(raw, CAPTURE, jpeg=True)
    n0 = c.launch_count()
    c.live_host(raw, CAPTURE)
    n1 = c.launch_count()
    c.live_host(raw, CAPTURE, jpeg=True)
    assert (n1 - n0) + 4 == c.launch_count() - n1

"""The JPEG encoder's CPU tier: the numpy model (tests/jpeg_util.py) against cv2.imencode byte for byte and against the
recorded bytes of tests/golden/jpeg_cv2.npz; the host build of csrc/jpeg.cuh (the kernels' step code) against the model
stage by stage -- colour conversion and downsampling, the DCT and quantisation, bit counts, packing and stuffing on
random and extreme coefficient blocks -- and whole; install_into(stream=True) on stand-ins."""
import ctypes
import importlib
import os
import subprocess

import cv2
import numpy as np
import pytest

from tests import jpeg_util as J
from tests.live_util import ROOT

api = importlib.import_module("low-cost-mocap_b200.api")
pkg = importlib.import_module("low-cost-mocap_b200")
P, I, U64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("jpeg")), "libjpeg_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-ffp-contract=off", "-std=c++17", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "jpeg_host.cpp")])
    lib = ctypes.CDLL(out)
    for name, res, args in (("hc_tables_size", I, []), ("hc_header", None, [I, I, I, P]), ("hc_bound", U64, [I, I]),
                            ("hc_ycc", None, [I, P, P]), ("hc_samples", None, [P, I, I, I, P]), ("hc_fdct", None, [I, P, P]),
                            ("hc_quantize", None, [I, I, P, P, P]), ("hc_block_bits", None, [I, P, P, P, P, P]),
                            ("hc_pack", None, [I, P, P, P, P, U64, P]), ("hc_stuff", U64, [P, U64, I, P]),
                            ("hc_encode", ctypes.c_int64, [P, I, I, I, I, P, U64])):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def _p(a):
    return a.ctypes.data_as(P)


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


# ---------------------------------------------------------------------------------------------- the model and cv2
@pytest.mark.parametrize("content", J.CONTENTS)
@pytest.mark.parametrize("h,w", J.SIZES)
def test_model_equals_cv2(h, w, content):
    for q in J.QUALITIES:
        img = J.make_image(content, h, w)
        assert np.array_equal(J.encode(img, q), J.cv2_encode(img, q)), q


def test_model_equals_the_golden_bytes():
    """cv2 4.13 / libjpeg-turbo 3.1.2's bytes as recorded: a cv2 here that encodes otherwise cannot move the target."""
    for name, img, q, want in J.load_golden():
        assert np.array_equal(J.encode(img, q), want), name


def test_reciprocal_quantisation_is_rounded_division():
    """libjpeg-turbo's reciprocal multiply ((|x| + corr) * recip) >> shift equals |x| / d rounded half up for every
    divisor 8 * table (8..2040, every quality) and every |x| < 2^14 (the islow output is within +-8192)."""
    d = np.arange(8, 2041, 8)[:, None]
    x = np.arange(0, 1 << 14)[None, :]
    fq, c, r = J.reciprocal(d)
    assert np.array_equal(((x + c) * fq) >> r, (x + d // 2) // d)


def test_header_is_cv2s():
    for w, h, q in ((1, 1, 1), (1280, 320, 95), (65500, 7, 100)):
        img = np.zeros((h, w, 3), np.uint8) if w * h < 10 ** 6 else None
        want = J.header(w, h, q)
        assert len(want) == 623
        if img is not None:
            assert bytes(J.cv2_encode(img, q)[:623]) == want


# ---------------------------------------------------------------------------------------------- the host build, by stage
def test_tables_and_header(lib):
    for q in (1, 10, 50, 75, 95, 100):
        h = np.zeros(623, np.uint8)
        lib.hc_header(1280, 320, q, _p(h))
        assert bytes(h) == J.header(1280, 320, q), q
    assert lib.hc_bound(16, 16) == 623 + 2 * (9960 // 8) + 2


def test_colour_conversion(lib):
    rng = np.random.default_rng(0)
    px = np.concatenate([rng.integers(0, 256, (20000, 3)), np.array(np.meshgrid([0, 1, 127, 128, 254, 255], [0, 255], [0, 128, 255])).reshape(3, -1).T])
    px = np.ascontiguousarray(px, np.uint8)
    out = np.zeros((len(px), 3), np.int32)
    lib.hc_ycc(len(px), _p(px), _p(out))
    assert np.array_equal(out, np.stack(J.rgb_ycc(px), -1))


@pytest.mark.parametrize("h,w,tiles", [(1, 1, 1), (8, 8, 1), (17, 23, 1), (33, 47, 1), (15, 9, 3), (37, 29, 4), (240, 320, 1), (16, 16, 8)])
def test_samples_colour_and_downsampling(lib, h, w, tiles):
    """The samples each block reads: colour conversion, h2v2 with its alternating bias, and the edge padding (right
    edge, odd rows, the last downsampled row), on random pixels, tiled input included."""
    rng = np.random.default_rng(h * w + tiles)
    frames = rng.integers(0, 256, (tiles, h, w, 3), dtype=np.uint8)
    img = np.hstack(list(frames))
    W = tiles * w
    mh, mw = -(-h // 16), -(-W // 16)
    got = np.zeros((mh * mw, 6, 64), np.int32)
    lib.hc_samples(_p(frames), tiles, w, h, _p(got))
    Y, Cb, Cr = J.planes(img)
    got = got.reshape(mh, mw, 6, 8, 8)
    hb, wb = -(-h // 8), -(-W // 8)
    yb = J.blocks_of(Y)
    for b, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        want = yb[dy::2, dx::2]
        real = (np.arange(mh)[:, None] * 2 + dy < hb) & (np.arange(mw)[None, :] * 2 + dx < wb)
        assert np.array_equal(got[:, :, b][real], want[real]), b
    assert np.array_equal(got[:, :, 4], J.blocks_of(Cb))
    assert np.array_equal(got[:, :, 5], J.blocks_of(Cr))


def _sample_blocks(rng, n):
    blocks = [rng.integers(0, 256, (n, 64)), np.zeros((1, 64)), np.full((1, 64), 255),
              (np.indices((8, 8)).sum(0) % 2 * 255).reshape(1, 64), ((np.indices((8, 8))[1] < 4) * 255).reshape(1, 64),
              ((np.indices((8, 8))[0] < 4) * 255).reshape(1, 64), np.tile([0, 255], 32).reshape(1, 64)]
    return _i32(np.concatenate(blocks))


def test_fdct_and_quantisation(lib):
    rng = np.random.default_rng(1)
    s = _sample_blocks(rng, 5000)
    d = np.zeros_like(s)
    lib.hc_fdct(len(s), _p(s), _p(d))
    want = J.fdct_islow(s.reshape(-1, 8, 8)).reshape(-1, 64)
    assert np.array_equal(d, want)
    assert np.abs(d).max() >= 8000                   # the extremes reach the DC's range
    tabs = _i32(rng.integers(0, 2, len(d)))
    for q in (1, 10, 50, 75, 95, 100):
        zz = np.zeros(d.shape, np.int16)
        lib.hc_quantize(len(d), q, _p(tabs), _p(d), _p(zz))
        qt = J.quant_tables(q)
        want = np.where(tabs[:, None] == 0, J.quantize(d, qt[0]), J.quantize(d, qt[1]))[:, J.ZIGZAG]
        assert np.array_equal(zz, want), q


def _coef_blocks(rng):
    """zigzag blocks with their DC differences and tables: random, and the extremes the entropy coder must get right"""
    n = 3000
    zz = np.zeros((n, 64), np.int64)
    dens = rng.uniform(0, 1, n)[:, None]
    mag = rng.integers(1, 1 << rng.integers(1, 11, (n, 1)), (n, 64))
    zz[:] = np.where(rng.uniform(size=(n, 64)) < dens ** 3, mag * rng.choice([-1, 1], (n, 64)), 0)
    zz = np.clip(zz, -1023, 1023)
    diffs = rng.integers(-2047, 2048, n) >> rng.integers(0, 11, n)
    ext = []
    for t in (0, 1):
        for d in (2047, -2047, 1024, -1024, 1, -1, 0):
            ext.append((np.zeros(64, np.int64), d, t))
        for v in (1023, -1023, 512, -512, 1, -1):
            for k in (1, 16, 17, 31, 32, 33, 48, 49, 62, 63):
                b = np.zeros(64, np.int64)
                b[k] = v
                ext.append((b, 0, t))
        b = np.zeros(64, np.int64); b[63] = 5; b[1] = 1
        ext.append((b, 3, t))                                        # non-zero 63: no EOB
        b = np.full(64, 1023, np.int64)
        ext.append((b, 2047, t))                                     # the longest block
        b = np.full(64, -1023, np.int64)
        ext.append((b, -2047, t))
        b = np.zeros(64, np.int64); b[16:64:16] = 1023
        ext.append((b, -2047, t))                                    # runs of 15 then ZRL-free
        b = np.zeros(64, np.int64); b[[17, 34, 51]] = [1023, -1023, 1023]
        ext.append((b, 0, t))                                        # runs of exactly 16 zeros: ZRL + (0, size)
    zz = np.concatenate([zz, np.stack([e[0] for e in ext])])
    diffs = np.concatenate([diffs, [e[1] for e in ext]])
    tabs = np.concatenate([rng.integers(0, 2, n), [e[2] for e in ext]])
    return np.ascontiguousarray(zz, np.int16), _i32(diffs), _i32(tabs)


def test_bits_packing_and_stuffing(lib):
    """Per-block DC and AC bit counts, packing at any bit offset (each block its own writer, the words shared with the
    neighbours OR-ed, the tail padded with 1-bits) and stuffing in chunks, against the model's token stream."""
    rng = np.random.default_rng(2)
    zz, diffs, tabs = _coef_blocks(rng)
    n = len(zz)
    vals, lens, blk = J.block_tokens(zz, diffs, tabs)
    s = J.nbits(diffs)
    want_dc = np.where(tabs == 0, J.DC_CODES[0][1][s], J.DC_CODES[1][1][s]) + s
    want_all = np.bincount(blk, weights=lens, minlength=n).astype(np.int64)
    dc, ac = np.zeros(n, np.int32), np.zeros(n, np.int32)
    lib.hc_block_bits(n, _p(zz), _p(diffs), _p(tabs), _p(dc), _p(ac))
    assert np.array_equal(dc, want_dc) and np.array_equal(dc + ac, want_all)
    assert 1600 < (dc + ac).max() <= 1660                            # JPEG_BLOCK_MAX_BITS bounds the longest block
    offs = np.ascontiguousarray(np.cumsum(want_all) - want_all, np.uint64)
    total = int(want_all.sum())
    words = np.zeros(total // 32 + 2, np.uint32)
    lib.hc_pack(n, _p(zz), _p(diffs), _p(tabs), _p(offs), total, _p(words))
    want = J.pack(vals, lens)
    got = words.byteswap().view(np.uint8)[:len(want)]
    assert np.array_equal(got, want)
    assert (want == 0xFF).sum() > 100                                # the stream holds many bytes to stuff
    for chunk in (1, 3, 16, 4096):
        out = np.zeros(2 * len(want) + 16, np.uint8)
        m = lib.hc_stuff(_p(words), len(want), chunk, _p(out))
        assert np.array_equal(out[:m], J.stuff(want)), chunk


def test_stuffing_of_a_stream_of_ones(lib):
    """0xFF bytes back to back, at the start, the end and across every chunk boundary."""
    data = np.full(100, 0xFF, np.uint8)
    data[[0, 50, 51]] = [0xFF, 0x12, 0x00]
    words = np.frombuffer(np.concatenate([data, np.zeros(4, np.uint8)]).tobytes(), np.uint32).byteswap().copy()
    for chunk in (1, 2, 7, 16):
        out = np.zeros(256, np.uint8)
        m = lib.hc_stuff(_p(words), 100, chunk, _p(out))
        assert np.array_equal(out[:m], J.stuff(data)), chunk


@pytest.mark.parametrize("h,w", J.SIZES[:7])
def test_host_build_equals_cv2(lib, h, w):
    """The whole encoder through the kernels' step code, walked as the kernels walk it (the pack step MCUs in reverse)."""
    for content in J.CONTENTS:
        for q in (1, 50, 95, 100):
            img = J.make_image(content, h, w, seed=3)
            cap = lib.hc_bound(w, h)
            out = np.zeros(cap, np.uint8)
            n = lib.hc_encode(_p(img), 1, w, h, q, _p(out), cap)
            want = J.cv2_encode(img, q)
            assert n == len(want) and np.array_equal(out[:n], want), (content, q)
            assert lib.hc_encode(_p(img), 1, w, h, q, _p(out), len(want) - 1) == -1


def test_host_build_tiles_equal_hstack(lib):
    for tiles, th, tw in ((2, 37, 29), (4, 320, 320), (8, 9, 5)):
        frames = np.stack([J.make_image("dots", th, tw, seed=s) for s in range(tiles)])
        cap = lib.hc_bound(tiles * tw, th)
        out = np.zeros(cap, np.uint8)
        n = lib.hc_encode(_p(frames), tiles, tw, th, 95, _p(out), cap)
        assert np.array_equal(out[:n], J.cv2_encode(np.hstack(list(frames)), 95)), tiles


# ---------------------------------------------------------------------------------------------- install_into(stream=True)
def _modules(monkeypatch):
    from tests.test_host_cpu import _reference_like_modules
    api_, helpers, index = _reference_like_modules(np.array([[600.0, 0, 320], [0, 600, 240], [0, 0, 1]]))
    index.cv = cv2
    monkeypatch.setattr(api.MocapSession, "_default", None)
    cls = type(helpers.Cameras.instance())
    monkeypatch.setattr(cls, "_camera_read", lambda self: "cpu", raising=False)
    monkeypatch.setattr(cls, "get_frames", lambda self: "cpu frames", raising=False)
    return helpers, index, cls


def test_stream_needs_live(monkeypatch):
    helpers, index, cls = _modules(monkeypatch)
    with pytest.raises(ValueError, match="live=True"):
        pkg.install_into(helpers, index, stream=True)
    assert index.cv is cv2 and helpers.Cameras.instance().get_frames() == "cpu frames"


def test_default_leaves_cv_and_get_frames(monkeypatch):
    helpers, index, cls = _modules(monkeypatch)
    pkg.install_into(helpers, index, live=True)
    assert index.cv is cv2 and helpers.Cameras.instance().get_frames() == "cpu frames"


def test_install_into_stream_rebinds_get_frames_and_cv(monkeypatch):
    """get_frames is replaced on the class behind the Singleton wrapper; index.cv becomes a proxy whose attributes are
    cv2's own objects and whose imencode is cv2's for anything but a StreamFrames; without a GPU the new get_frames
    fails loudly."""
    import torch
    helpers, index, cls = _modules(monkeypatch)
    pkg.install_into(helpers, index, live=True, stream=True)
    assert isinstance(index.cv, api.StreamCv) and cls.get_frames.__mocap_b200__
    for name in ("findFundamentalMat", "recoverPose", "Rodrigues", "projectPoints", "IMWRITE_JPEG_QUALITY", "COLOR_RGB2GRAY",
                 "imdecode"):
        assert getattr(index.cv, name) is getattr(cv2, name), name
    if hasattr(cv2, "sfm"):
        assert index.cv.sfm is cv2.sfm
    pkg.install_into(helpers, index, live=True, stream=True)
    assert index.cv._cv is cv2                                       # installed twice: one proxy, not a proxy of a proxy
    img = J.make_image("dots", 40, 56)
    for params in ((), [cv2.IMWRITE_JPEG_QUALITY, 80]):
        ok, buf = index.cv.imencode(".jpg", img, *([params] if params else []))
        assert ok and np.array_equal(buf, cv2.imencode(".jpg", img, *([params] if params else []))[1])
    if not torch.cuda.is_available():
        cams = helpers.Cameras.instance()
        cams.cameras = type("Drv", (), {"read": lambda s: ([np.zeros((240, 320, 3), np.uint8)] * 4, None)})()
        cams.num_cameras = 4
        cams.is_capturing_points = cams.is_triangulating_points = cams.is_locating_objects = False
        with pytest.raises(pkg.MocapError):
            cams.get_frames()


def test_stream_cv_returns_the_carried_bytes_only_when_they_answer_the_call():
    """The proxy hands back the carried bytes for '.jpg' / '.jpeg' with no params or only the quality they were made
    at, as (True, uint8 (N,)); for another quality, another format, other params or a plain array it calls cv2."""
    img = J.make_image("frames", 32, 48)
    carried = np.arange(10, dtype=np.uint8)
    f = api.stream_frames([img[:, :24], img[:, 24:]], carried, 95)
    assert isinstance(f, api.StreamFrames) and np.array_equal(np.asarray(f), img) and not f.flags.writeable
    cv = api.StreamCv(cv2)
    for ext, params in ((".jpg", None), (".JPG", None), (".jpeg", [cv2.IMWRITE_JPEG_QUALITY, 95]), (".jpg", (cv2.IMWRITE_JPEG_QUALITY, 95))):
        ok, buf = cv.imencode(ext, f) if params is None else cv.imencode(ext, f, params)
        assert ok and buf.dtype == np.uint8 and np.array_equal(buf, carried), (ext, params)
        buf[0] = 99
        assert f.jpeg[0] == 0                                        # each call gets its own copy
    for ext, params in ((".jpg", [cv2.IMWRITE_JPEG_QUALITY, 90]), (".png", None),
                        (".jpg", [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_PROGRESSIVE, 1]),
                        (".jpg", [cv2.IMWRITE_JPEG_OPTIMIZE, 1])):
        ok, buf = cv.imencode(ext, f) if params is None else cv.imencode(ext, f, params)
        want = cv2.imencode(ext, img) if params is None else cv2.imencode(ext, img, params)
        assert ok and np.array_equal(buf, want[1]), (ext, params)
    f90 = api.stream_frames([img], carried, 90)
    assert np.array_equal(cv.imencode(".jpg", f90)[1], cv2.imencode(".jpg", img)[1])     # no params: cv2's 95
    assert np.array_equal(cv.imencode(".jpg", f90, [cv2.IMWRITE_JPEG_QUALITY, 90])[1], carried)
    assert np.array_equal(cv.imencode(".jpg", f[:, :10])[1], cv2.imencode(".jpg", np.ascontiguousarray(img[:, :10]))[1])
    assert np.array_equal(cv.imencode(".jpg", np.array(f))[1], cv2.imencode(".jpg", img)[1])

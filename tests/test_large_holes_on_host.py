"""The whole-image window of S1's RETR_TREE slow path (mocap_set_large_holes), as device code run on the host: the
full-size reduction of csrc/blob_device.cuh through tests/hostcheck/simt_emu.h with the window set
(tests/hostcheck/blob_large_holes_host.cpp), held to cv.findContours(RETR_TREE) + cv.moments exactly -- count, centres,
order, A2 / SX6 / SY6 of every contour, the pixel count of every hole region -- on holed blobs wider or taller than
62 px: rings and frames up to the whole image, shapes across the border, a spiral, 16 and 40 nested frames, blobs and
holed blobs inside large holes, 64-hole bands, and both windows in one image."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import hostbuild
from tests.hostbuild import HC, ROOT, ptr
from tests.large_holes_util import large_holes_fuzz, nested_frames, spiral, wide_porous
from tests.util import retr_tree_blobs, set_pixel_blobs

pytestmark = pytest.mark.timeout(600)

F_BLOBS, F_HOLES = 2, 32


@pytest.fixture(scope="module")
def large_emu():
    lib = hostbuild.load("blob_large_holes")

    def detect(img, large=1, max_blobs=64, E=4096, seed=1):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        H, W = img.shape
        xy = np.zeros((max_blobs, 2), np.int32); n = np.zeros(1, np.int32)
        mom = np.zeros((max_blobs, 4), np.int64); fl = np.zeros(1, np.int32)
        rc = lib.hc_blob_detect_large(ptr(img), W, H, 51, max_blobs, E, large, seed, ptr(xy), ptr(n), ptr(mom), ptr(fl))
        assert rc >= 0, rc
        k = int(n[0])
        return [tuple(int(v) for v in mom[i]) + tuple(int(v) for v in xy[i]) for i in range(k)], int(fl[0])
    return detect


def named_images():
    """(name, image) of holed blobs the 64 x 64 window does not take; 160 x 120 unless said otherwise."""
    import cv2
    H, W = 120, 160

    def new(h=H, w=W):
        return np.zeros((h, w), np.uint8)
    out = []
    for side in (63, 64, 100, 159):
        img = new(); cv2.rectangle(img, (0, 10), (side - 1, 60), 255, 1); img[11:14, 1:6] = 255      # lopsided frame
        out.append((f"frame{side}", img))
    img = new(); cv2.circle(img, (80, 60), 45, 255, 2); out.append(("ring90", img))
    img = new(); cv2.rectangle(img, (20, 2), (60, 117), 255, 2); out.append(("tall116", img))
    img = new(); cv2.rectangle(img, (0, 0), (W - 1, H - 1), 255, 1); cv2.circle(img, (80, 60), 7, 255, 2)
    img[100:104, 120:130] = 255; out.append(("around_image", img))
    img = new(); cv2.rectangle(img, (-2, 10), (100, 80), 255, 5); cv2.circle(img, (130, 95), 30, 255, 16)   # walls cut by
    out.append(("across_borders", img))                                                                    # three borders
    img = new(); cv2.ellipse(img, (78, 60), (68, 20), 15.0, 0, 360, 255, 1); out.append(("ellipse", img))
    img = new(); spiral(img, 2, 2, 157, 117); out.append(("spiral", img))
    img = new(); nested_frames(img, 10, 10, 16, gap=3); out.append(("nested16", img))
    img = new(); nested_frames(img, 22, 2, 28, gap=2); out.append(("nested28", img))
    img = new(176, 208); nested_frames(img, 20, 5, 40, gap=2); out.append(("nested40", img))
    img = new(); cv2.circle(img, (80, 60), 55, 255, 2); cv2.circle(img, (80, 60), 35, 255, 3)       # a large holed blob in
    cv2.circle(img, (80, 60), 4, 255, -1); cv2.circle(img, (60, 40), 2, 255, -1)                  # another's hole, blobs in both
    cv2.circle(img, (20, 20), 6, 255, 1); out.append(("holed_in_hole", img))
    img = new(); wide_porous(img, 30, 10, 64); out.append(("porous64", img))
    img = new(); wide_porous(img, 30, 10, 40); cv2.circle(img, (80, 90), 10, 255, 1)            # both windows in one image
    wide_porous(img, 100, 20, 23, w=47); out.append(("both_windows", img))
    return out


@pytest.mark.parametrize("name", [n for n, _ in named_images()])
def test_whole_image_window_equals_cv2(large_emu, name):
    """Exact against cv2, 56 contours nested 56 deep included (28 frames: the emission walk's stack once held 34).  40
    nested frames (80 contours, 80 deep) need some 6500 runs, more than the 4096 the device allows per image (there
    the image gets MOCAP_F_SEGMENTS); the same code is driven past that capacity here (E = 8192) to reach that depth."""
    img = dict(named_images())[name]
    E = 8192 if name == "nested40" else 4096
    items, _, side, holes = retr_tree_blobs(img > 51)
    assert side > 62 and holes <= 64                       # the 64 x 64 window cannot take it ...
    got, fl = large_emu(img, max_blobs=128, E=E)
    assert fl == (F_BLOBS if len(items) > 128 else 0) and got == items[:128], (name, fl, got[:3], items[:3])
    off, fl_off = large_emu(img, large=0, max_blobs=128, E=E)
    assert fl_off & F_HOLES and off == set_pixel_blobs(img > 51)[:128]       # ... and without the window it says so


def test_named_images_are_what_they_claim():
    imgs = dict(named_images())
    assert retr_tree_blobs(imgs["nested40"] > 0)[3] == 40 and len(retr_tree_blobs(imgs["nested40"] > 0)[0]) == 80
    assert retr_tree_blobs(imgs["nested16"] > 0)[3] == 16 and retr_tree_blobs(imgs["nested28"] > 0)[3] == 28
    assert retr_tree_blobs(imgs["porous64"] > 0)[3] == 64
    from scipy import ndimage
    sp = imgs["spiral"] > 0
    assert ndimage.label(sp, np.ones((3, 3)))[1] == 1 and retr_tree_blobs(sp)[3] == 1
    assert ndimage.binary_fill_holes(sp).sum() - sp.sum() > 4000              # one corridor across the whole spiral


def test_more_than_64_holes_keeps_the_flag(large_emu):
    """With the window on, only a 65th hole leaves MOCAP_F_HOLES; the image then reports the set-pixel polygon of every
    blob, also of the large holed blobs filled before the cap was met."""
    import cv2
    img = np.zeros((120, 160), np.uint8)
    wide_porous(img, 2, 10, 64)                             # a band of 64 holes, filled first (its first pixel comes first)
    cv2.circle(img, (80, 70), 45, 255, 2)                   # then a 92-px ring: its hole is the 65th
    got, fl = large_emu(img)
    assert fl == F_HOLES and got == set_pixel_blobs(img > 0)
    img = np.zeros((120, 160), np.uint8)
    wide_porous(img, 30, 10, 65)
    got, fl = large_emu(img)
    assert fl == F_HOLES and got == set_pixel_blobs(img > 0)


def test_fuzz_vs_cv2_and_the_window_changes_nothing_it_need_not(large_emu):
    """Random frames of holed blobs 40-400 px (cut by the border) beside small ones: with the window equal to cv2; an
    image the 64 x 64 window already takes gives the same bits with and without it."""
    rng = np.random.default_rng(5)
    frames, refs = large_holes_fuzz(rng, 24, 120, 160)
    large = small = 0
    for i, (img, (items, kept, side)) in enumerate(zip(frames, refs)):
        got, fl = large_emu(img, seed=i)
        assert fl == 0 and got == items, (i, fl)
        if side > 62:
            large += 1
        else:
            small += 1
            assert large_emu(img, large=0, seed=i) == (got, fl)
    assert large >= 12


def test_whole_image_window_has_no_data_races(tmp_path):
    """ThreadSanitizer over the emulated CTA on large-window images (the spiral, nested frames, a holed blob in a large
    hole, a 65-hole band): the band flood, the CTA-wide minimum and sums and the hole records are race-free.  The
    union-find races by design and is suppressed, as in test_device_code_on_host.py; so would the 64 x 64 window's
    one-warp flood (it reads rows other lanes are growing), which is why no holed blob here fits that window."""
    env = hostbuild.tsan_env(tmp_path, ["race:uf_find", "race:uf_unite", "race:atomicMin"])
    lib = hostbuild.build("blob_large_holes", tsan=True)
    import cv2
    imgs = []
    img = np.zeros((64, 96), np.uint8); spiral(img, 1, 1, 94, 62); imgs.append(img)
    img = np.zeros((80, 96), np.uint8)
    for k in range(4):                                                          # four nested frames, 75 .. 63 px
        cv2.rectangle(img, (10 + 2 * k, 4 + 2 * k), (84 - 2 * k, 78 - 2 * k), 255, 1)
    imgs.append(img)
    img = np.zeros((96, 160), np.uint8); cv2.circle(img, (80, 48), 45, 255, 2); cv2.circle(img, (80, 48), 33, 255, 2)
    cv2.circle(img, (80, 48), 2, 255, -1); imgs.append(img)                     # every holed blob takes the large window
    img = np.zeros((64, 160), np.uint8); wide_porous(img, 20, 10, 65); imgs.append(img)
    cases = {}
    for k, img in enumerate(imgs):
        want, flags = (set_pixel_blobs(img > 0), F_HOLES) if k == 3 else (retr_tree_blobs(img > 0)[0], 0)
        cases.update({f"img{k}": img, f"want{k}": np.array(want, np.int64).reshape(-1, 6), f"flags{k}": flags})
    np.savez(tmp_path / "cases.npz", **cases)
    r = subprocess.run([shutil.which("python") or "python", os.path.join(HC, "tsan_large_holes_run.py"), ROOT, lib, str(tmp_path / "cases.npz")],
                       capture_output=True, text=True, env=env, timeout=560)
    out = r.stdout + r.stderr
    assert out.count("LARGE True") == 4, out[-2000:]
    assert "WARNING: ThreadSanitizer" not in out, out[:4000]

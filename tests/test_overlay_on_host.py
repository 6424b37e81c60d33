"""The detection overlay's CPU tier: the host build of csrc/overlay.cuh (the drawing code of the overlay kernels) against
cv2 -- the contour stencil, the plus marks, the '(x, y)' labels, the line rasteriser -- and the whole of _find_dot's
drawing on random frames and on the live session's frames."""
import cv2
import numpy as np
import pytest

from tests import hostbuild
from tests.hostbuild import ptr
from tests.overlay_util import drawline_of, find_dot_drawn, random_scene

MARK = (100, 255, 100)


@pytest.fixture(scope="module")
def lib():
    return hostbuild.load("overlay")


def _overlay(lib, img, pts):
    """The host build's overlay of one undrawn frame with its blob list."""
    out = np.ascontiguousarray(img.copy())
    H, W = img.shape[:2]
    xy = np.array(pts if pts else [[0, 0]], np.int32).reshape(1, -1, 2)
    lib.hc_overlay(ptr(out), 1, W, H, xy.shape[1], ptr(xy), ptr(np.array([len(pts)], np.int32)))
    return out


@pytest.mark.parametrize("kind", ["noise", "blobs", "holes"])
def test_find_dot_drawing_equals_cv2_on_random_frames(lib, kind):
    """Contours of noise of every density, dilated and closed noise (holes, rings, 1-px blobs, blobs on the edge), then
    every blob's label and plus: the host build equals cv2's drawing byte for byte, over frames of 5 to 200 pixels a side."""
    rng = np.random.default_rng({"noise": 1, "blobs": 2, "holes": 3}[kind])
    labels = 0
    for t in range(400):
        H, W = (int(v) for v in (rng.integers(5, 60, 2) if t % 2 else rng.integers(40, 200, 2)))
        img = random_scene(rng, H, W, kind)
        want, pts = find_dot_drawn(img.copy())
        assert np.array_equal(_overlay(lib, img, pts), want), (t, W, H)
        labels += len(pts)
    assert labels > 2000


def test_contour_stencil_alone_on_rings():
    """drawContours of RETR_TREE on rings, nested rings and a frame-filling blob paints the foreground pixels with a
    background or outside 4-neighbour: the claim the contour kernel rests on, pinned on shapes the noise rarely makes."""
    img = np.zeros((120, 160), np.uint8)
    cv2.circle(img, (40, 40), 30, 255, 6)
    cv2.circle(img, (40, 40), 12, 255, 3)
    cv2.circle(img, (40, 40), 2, 255, -1)
    cv2.rectangle(img, (90, 10), (159, 119), 255, -1)
    cv2.rectangle(img, (110, 40), (140, 80), 0, -1)
    cv2.ellipse(img, (60, 95), (40, 12), 20, 0, 360, 255, 1)
    for b in (img, np.full_like(img, 255), np.pad(np.full((10, 10), 255, np.uint8), 1)):
        contours, _ = cv2.findContours(b, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
        drawn = cv2.drawContours(np.zeros_like(b), contours, -1, 255, 1) > 0
        fg = np.pad(b > 0, 1)
        inner = fg[1:-1, 1:-1] & fg[:-2, 1:-1] & fg[2:, 1:-1] & fg[1:-1, :-2] & fg[1:-1, 2:]
        assert np.array_equal(drawn, (b > 0) & ~inner)


def test_plus_at_every_position(lib):
    """cv.circle(img, (x, y), 1, colour, -1) at every pixel of a 9 x 7 frame and one step outside it."""
    for y in range(-1, 8):
        for x in range(-1, 10):
            want = np.zeros((7, 9, 3), np.uint8)
            cv2.circle(want, (x, y), 1, MARK, -1)
            got = np.zeros_like(want)
            lib.hc_plus(ptr(got), 9, 7, x, y)
            assert np.array_equal(got, want), (x, y)


def test_labels_of_every_coordinate_pair_up_to_1023(lib):
    """The label of every centre (x, y) with x, y in 0..1023 whose digits differ from its neighbours' (a dense sample:
    every x with a fixed y, every y with a fixed x, and random pairs), on a 1024-pixel frame, and at origins that clip on
    every side: the host build equals cv2.putText."""
    S = 1040
    rng = np.random.default_rng(5)
    pairs = [(x, 500) for x in range(1024)] + [(7, y) for y in range(1024)]
    pairs += [tuple(int(v) for v in rng.integers(0, 1024, 2)) for _ in range(600)]
    pairs += [(0, 0), (1023, 1023), (1023, 5), (3, 1023), (1000, 14), (1020, 16), (0, 1039)]
    frame = np.zeros((S, S, 3), np.uint8)
    for x, y in pairs:
        want = np.zeros((S, S, 3), np.uint8)
        cv2.putText(want, f'({x}, {y})', (x, y - 15), cv2.FONT_HERSHEY_SIMPLEX, 0.3, MARK, 1)
        frame[:] = 0
        lib.hc_label(ptr(frame), S, S, x, y)
        y0, y1, x0, x1 = max(0, y - 30), min(S, y + 10), max(0, x - 5), min(S, x + 80)
        assert np.array_equal(frame[y0:y1, x0:x1], want[y0:y1, x0:x1]) and frame.sum() == want.sum(), (x, y)
    # small frames: the labels of centres near every edge clip at the frame's sides; centres off the frame, negative
    # ones included, as the batched entry may be given
    for W, H in ((24, 20), (64, 16), (100, 40)):
        for y in range(-2, H + 16):
            for x in range(-40, W, 3):
                want = np.zeros((H, W, 3), np.uint8)
                cv2.putText(want, f'({x}, {y})', (x, y - 15), cv2.FONT_HERSHEY_SIMPLEX, 0.3, MARK, 1)
                got = np.zeros_like(want)
                lib.hc_label(ptr(got), W, H, x, y)
                assert np.array_equal(got, want), (W, H, x, y)


def test_lines_equal_cv2(lib):
    """cv.line with thickness 1 and LINE_8 between integer end points -- inside, crossing the frame, far outside as
    the reference's drawlines can make them, near-vertical and near-horizontal -- and between 16.16 fixed-point end
    points (putText's strokes, cv.line(shift=16))."""
    rng = np.random.default_rng(9)
    W, H = 48, 40
    for t in range(3000):
        if t % 4 == 0:
            p = rng.integers(-100000, 100000, 4)
        elif t % 4 == 1:
            p = rng.integers(-60, 110, 4)
        elif t % 4 == 2:      # near-vertical / near-horizontal
            a, b = rng.integers(-20, 70, 2)
            p = np.array([a, -30, a + rng.integers(-2, 3), 80]) if t % 8 == 2 else np.array([-30, b, 90, b + rng.integers(-2, 3)])
        else:
            p = rng.integers(0, 48, 4)
        want = np.zeros((H, W, 3), np.uint8)
        cv2.line(want, (int(p[0]), int(p[1])), (int(p[2]), int(p[3])), MARK, 1, cv2.LINE_8)
        got = np.zeros_like(want)
        lib.hc_line(ptr(got), W, H, *[int(v) for v in p], 0)
        assert np.array_equal(got, want), p
        q = rng.integers(-8 << 16, 56 << 16, 4)
        want = np.zeros((H, W, 3), np.uint8)
        cv2.line(want, (int(q[0]), int(q[1])), (int(q[2]), int(q[3])), MARK, 1, cv2.LINE_8, 16)
        got = np.zeros_like(want)
        lib.hc_line(ptr(got), W, H, *[int(v) for v in q], 1)
        assert np.array_equal(got, want), q


def test_live_session_frames(lib):
    """The processed frames of the golden live session (RefPort preprocessing of its rendered reads), drawn."""
    from oracle.ref_port import RefPort
    from tests.live_util import DIST, K, golden_scene, load_golden, render_read
    g = load_golden()
    scene = golden_scene(g)
    port = RefPort([K] * 4)
    n = 0
    for k in range(0, len(g["mode"]), 7):
        raw = render_read(scene, k, bool(g["dark"][k]))
        for c in range(4):
            frame = port.preprocess(raw[c], c, DIST, scene["rotations"][c])
            want, pts = find_dot_drawn(frame.copy())
            assert np.array_equal(_overlay(lib, frame, pts), want), (k, c)
            n += len(pts)
    assert n > 100


def test_palette_is_numpys_legacy_randint(lib):
    """np.random.RandomState(seed).randint(0, 255, (L, 3)), and it is what L calls of np.random.randint(0, 255, 3) give
    after np.random.seed(seed), as the reference draws its line colours."""
    for seed in (0, 11, 2 ** 32 - 1):
        got = np.zeros((5000, 3), np.uint8)
        lib.hc_palette(seed, 5000, ptr(got))
        assert np.array_equal(got, np.random.RandomState(seed).randint(0, 255, (5000, 3)))
        state = np.random.get_state()
        try:
            np.random.seed(seed)
            assert np.array_equal(got[:300], np.array([np.random.randint(0, 255, 3) for _ in range(300)]))
        finally:
            np.random.set_state(state)


def test_epipolar_line_end_points_and_skips(lib):
    """drawlines' float32 end points of random lines -- ordinary, near-horizontal (b near 0), vertical (b == 0, inf and
    NaN), reaching past 32 bits -- equal the reference's arithmetic, and the lines skipped are exactly those where the
    reference's int() or cv.line raises; the drawn pixels (1 and 32 lanes) equal cv.line's."""
    rng = np.random.default_rng(21)
    W = H = 48
    skipped = drawn = 0
    for t in range(4000):
        ang = rng.uniform(0, 2 * np.pi)
        a, b = np.cos(ang), np.sin(ang)
        if t % 5 == 1:
            b = rng.choice([0.0, -0.0, 1e-30, -3e-12, 1e-8, 4e-5])
        c = rng.uniform(-1, 1) * 10.0 ** rng.integers(0, 8) if t % 7 else 0.0
        r = np.array([a, b, c], np.float32)
        y0, y1 = np.zeros(1, np.int64), np.zeros(1, np.int64)
        ok = lib.hc_epiline_ends(float(r[0]), float(r[1]), float(r[2]), W, ptr(y0), ptr(y1))
        want = np.zeros((H, W, 3), np.uint8)
        ref_ok = drawline_of(want, r, (3, 200, 17))
        assert bool(ok) == ref_ok, r
        if not ok:
            skipped += 1
            continue
        drawn += 1
        with np.errstate(all="ignore"):
            assert (y0[0], y1[0]) == (int(-r[2] / r[1]), int(-(r[2] + r[0] * W) / r[1])), r
        for lanes in (1, 32):
            got = np.zeros_like(want)
            lib.hc_line_lanes(ptr(got), W, H, 0, int(y0[0]), W, int(y1[0]), lanes)
            assert np.array_equal(got.any(2), want.any(2)), (r, lanes)
    assert skipped > 100 and drawn > 2000

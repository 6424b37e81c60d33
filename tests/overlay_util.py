"""Shared by the overlay tests (tests/test_overlay_on_host.py, tests/test_overlay_oracle_pinned.py,
tests/test_gpu_overlay.py) and tools/overlay_time.py: the drawing of the reference's _find_dot (helpers.py:143-163) as
its own cv2 call sequence -- the oracle of the detection overlay -- and random binary scenes for it."""
import cv2
import numpy as np
import scipy.ndimage as nd


def find_dot_drawn(img):
    """helpers.py:143-163 with its drawing: contours, then per contour with m00 != 0 the '(x, y)' label and the filled
    radius-1 circle, into img (H x W x 3 uint8, in place).  Returns (img, points) with points a list of [x, y]."""
    grey = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
    grey = cv2.threshold(grey, 255 * 0.2, 255, cv2.THRESH_BINARY)[1]
    contours, _ = cv2.findContours(grey, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
    img = cv2.drawContours(img, contours, -1, (0, 255, 0), 1)
    pts = []
    for contour in contours:
        m = cv2.moments(contour)
        if m["m00"] != 0:
            x, y = int(m["m10"] / m["m00"]), int(m["m01"] / m["m00"])
            cv2.putText(img, f'({x}, {y})', (x, y - 15), cv2.FONT_HERSHEY_SIMPLEX, 0.3, (100, 255, 100), 1)
            cv2.circle(img, (x, y), 1, (100, 255, 100), -1)
            pts.append([x, y])
    return img, pts


def random_scene(rng, H, W, kind):
    """An H x W x 3 frame whose grey is > 51 exactly on a random binary mask: noise of a random density, dilated
    ('blobs'), closed ('holes': rings and holed blobs), or as drawn ('noise').  The colours are random on both sides of
    the threshold, so the contour stage sees real RGB2GRAY values."""
    density = rng.uniform(0.0005, 0.02) if kind == "blobs" else rng.uniform(0.01, 0.6)
    b = rng.uniform(size=(H, W)) < density
    if kind == "blobs":
        b = nd.binary_dilation(b, iterations=int(rng.integers(1, 5)))
    elif kind == "holes":
        b = nd.binary_erosion(nd.binary_dilation(b, iterations=2))
    img = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
    img[b & (g <= 51)] = rng.integers(120, 256, 3).astype(np.uint8)
    img[~b & (g > 51)] = rng.integers(0, 40, 3).astype(np.uint8)
    return img


def sparse_scene(rng, H, W, n):
    """An H x W x 3 frame of n marker-like shapes on dark noise, few enough for S1's per-image blob list: discs, 1-px
    dots, rings (a blob and a hole contour each) and holed squares, some cut by the frame's edges."""
    img = rng.integers(0, 30, (H, W, 3)).astype(np.uint8)
    for _ in range(n):
        x = int(rng.integers(-3, W + 3)) if rng.uniform() < 0.2 else int(rng.integers(0, W))
        y = int(rng.integers(-3, H + 3)) if rng.uniform() < 0.2 else int(rng.integers(0, H))
        colour = tuple(int(v) for v in rng.integers(90, 256, 3))
        kind = rng.integers(0, 4)
        if kind == 0:
            cv2.circle(img, (x, y), int(rng.integers(1, 7)), colour, -1)
        elif kind == 1:
            img[min(max(y, 0), H - 1), min(max(x, 0), W - 1)] = colour
        elif kind == 2:
            cv2.circle(img, (x, y), int(rng.integers(4, 14)), colour, int(rng.integers(1, 3)))
        else:
            r = int(rng.integers(3, 9))
            cv2.rectangle(img, (x - r, y - r), (x + r, y + r), colour, -1)
            cv2.rectangle(img, (x - r // 3, y - r // 3), (x + r // 3, y + r // 3), (5, 5, 5), -1)
    return img


def drawline_of(img, r, colour):
    """drawlines (helpers.py:497-504) for one float32 line r = (a, b, c) in a given colour -- the reference's own
    arithmetic and cv.line call.  Where the reference raises (int() of inf or NaN, an end point outside cv.line's 32
    bits) nothing is drawn; returns whether the line was drawn."""
    r = np.asarray(r, dtype=np.float32)
    c = img.shape[1]
    with np.errstate(all="ignore"):
        try:
            x0, y0 = map(int, [0, -r[2] / r[1]])
            x1, y1 = map(int, [c, -(r[2] + r[0] * c) / r[1]])
        except (OverflowError, ValueError):
            return False
    if not all(-2 ** 31 <= v < 2 ** 31 for v in (y0, y1)):
        return False
    cv2.line(img, (x0, y0), (x1, y1), tuple(int(v) for v in colour), 1)
    return True


def epilines_drawn(port, frames, image_points, poses, palette, n0):
    """The lines find_point_correspondance_and_object_points draws into frames (helpers.py:357-406, in place): for each
    camera i >= 1, the line of every root that exists before it (RefPort.epipolar_line), in root order, line n of the
    session in palette[n % len(palette)].  The roots follow helpers.py:357,391,402-406.  Returns the session's line count
    after this call."""
    pts = [[list(p) for p in cam if not (p[0] is None and p[1] is None)] for cam in image_points]
    roots = [(0, p) for p in pts[0]]
    n = n0
    for cam in range(1, len(poses)):
        lines = [port.epipolar_line(rc, cam, rp, poses) for rc, rp in roots]
        for line in lines:
            drawline_of(frames[cam], line, palette[n % len(palette)])
            n += 1
        here = np.array(pts[cam])
        unmatched = [list(p) for p in pts[cam]]
        for a, b, c in lines:
            if len(here) == 0:
                continue
            dist = np.abs(a * here[:, 0] + b * here[:, 1] + c) / np.sqrt(a ** 2 + b ** 2)
            near = dist < 5
            cands = here[near][dist[near].argsort()].tolist()
            if cands:
                unmatched = [p for p in unmatched if p != cands[0]]
        roots += [(cam, p) for p in unmatched]
    return n


def palette_of(seed, L=65536):
    return np.random.RandomState(seed).randint(0, 255, (L, 3))

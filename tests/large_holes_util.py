"""Images for the whole-image window of S1's RETR_TREE slow path (mocap_set_large_holes), shared by the CPU and GPU
tests: holed blobs wider or taller than 62 pixels, which the 64 x 64 window does not take."""
import numpy as np

from tests.util import porous_patch


def spiral(img, x0, y0, x1, y1, step=3, v=255):
    """A 1-px frame (x0, y0)-(x1, y1) and a square spiral wall that starts on its left side and winds inwards, walls
    `step` px apart: one blob whose single hole is a corridor along the whole spiral -- the flood's worst case, one
    round per turn."""
    import cv2
    cv2.rectangle(img, (x0, y0), (x1, y1), v, 1)
    pts = [(x0, y0 + step)]
    left, top, right, bottom = x0 + step, y0 + step, x1 - step, y1 - step
    while right - left > step and bottom - top > step:
        pts += [(right, top), (right, bottom), (left, bottom), (left, top + step)]
        left, top, right, bottom = left + step, top + step, right - step, bottom - step
    cv2.polylines(img, [np.array(pts, np.int32)], False, v, 1)


def nested_frames(img, x0, y0, n, gap=2, v=255):
    """n concentric 1-px square frames, `gap` px apart, the outermost at (x0, y0): 2n contours nested 2n deep."""
    import cv2
    side = 2 * gap * n + 1
    for k in range(n):
        cv2.rectangle(img, (x0 + gap * k, y0 + gap * k), (x0 + side - 1 - gap * k, y0 + side - 1 - gap * k), v, 1)


def wide_porous(img, y, x, n_holes, w=135):
    """A 5 x w block with n_holes one-pixel holes (wider than the 64-px window once w > 62)."""
    img[y:y + 5, x:x + w] = porous_patch(n_holes, h=5, w=w)


def large_holes_fuzz(rng, n, H, W, channels=1, lo=40, hi=400):
    """n random frames with holed blobs of lo..hi px (rings, frames, ellipse rings, porous bands, nested rings, blobs in
    their holes, cut by the image border) beside small holed and solid blobs, on dark clutter; channels == 3: unequal
    channels.  Frames with more than 64 holes or contours are drawn again.  Returns (frames, [(items, holes kept)])."""
    import cv2
    from tests.util import retr_tree_blobs
    frames, refs = [], []
    while len(frames) < n:
        img = np.zeros((H, W, 3) if channels == 3 else (H, W), np.uint8)

        def colour():
            if channels == 1:
                return int(rng.integers(52, 256))
            c = rng.integers(0, 256, size=3)
            if rng.uniform() < 0.2:
                c = [(0, 0, 255), (255, 0, 0), (52, 52, 52)][int(rng.integers(0, 3))]
            return tuple(int(v) for v in c)
        for _ in range(int(rng.integers(1, 4))):
            size = int(rng.integers(lo, hi + 1))
            cx, cy = int(rng.integers(-size // 4, W + size // 4)), int(rng.integers(-size // 4, H + size // 4))
            kind = int(rng.integers(0, 5))
            v = colour()
            if kind == 0:
                cv2.circle(img, (cx, cy), size // 2, v, int(rng.integers(1, 4)))
            elif kind == 1:
                w, h = size, int(rng.integers(8, size + 1))
                cv2.rectangle(img, (cx - w // 2, cy - h // 2), (cx + w // 2, cy + h // 2), v, int(rng.integers(1, 3)))
                if rng.uniform() < 0.6:
                    cv2.circle(img, (cx, cy), int(rng.integers(1, 6)), colour(), -1)
            elif kind == 2:
                cv2.ellipse(img, (cx, cy), (size // 2, int(rng.integers(4, size // 2 + 1))), float(rng.uniform(0, 180)), 0, 360, v, 1)
            elif kind == 3:
                cv2.circle(img, (cx, cy), size // 2, v, 1)
                cv2.circle(img, (cx, cy), max(3, size // 3), colour(), int(rng.integers(1, 3)))
                cv2.circle(img, (cx, cy), max(1, size // 8), colour(), 1)
            else:
                h = int(rng.integers(5, 10))
                m = rng.uniform(size=(h, size)) < 0.93
                m[0] = m[-1] = m[:, 0] = m[:, -1] = True
                y0, x0 = min(max(cy, 0), H - h), min(max(cx, 0), max(W - size, 0))
                ww = min(size, W - x0)
                img[y0:y0 + h, x0:x0 + ww][m[:, :ww]] = v
        for _ in range(int(rng.integers(0, 5))):
            cx, cy = int(rng.integers(0, W)), int(rng.integers(0, H))
            if rng.uniform() < 0.5:
                cv2.circle(img, (cx, cy), int(rng.integers(3, 12)), colour(), int(rng.integers(1, 3)))
            else:
                cv2.circle(img, (cx, cy), int(rng.integers(1, 6)), colour(), -1)
        img = np.maximum(img, rng.integers(0, 46 if channels == 3 else 52, size=img.shape, dtype=np.uint8))
        grey = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY) if channels == 3 else img
        items, kept, side, holes = retr_tree_blobs(grey > 51)
        if holes > 64 or len(items) > 64:
            continue
        frames.append(img)
        refs.append((items, kept, side))
    return np.stack(frames), refs

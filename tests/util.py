"""Helpers shared by the CPU and GPU test files."""
import importlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
synth = importlib.import_module("low-cost-mocap_b200.synth")


def load_golden(name, n=None, frames=True):
    """Golden vectors written by tests/golden/make_golden.py from the real reference.  ``n``: only the first n
    frame-sets / frames (every per-frame-set array is cut; the deterministic clutter of a pixel depends on its flat
    index only, so the first n frames get the same clutter as in the full set).  ``frames=False``: skip rebuilding
    the frames (tests that start from the blob lists)."""
    z = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    if n is not None and "frames_clean" in z:
        full = z["frames_clean"].shape[0]
        for k, v in list(z.items()):
            if isinstance(v, np.ndarray) and v.ndim >= 1 and v.shape[0] == full:
                z[k] = v[:n]
    if "frames_clean" in z and frames:
        z["frames"] = synth.add_clutter(z["frames_clean"], int(z["clutter_max"]), salt=int(z["clutter_salt"]))
    return z


def poses_from(z, prefix=""):
    R, t = z["R" + prefix], z["t" + prefix]
    return [{"R": R[i], "t": t[i]} for i in range(len(R))]


def obs_from(z):
    """(F,C,2) float array + (F,C) mask  ->  object array with None for missing views."""
    obs, mask = z["obs"], z["mask"]
    F, C, _ = obs.shape
    out = np.empty((F, C, 2), dtype=object)
    for f in range(F):
        for c in range(C):
            if mask[f, c]:
                v0, v1 = obs[f, c]
                out[f, c, 0] = int(v0) if float(v0).is_integer() else float(v0)
                out[f, c, 1] = int(v1) if float(v1).is_integer() else float(v1)
            else:
                out[f, c, 0] = None
                out[f, c, 1] = None
    return out


def as3(img):
    return np.repeat(img[:, :, None], 3, axis=2).copy()


# ------------------------------------------------------------------------- S1 references for blobs with holes
def porous_patch(n_holes, h=17, w=21):
    """An h x w block with n_holes one-pixel holes on the odd rows and columns, filled from the top: each hole opens
    the four cells around it, so the set-pixel and the filled polygon differ in area and in centre."""
    m = np.full((h, w), 255, np.uint8)
    spots = [(y, x) for y in range(1, h - 1, 2) for x in range(1, w - 1, 2)]
    assert n_holes <= len(spots)
    for y, x in spots[:n_holes]:
        m[y, x] = 0
    return m


def _centre(A2, SX6, SY6):
    """int(m10/m00) of the device's emission, in the same float64 operations."""
    m00 = float(A2) * 0.5
    return [int(float(SX6) * 0.16666666666666666 / m00), int(float(SY6) * 0.16666666666666666 / m00)]


def retr_tree_blobs(binary):
    """What cv.findContours(RETR_TREE, CHAIN_APPROX_SIMPLE) + cv.moments make of a binary image, in cv2's order, contours
    of zero area dropped (helpers.py:147-158): a list of (A2, SX6, SY6, npix, x, y) -- the integers 2*m00, 6*m10, 6*m01;
    npix is a blob's pixel count (connectedComponentsWithStats, 8-connectivity) or, for a hole, the size of the region
    it encloses: its 4-connected component of the complement of the blob around it, nested blobs included.
    Returns (items, number of kept hole contours, the holed blobs' largest bounding-box side, number of holes)."""
    import cv2
    from scipy import ndimage
    binary = (np.asarray(binary) != 0).astype(np.uint8)
    contours, hier = cv2.findContours(binary, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
    if not contours:
        return [], 0, 0, 0
    _, lab, stats, _ = cv2.connectedComponentsWithStats(binary, connectivity=8)
    parent = hier[0][:, 3]
    items, kept_holes, side, holes, fills = [], 0, 0, 0, {}
    for i, cnt in enumerate(contours):
        depth, p = 0, parent[i]
        while p >= 0:
            depth, p = depth + 1, parent[p]
        x0, y0 = (int(v) for v in cnt[0, 0])
        blob = lab[y0, x0]
        if depth % 2:                                  # a hole border runs through pixels of the blob around the hole
            if blob not in fills:                      # the complement's 4-components inside the blob's bounding box
                bx, by, bw, bh = (int(v) for v in stats[blob, :4])
                fills[blob] = (bx, by, lab[by:by + bh, bx:bx + bw] != blob)
                fills[blob] += (ndimage.label(fills[blob][2])[0],)
                side = max(side, bw, bh)
            bx, by, other, region = fills[blob]
            inside = np.zeros(other.shape, np.uint8)
            cv2.drawContours(inside, [cnt], 0, 1, thickness=cv2.FILLED, offset=(-bx, -by))
            ids = np.unique(region[(inside != 0) & other])
            assert len(ids) == 1, ids                  # exactly one enclosed region per hole contour
            npix = int((region == ids[0]).sum())
            holes += 1
        else:
            npix = int(stats[blob, cv2.CC_STAT_AREA])
        m = cv2.moments(cnt)
        if m["m00"] != 0:
            items.append((round(m["m00"] * 2), round(m["m10"] * 6), round(m["m01"] * 6), npix,
                          int(m["m10"] / m["m00"]), int(m["m01"] / m["m00"])))
            kept_holes += depth % 2
    return items, kept_holes, side, holes


def set_pixel_blobs(binary):
    """One item (A2, SX6, SY6, npix, x, y) per 8-connected blob from the polygon through its own set pixels' centres --
    the 2x2-cell sums of DESIGN.md section 5, holes left open -- in descending raster order of the blob's first pixel,
    blobs of zero area dropped: what S1 reports for an image it flags with MOCAP_F_HOLES."""
    import cv2
    b = (np.asarray(binary) != 0)
    n, lab, stats, _ = cv2.connectedComponentsWithStats(b.astype(np.uint8), connectivity=8)
    tl, tr, bl, br = (c.astype(np.int64) for c in (b[:-1, :-1], b[:-1, 1:], b[1:, :-1], b[1:, 1:]))
    cnt = tl + tr + bl + br
    y, x = np.mgrid[:b.shape[0] - 1, :b.shape[1] - 1].astype(np.int64)
    full, tri = cnt == 4, cnt == 3
    a2 = 2 * full + tri
    sx6 = np.where(full, 6 * x + 3, 0) + np.where(tri, tl * x + tr * (x + 1) + bl * x + br * (x + 1), 0)
    sy6 = np.where(full, 6 * y + 3, 0) + np.where(tri, (tl + tr) * y + (bl + br) * (y + 1), 0)
    cell_lab = np.maximum(np.maximum(lab[:-1, :-1], lab[:-1, 1:]), np.maximum(lab[1:, :-1], lab[1:, 1:]))   # one blob per cell
    sums = np.zeros((n, 3), np.int64)
    for k, v in enumerate((a2, sx6, sy6)):
        np.add.at(sums[:, k], cell_lab.ravel(), v.ravel())
    labels, first = np.unique(lab.ravel(), return_index=True)
    out = []
    for k in labels[np.argsort(-first)]:
        if k == 0 or sums[k, 0] == 0:
            continue
        A2, SX6, SY6 = (int(v) for v in sums[k])
        out.append((A2, SX6, SY6, int(stats[k, cv2.CC_STAT_AREA])) + tuple(_centre(A2, SX6, SY6)))
    return out


# ------------------------------------------------------------- DLT at near-degenerate geometry (S3 null vector)
def _yaw(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


def _dlt_rig(C, baseline, yaw_deg=0.0):
    """C cameras along x, `baseline` apart, each turned by yaw_deg more than the last; a slightly different K per camera
    so that the reference's "K of the k-th present view" (helpers.py:305-307) matters."""
    Ks = [np.array([[600.0 + 7 * c, 0, 320 - c], [0, 600.0 + 7 * c, 240 + c], [0, 0, 1]]) for c in range(C)]
    poses = [{"R": _yaw(np.radians(yaw_deg * c)), "t": np.array([-baseline * c, 0.0, 0.0])} for c in range(C)]
    return Ks, poses


def dlt_cases(n=200, seed=0):
    """Triangulation inputs where the smallest two eigenvalues of A^T A lie close together or B is badly scaled:
    (name, Ks, poses, obs f64 [n, C, 2], mask uint8 [n, C]).  Pixels are integers, as S1 delivers them."""
    rng = np.random.default_rng(seed)

    def observe(Ks, poses, X, noise, drop):
        C = len(poses)
        mask = np.ones((len(X), C), np.uint8)
        if drop:
            mask = (rng.uniform(size=(len(X), C)) > drop).astype(np.uint8)
            for f in range(len(X)):
                if mask[f].sum() < 2:
                    mask[f, rng.choice(C, 2, replace=False)] = 1
        obs = np.zeros((len(X), C, 2))
        for f in range(len(X)):
            k = 0
            for c in range(C):
                if not mask[f, c]:
                    continue
                x = Ks[k] @ (poses[c]["R"] @ X[f] + poses[c]["t"])      # the k-th present view is seen through K_k
                obs[f, c] = np.round(x[:2] / x[2] + rng.normal(0, noise, 2))
                k += 1
        return obs, mask

    cases = []
    Ks, poses = _dlt_rig(2, 0.01)
    X = rng.uniform(-0.5, 0.5, (n, 3)) + [0, 0, 3]
    cases.append(("baseline_1cm",) + (Ks, poses) + observe(Ks, poses, X, 0.0, 0))
    Ks, poses = _dlt_rig(2, 0.5)
    X = np.c_[rng.uniform(-2, 2, n), rng.uniform(-0.01, 0.01, n), rng.uniform(0.02, 0.08, n)]
    cases.append(("near_baseline_epipole",) + (Ks, poses) + observe(Ks, poses, X, 0.0, 0))
    X = np.c_[rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n), rng.uniform(1e-3, 1e-2, n)]
    cases.append(("in_front_of_camera0_plane",) + (Ks, poses) + observe(Ks, poses, X, 0.0, 0))
    Ks, poses = _dlt_rig(16, 0.1, 0.3)
    X = rng.uniform(-5, 5, (n, 3)) + [0, 0, 200]
    cases.append(("far_z200_16_views",) + (Ks, poses) + observe(Ks, poses, X, 0.0, 0.3))
    Ks, poses = _dlt_rig(4, 0.3, 5)
    X = rng.uniform(-0.5, 0.5, (n, 3)) + [0, 0, 3]
    cases.append(("wrong_correspondences_80px",) + (Ks, poses) + observe(Ks, poses, X, 80.0, 0.25))
    return cases


def dlt_matrix(Ks, poses, views, present):
    """A of helpers.py:314-316 from exactly the float64 entries numpy forms: P = K_k @ [R_c | t_c] for the k-th
    present view, rows y P[2] - P[1] and P[0] - x P[2]."""
    rows = []
    for k, c in enumerate(np.flatnonzero(present)):
        P = Ks[k] @ np.c_[poses[c]["R"], poses[c]["t"]]
        x, y = views[c]
        rows.append(y * P[2, :] - P[1, :])
        rows.append(P[0, :] - x * P[2, :])
    return np.array(rows)


def exact_dlt_point(A, dps=60):
    """X from the null vector of A^T A (the eigenvector of its smallest eigenvalue), A's float64 entries taken as
    exact, in `dps`-digit arithmetic; None where that vector's last component is 0 (a point at infinity)."""
    import mpmath as mp
    with mp.workdps(dps):
        Am = mp.matrix([[mp.mpf(float(v)) for v in row] for row in A])
        E, Q = mp.eigsy(Am.T * Am)
        i = min(range(4), key=lambda k: abs(E[k]))
        v = [Q[r, i] for r in range(4)]
        if v[3] == 0:
            return None
        return np.array([float(v[0] / v[3]), float(v[1] / v[3]), float(v[2] / v[3])])

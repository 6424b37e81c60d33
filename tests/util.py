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

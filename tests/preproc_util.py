"""Cameras, distortions and frames for the tests of the capture-side preprocessing (csrc/preproc.cu,
csrc/preproc_tile.cuh) against the reference's cv2 chain (helpers.py:70-82, restated by oracle.ref_port)."""
import numpy as np

# distortion_coef of the reference's camera-params.json: k1 k2 p1 p2 k3
DIST = np.array([-1.26372388e-01, 2.62661497e-01, 1.21306197e-03, 2.24507008e-04, -2.48534118e-01])

FRAME_KINDS = ("noise", "white", "black", "binary")


def fuzz_camera(rng, S):
    """One camera of the host-stepped fuzz: focal length 0.5 S .. 1.5 S, fy within 10 % of fx, principal point up to
    5 px off centre, the camera-params.json distortion scaled by a factor in [-3, 3]."""
    f0 = float(rng.uniform(0.5, 1.5) * S)
    K = np.array([[f0, 0, S / 2.0 + rng.uniform(-5, 5)], [0, f0 * rng.uniform(0.9, 1.1), S / 2.0 + rng.uniform(-5, 5)], [0, 0, 1]])
    dist = np.array([-0.126, 0.263, 0.0012, 0.0002, -0.249]) * rng.uniform(-3.0, 3.0)
    return K, dist


def rig(rng, C, S, clamp=False):
    """C cameras that share nothing: each its own K (fx != fy, both in 0.5 S .. 1.5 S, principal point up to 0.15 S off
    centre), its own distortion (camera-params.json scaled by a factor in [-3, 3]; camera 1 tangential only) and its
    own rotation (0 and 2 both present).  clamp: the last camera instead has a k3 so strong that its undistortion map
    runs into the int16 clamp of CV_16SC2 (|source| > 32767 px, far below where u * 32 would leave int range).
    Returns (K list, distortion list, rotation list)."""
    Ks, dists = [], []
    for c in range(C):
        fx, fy = rng.uniform(0.5, 1.5, 2) * S
        if abs(fx - fy) < 0.02 * S:
            fy = fx + 0.1 * S if fx < S else fx - 0.1 * S
        cx, cy = S * (0.5 + rng.uniform(-0.15, 0.15, 2))
        Ks.append(np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]]))
        d = DIST * rng.uniform(-3.0, 3.0)
        if c == 1:
            d = d * np.array([0, 0, 1, 1, 0])
        dists.append(d)
    if clamp:
        Ks[-1] = np.array([[1.1 * S, 0, 0.47 * S], [0, 0.9 * S, 0.53 * S], [0, 0, 1]])
        dists[-1] = np.array([0, 0, 0, 0, 2000.0])
    rots = [int(r) for r in rng.choice([0, 2], C)]
    if C > 1 and len(set(rots)) == 1:
        rots[int(rng.integers(C))] = 2 - rots[0]
    return Ks, dists, rots


def frame(rng, kind, in_h, in_w):
    """One raw camera frame: uniform noise (worst case for every rounding), saturated 255, zero, or binary 0 / 255
    noise (drives the sharpening filter past both ends of the byte range)."""
    if kind == "noise":
        return rng.integers(0, 256, size=(in_h, in_w, 3), dtype=np.uint8)
    if kind == "white":
        return np.full((in_h, in_w, 3), 255, dtype=np.uint8)
    if kind == "black":
        return np.zeros((in_h, in_w, 3), dtype=np.uint8)
    return (rng.integers(0, 2, size=(in_h, in_w, 3)) * 255).astype(np.uint8)


def rig_poses(C):
    """World-to-camera poses of a row of cameras 0.3 apart along x, all looking down +z."""
    return [{"R": np.eye(3), "t": np.array([0.3 * (c - (C - 1) / 2.0), 0.0, 0.0])} for c in range(C)]


def marker_frames(rng, B, S, in_h, Ks, dists, rots, poses, n_points=4, clutter=25):
    """Raw frames [B, C, in_h, S, 3] of a marker scene: dark clutter and bright Gaussian spots.  Each spot is a 3D point
    projected through its camera's pose, K and distortion (cv2.projectPoints), so that after undistortion it sits
    where the pinhole model puts it; then carried from make_square's frame into the raw one (row offset, rotation)."""
    import cv2
    C = len(Ks)
    ay = (S - in_h) // 2
    raw = rng.integers(0, clutter, size=(B, C, in_h, S, 3), dtype=np.uint8)
    yy, xx = np.mgrid[:in_h, :S]
    for b in range(B):
        X = np.stack([rng.uniform(-0.3, 0.3, n_points), rng.uniform(-0.2, 0.2, n_points), rng.uniform(2.0, 3.0, n_points)], axis=1)
        for c in range(C):
            t = np.asarray(poses[c]["t"], dtype=np.float64)
            uv, _ = cv2.projectPoints(X, np.zeros(3), t, Ks[c], np.asarray(dists[c], dtype=np.float64))
            for u, v in uv.reshape(-1, 2):
                v = v - ay
                if rots[c] == 2:
                    u, v = S - 1 - u, in_h - 1 - v
                if -4 <= u < S + 4 and -4 <= v < in_h + 4:
                    spot = (255 * np.exp(-((yy - v) ** 2 + (xx - u) ** 2) / (2 * 2.0 ** 2))).astype(np.uint8)
                    raw[b, c] = np.maximum(raw[b, c], spot[:, :, None])
    return raw


def cv2_chain(raw, Ks, dists, rots):
    """The reference's preprocessing of raw frames [B, C, in_h, in_w, 3], each with its own camera's K, distortion and
    rotation -> [B, C, S, S, 3]."""
    from oracle.ref_port import RefPort
    port = RefPort(Ks)
    B, C = raw.shape[:2]
    return np.stack([np.stack([port.preprocess(raw[b, c], c, dists[c], rots[c]) for c in range(C)]) for b in range(B)])

"""Shared by the live-loop tests (tests/test_live_on_host.py, tests/test_gpu_live.py), the golden generator
tests/golden/make_golden_live.py and tools/live_time.py: a seeded scene of two drones and clutter seen by cameras of the
reference's shipped camera-params.json, the raw frames of each read rendered from it (the same bytes wherever they are
rendered, so no frame is stored), the session script, and the oracle chain of one read -- RefPort preprocessing ->
find_dot -> match_and_triangulate + the reference's world transform -> RefPort.locate_objects ->
track_util.OracleKalmanFilter -- in the layout of the live result."""
import json
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "live_loop.npz")

IN_W, IN_H = 320, 240
S = 320
K = np.array([[320.0, 0, 160], [0, 320.0, 160], [0, 0, 1]])
# camera-params.json of the reference (every camera ships the same values)
DIST = np.array([-1.26372388e-01, 2.62661497e-01, 1.21306197e-03, 2.24507008e-04, -2.48534118e-01])
DRONE_HALF, DRONE_H = 0.075, np.sqrt(0.095 ** 2 - 0.075 ** 2)     # synth.make_drone_points: markers 0.15 apart, third 0.095 from both
FLOOR_Y = 0.6                                                       # the floor plane in scene coordinates (cameras at y = -1)


def look_at(centre, target=(0.0, 0.0, 0.0)):
    z = np.asarray(target, float) - centre
    z /= np.linalg.norm(z)
    x = np.cross(z, [0.0, -1.0, 0.0])
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return {"R": R, "t": -R @ centre}


def rig(C, rng):
    """C cameras on a 1.4 m circle 1.3 m above the scene origin, looking at it."""
    poses = []
    for c in range(C):
        a = 2 * np.pi * c / C + rng.uniform(-0.15, 0.15)
        poses.append(look_at(np.array([1.4 * np.sin(a), -1.3 + rng.uniform(-0.1, 0.1), -1.4 * np.cos(a)])))
    return poses


# ---------------------------------------------------------------------------------------------- world transform
def world_of(p, M):
    """helpers.py:96-103 for one point: flip x and y, the 4x4 matrix, dehomogenise, swap y and z (the reference's own
    arithmetic, in its order)."""
    q = np.array([[-1, 0, 0], [0, -1, 0], [0, 0, 1]]) @ np.asarray(p, dtype=np.float64)
    q = np.concatenate((q, [1]))
    q = np.array(M) @ q
    q = q[:3] / q[3]
    q[1], q[2] = q[2], q[1]
    return q


def scene_of(w, M):
    """Inverse of world_of for an affine M."""
    q = np.array([w[0], w[2], w[1], 1.0])
    p = np.linalg.solve(np.asarray(M, dtype=np.float64), q)[:3]
    return np.array([-p[0], -p[1], p[2]])


def floor_points(seed):
    """Recorded floor points as the UI sends them to acquire-floor (one list of points per frame), in the frame the
    identity world matrix gives."""
    rng = np.random.default_rng(seed + 1)
    pts = []
    for _ in range(12):
        x, z = rng.uniform(-0.8, 0.8, 2)
        pts.append([world_of([x, FLOOR_Y + 0.04 * x - 0.02 * z, z], np.eye(4)).tolist()])
    return pts


# ---------------------------------------------------------------------------------------------- scene
def make_scene(seed, M, C=4, rotations=None, radius=(2, 4), drones=2, clutter=1, large=False):
    """Drones defined in the world frame of M (horizontal triplets, the third marker on the side that gives drone d
    droneIndex d), mapped back to scene coordinates; clutter points; the rig."""
    rng = np.random.default_rng(seed)
    poses = rig(C, rng)
    if rotations is None:
        rotations = [0, 2] * (C // 2) + [0] * (C % 2)
    centres = [np.array([0.35 * (2 * d - drones + 1), 0.0, 0.0]) + rng.uniform(-0.05, 0.05, 3) for d in range(drones)]
    return dict(seed=seed, C=C, poses=poses, rotations=list(rotations), M=np.asarray(M, dtype=np.float64),
                centres=[world_of(c, M) for c in centres], phase=rng.uniform(0, 2 * np.pi, drones),
                yaw0=rng.uniform(-1.2, 1.2, drones), radius=radius, clutter=clutter, large=large)


def marker_points(scene, k):
    """Scene-space marker points of read k: per drone a triplet (pair, then the third marker), then the clutter."""
    rng = np.random.default_rng([scene["seed"], k])
    M = scene["M"]
    pts = []
    for d, cw in enumerate(scene["centres"]):
        t = 0.03 * k + scene["phase"][d]
        c = cw + np.array([0.12 * np.sin(t), 0.12 * np.cos(0.7 * t), 0.03 * np.sin(1.3 * t)])
        yaw = scene["yaw0"][d] + 0.2 * np.sin(0.05 * k)
        u = np.array([np.cos(yaw), np.sin(yaw), 0.0])
        side = np.array([-np.sin(yaw), np.cos(yaw), 0.0])
        side *= 1.0 if (side[1] > 0) == (d == 0) else -1.0
        for w in (c + DRONE_HALF * u, c - DRONE_HALF * u, c + DRONE_H * side):
            pts.append(scene_of(w + rng.normal(0, 0.001, 3), M))
    for _ in range(scene["clutter"]):
        pts.append(rng.uniform(-0.6, 0.6, 3) * [1, 0.4, 1])
    return np.array(pts)


def render_read(scene, k, dark=False):
    """Raw frames of read k, uint8 [C, IN_H, IN_W, 3]: dark noise, and unless `dark` a disc per marker at
    cv2.projectPoints(X, ..., K, DIST) less make_square's row offset, drawn in the rotated frame and turned back, so that
    preprocessing puts it on the pinhole projection."""
    rng = np.random.default_rng([scene["seed"], k, 7])
    C = scene["C"]
    X = marker_points(scene, k)
    out = np.empty((C, IN_H, IN_W, 3), np.uint8)
    ay = (S - IN_H) // 2
    for c in range(C):
        img = rng.integers(0, 12, (IN_H, IN_W, 3), dtype=np.uint8)
        if not dark:
            p = scene["poses"][c]
            rvec, _ = cv2.Rodrigues(p["R"])
            uv, _ = cv2.projectPoints(X, rvec, p["t"], K, DIST)
            for j, (u, v) in enumerate(uv[:, 0]):
                if not (0 <= u < S and ay <= v < ay + IN_H):
                    continue
                r = int(rng.integers(scene["radius"][0], scene["radius"][1] + 1))
                val = int(rng.integers(200, 256))
                centre = (int(round(u * 16)), int(round((v - ay) * 16)))
                if scene["large"]:
                    cv2.circle(img, centre, r * 16, (val, val, val), -1, cv2.LINE_8, 4)
                else:
                    cv2.circle(img, centre, r * 16, (val, val, val), -1, cv2.LINE_AA, 4)
        out[c] = np.rot90(img, k=-scene["rotations"][c])
    return out


# ---------------------------------------------------------------------------------------------- session script
CAPTURE, TRIANGULATE, LOCATE = 1, 2, 4


def session_script():
    """Per read: (mode, dark, filter generation, world matrix index).  15 capture-only reads; triangulation starts
    (filter 1, matrix 0); 10 reads; locating starts: 60 reads with 5 all-dark ones in a row; set-origin (matrix 1); stop
    and start of triangulation (filter 2); 20 reads."""
    reads = [(CAPTURE, False, 0, -1)] * 15
    reads += [(CAPTURE | TRIANGULATE, False, 1, 0)] * 10
    reads += [(CAPTURE | TRIANGULATE | LOCATE, 30 <= i < 35, 1, 0) for i in range(60)]
    reads += [(CAPTURE | TRIANGULATE | LOCATE, False, 2, 1)] * 20
    return reads


def timestamp(k):
    return 1000.0 + k / 90.0


# ---------------------------------------------------------------------------------------------- oracle chain
def oracle_read(port, scene, raw, mode, M, kf, now, num_objects=2, max_roots=128):
    """One read through the oracle chain, in the layout of MocapContext.live_host's result for that read (numpy
    arrays of one read each) plus "frames", the processed frames with the drop-in's dots.  kf: an OracleKalmanFilter
    whose clock reads now[0]."""
    from oracle.ref_port import RefPort  # noqa: F401  (port is a RefPort)
    C = scene["C"]
    frames = np.stack([port.preprocess(raw[c], c, DIST, scene["rotations"][c]) for c in range(C)])
    res = dict(flags=np.zeros(1, np.int32), gate=np.zeros(1, np.uint8), blob_n=np.zeros((1, C), np.int32),
               first=np.full((1, C, 2), -1, np.int32), n=np.zeros(1, np.int32), obj=np.zeros((1, max_roots, 3)),
               err=np.zeros((1, max_roots)), n_objects=np.zeros(1, np.int32), objects=np.zeros((1, max_roots, 5)),
               drone_index=np.zeros((1, max_roots), np.int32), called=np.zeros(1, np.uint8),
               pos=np.zeros((1, num_objects, 3), np.float32), vel=np.zeros((1, num_objects, 3), np.float32),
               heading=np.zeros((1, num_objects)), present=np.zeros((1, num_objects), np.uint8),
               chosen=np.full((1, num_objects), -1, np.int32))
    if not mode & CAPTURE:
        res["frames"] = frames
        return res
    pts = [port.find_dot(frames[c]) for c in range(C)]
    for c in range(C):
        real = [p for p in pts[c] if p[0] is not None]
        res["blob_n"][0, c] = len(real)
        if real:
            res["first"][0, c] = real[0]
        for x, y in real:
            if 0 <= x < S and 0 <= y < S:
                frames[c, y, x] = (100, 255, 100)
    res["frames"] = frames
    res["gate"][0] = int((res["blob_n"][0] > 0).any())
    if not mode & TRIANGULATE or not res["gate"][0]:
        return res
    err, obj, _ = port.match_and_triangulate(pts, scene["poses"])
    obj = np.array([world_of(p, M) for p in obj]) if len(obj) else np.zeros((0, 3))
    res["n"][0] = len(err)
    res["obj"][0, :len(err)] = obj
    res["err"][0, :len(err)] = err
    if not mode & LOCATE:
        return res
    objects = port.locate_objects(obj, err) if len(err) else []
    res["n_objects"][0] = len(objects)
    for i, o in enumerate(objects):
        res["objects"][0, i] = [*o["pos"], o["heading"], o["error"]]
        res["drone_index"][0, i] = o["droneIndex"]
    res["called"][0] = 1
    rec, chosen = kf.predict_location(objects)
    for r in rec:
        d = r["droneIndex"]
        res["pos"][0, d], res["vel"][0, d], res["heading"][0, d], res["present"][0, d] = r["pos"], r["vel"], r["heading"], 1
    res["chosen"][0] = chosen
    return res


def encode_events(events):
    return json.dumps([[name, payload] for name, payload in events])


def encode_serial(lines):
    return json.dumps([b.decode("latin-1") for b in lines])


def load_golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


# ---------------------------------------------------------------------------------------------- replay of the golden
def golden_scene(g):
    scene = make_scene(int(g["seed"]), g["worlds"][0])
    assert all(np.array_equal(p["R"], R) and np.array_equal(p["t"], t) for p, R, t in zip(scene["poses"], g["R"], g["tvec"]))
    return scene


class StandinCameras:
    """The attributes of the reference's Cameras that _camera_read reads, with a scripted driver and recording socketio
    and serial port."""

    def __init__(self, g, scene):
        self.g, self.scene = g, scene
        self.camera_params = [{"intrinsic_matrix": K.tolist(), "distortion_coef": DIST.tolist(), "rotation": int(r)} for r in g["rotations"]]
        self.num_cameras = len(self.camera_params)
        self.num_objects = int(g["num_objects"])
        self.drone_armed = [bool(a) for a in g["drone_armed"]]
        self.camera_poses = [{"R": R.tolist(), "t": t.tolist()} for R, t in zip(g["R"], g["tvec"])]
        self.is_capturing_points = self.is_triangulating_points = self.is_locating_objects = False
        self.to_world_coords_matrix = None
        self.kalman_filter = None
        self.events, self.lines = [], []
        self.socketio = type("Sio", (), {"emit": lambda _s, name, payload: self.events.append((name, json.loads(json.dumps(payload))))})()
        self.ser = type("Ser", (), {"write": lambda _s, b: self.lines.append(bytes(b))})()
        self.serialLock = __import__("threading").Lock()
        self.frames = None
        self.cameras = type("Drv", (), {"read": lambda _s: ([f.copy() for f in self.frames], None)})()

    def set_read(self, k):
        """State and frames of golden read k."""
        g = self.g
        mode, gen, wi = int(g["mode"][k]), int(g["filter_gen"][k]), int(g["world_index"][k])
        self.is_capturing_points = bool(mode & CAPTURE)
        self.is_triangulating_points = bool(mode & TRIANGULATE)
        self.is_locating_objects = bool(mode & LOCATE)
        self.to_world_coords_matrix = g["worlds"][wi].tolist() if wi >= 0 else None
        if gen and (self.kalman_filter is None or self.kalman_filter[0] != gen):
            self.kalman_filter = (gen,)          # a new object: start_trangulating_points ran
        self.frames = list(render_read(self.scene, k, bool(g["dark"][k])))
        self.events, self.lines = [], []


def _close(a, b, atol, rtol=0.0):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all(np.abs(a - b) <= atol + rtol * np.abs(b)))


def compare_events(got, want, tol_track=5e-4):
    """The bars of the golden replay; returns a list of differences (empty: equal within the bars)."""
    bad = []
    if [n for n, _ in got] != [n for n, _ in want]:
        return [f"event names {[n for n, _ in got]} != {[n for n, _ in want]}"]
    for (name, g), (_, w) in zip(got, want):
        if name == "image-points":
            if g != w:
                bad.append(f"image-points {g} != {w}")
            continue
        if len(g["object_points"]) != len(w["object_points"]):
            bad.append(f"point count {len(g['object_points'])} != {len(w['object_points'])}")
            continue
        if w["object_points"] and not _close(g["object_points"], w["object_points"], 1e-7, 1e-7):
            bad.append("object_points")
        if w["errors"] and not _close(g["errors"], w["errors"], 0.0, 1e-9):
            bad.append("errors")
        if [o["droneIndex"] for o in g["objects"]] != [o["droneIndex"] for o in w["objects"]]:
            bad.append("objects: count / droneIndex")
        else:
            for a, b in zip(g["objects"], w["objects"]):
                if not (_close(a["pos"], b["pos"], 1e-7, 1e-7) and _close(a["error"], b["error"], 0.0, 1e-9)
                        and _close(a["heading"], b["heading"], 1e-9)):
                    bad.append(f"object {a} != {b}")
        if [o["droneIndex"] for o in g["filtered_objects"]] != [o["droneIndex"] for o in w["filtered_objects"]]:
            bad.append("filtered_objects: presence")
        else:
            for a, b in zip(g["filtered_objects"], w["filtered_objects"]):
                if not (_close(a["pos"], b["pos"], tol_track) and _close(a["vel"], b["vel"], tol_track)
                        and _close(a["heading"], b["heading"], 1e-9)):
                    bad.append(f"filtered {a} != {b}")
    return bad


def compare_serial(got, want, want_events, tol_track=5e-4, report=print):
    """Serial lines identical, except a value one unit apart in the 4th decimal where the unrounded value (the golden's
    filtered_objects entry) lies within the tracker's bar of a rounding midpoint; every such case is reported."""
    if len(got) != len(want):
        return [f"{len(got)} serial lines != {len(want)}"]
    bad = []
    filt = {o["droneIndex"]: o for _, p in want_events if "filtered_objects" in p for o in p["filtered_objects"]}
    for a, b in zip(got, want):
        if a == b:
            continue
        da, db = a.decode(), b.decode()
        if da[0] != db[0]:
            bad.append(f"{da} != {db}")
            continue
        d = int(db[0])
        ja, jb = json.loads(da[1:]), json.loads(db[1:])
        raw = list(filt[d]["pos"]) + [None] + list(filt[d]["vel"]) if d in filt else None
        for i, (x, y) in enumerate(zip(ja["pos"] + ja["vel"], jb["pos"] + jb["vel"])):
            if x == y:
                continue
            u = raw[i] if raw else None
            mid = (np.floor(u * 1e4) + 0.5) / 1e4 if u is not None else None
            if u is not None and abs(abs(x - y) - 1e-4) < 1e-9 and abs(u - mid) <= tol_track:
                report(f"serial: {x} vs {y}, unrounded {u!r} is {abs(u - mid):.1e} from the midpoint {mid}")
            else:
                bad.append(f"{da} != {db}")
    return bad

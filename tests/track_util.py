"""Helpers shared by the CPU and GPU tests of the drone tracker (csrc/track.cuh, csrc/track.cu), the golden generator
tests/golden/make_golden_track.py and tools/track_time.py: seeded streams of located frame-sets in the layout
mocap_locate_objects_dev writes, a restatement of the reference's KalmanFilter / LowPassFilter with an injectable clock
(the oracle of the tracker), and the host build of the step code behind api.Tracker's interface."""
import os

import cv2
import numpy as np
from scipy.signal import butter, lfilter

from tests.hostbuild import ptr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "track_live.npz")
MAXO = 8                 # object rows per frame-set in the streams


# ---------------------------------------------------------------------------------------------- streams
def make_stream(B, D=2, seed=0, t0=1.7e9 + 1234.5, hz=90.0, jitter=0.3, dropout=0.08, absence=None, empty_frac=0.03,
                extra_frac=0.1, clutter_frac=0.3, reset_at=-1):
    """B frame-sets of D drones flying smooth paths within +-2 m, as locate_objects reports them: each present drone
    one object (droneIndex d) near its position; sometimes a second, farther object with the same index; clutter
    objects with an index >= D, or with another present drone's index 0.5-1 m from that drone; some frame-sets
    without objects.  Drone d drops out with probability `dropout`; `absence` = (drone, first, count) keeps one away
    for `count` frame-sets.  Timestamps at `hz` with +-`jitter` relative jitter from the epoch-sized `t0`.  reset_at:
    the index of the frame-set before which reset() is called (-1: never), at reset_time just before it.
    Returns a dict of numpy arrays: objects f64 [B, MAXO, 5], drone_index int32 [B, MAXO], n int32 [B], t f64 [B],
    reset_at, reset_time."""
    rng = np.random.default_rng(seed)
    t = t0 + np.cumsum((1.0 + rng.uniform(-jitter, jitter, B)) / hz)
    centre = rng.uniform(-1.2, 1.2, (D, 3))
    amp = rng.uniform(0.2, 0.7, (D, 3))
    w = rng.uniform(0.3, 1.5, (D, 3))
    ph = rng.uniform(0, 2 * np.pi, (D, 3))
    objects = np.zeros((B, MAXO, 5))
    di = np.full((B, MAXO), -1, dtype=np.int32)
    n = np.zeros(B, dtype=np.int32)
    for s in range(B):
        if rng.uniform() < empty_frac:
            continue
        tt = t[s] - t0
        rows = []
        truth = centre + amp * np.sin(w * tt + ph)
        present = [d for d in range(D) if rng.uniform() >= dropout and not (absence and absence[0] == d and absence[1] <= s < absence[1] + absence[2])]
        for d in present:
            head = np.clip(0.8 * np.sin(0.4 * tt + d), -np.pi / 2, np.pi / 2) + rng.normal(0, 0.01)
            rows.append((truth[d] + rng.normal(0, 0.002, 3), head, d))
            if rng.uniform() < extra_frac:
                off = rng.normal(0, 1, 3)
                rows.append((truth[d] + off / np.linalg.norm(off) * rng.uniform(0.3, 1.0), rng.uniform(-1.5, 1.5), d))
        while rng.uniform() < clutter_frac and len(rows) < MAXO:
            if present and rng.uniform() < 0.5:
                host = present[rng.integers(len(present))]
                off = rng.normal(0, 1, 3)
                other = [d for d in present if d != host]
                idx = other[rng.integers(len(other))] if other else D
                rows.append((truth[host] + off / np.linalg.norm(off) * rng.uniform(0.5, 1.0), rng.uniform(-1.5, 1.5), idx))
            else:
                rows.append((rng.uniform(-2, 2, 3), rng.uniform(-1.5, 1.5), int(rng.integers(D, max(D + 1, 8)))))
        rows = rows[:MAXO]
        order = rng.permutation(len(rows))
        for i, r in enumerate(order):
            p, h, d = rows[r]
            objects[s, i, :3] = p
            objects[s, i, 3] = h
            objects[s, i, 4] = rng.uniform(0, 2)
            di[s, i] = d
        n[s] = len(rows)
    reset_time = t[reset_at] - 0.002 if reset_at >= 0 else 0.0
    return dict(objects=objects, drone_index=di, n=n, t=t, reset_at=int(reset_at), reset_time=float(reset_time))


def objects_of(stream, s):
    """Frame-set s as the list locate_objects returns (pos f64 [3], heading np.float64, error, droneIndex int)."""
    return [{"pos": stream["objects"][s, i, :3].copy(), "heading": np.float64(stream["objects"][s, i, 3]),
             "error": float(stream["objects"][s, i, 4]), "droneIndex": int(stream["drone_index"][s, i])}
            for i in range(int(stream["n"][s]))]


def load_golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


def golden_stream(g):
    return dict(objects=g["objects"], drone_index=g["drone_index"], n=g["n"], t=g["t"], reset_at=int(g["reset_at"]),
                reset_time=float(g["reset_time"]))


# ---------------------------------------------------------------------------------------------- oracle
class _LowPass:
    """LowPassFilter(cutoff 20, sampling 60, dims, order 5, buffer 300): lfilter from zero state over the buffer,
    the buffer cut to its last 150 samples once it holds 300."""

    def __init__(self, dims):
        self.b, self.a = butter(5, 20 / (60.0 / 2), btype="low")
        self.buf = np.empty((0, dims))

    def filter(self, sample):
        self.buf = np.vstack((self.buf, np.asarray(sample)[np.newaxis]))
        y = np.apply_along_axis(lambda col: lfilter(self.b, self.a, col), 0, self.buf)
        if self.buf.shape[0] >= 300:
            self.buf = self.buf[-150:]
        return y[-1]


class OracleKalmanFilter:
    """The reference's KalmanFilter(num_objects) restated with cv2.KalmanFilter and lfilter, with the clock injected
    (one reading per call).  Kept as the reference behaves: statePre and statePost share one buffer after the init
    step, so the returned state is the posterior; prev_positions starts (and restarts on reset) as an integer zero
    list.  predict_location also returns, per drone, the row of the object it chose (-1 if absent)."""

    def __init__(self, num_objects, clock):
        self.n, self.clock = num_objects, clock
        self.prev_time = 0
        self.kf, self.prev, self.lp_xy, self.lp_z, self.lp_h = [], [], [], [], []
        for _ in range(num_objects):
            k = cv2.KalmanFilter(9, 6)
            k.transitionMatrix = np.eye(9, dtype=np.float32)
            k.processNoiseCov = np.eye(9, dtype=np.float32) * 1e-2
            k.measurementNoiseCov = np.eye(6, dtype=np.float32)
            k.measurementMatrix = np.eye(6, 9, dtype=np.float32)
            k.statePost = np.zeros((9, 1), dtype=np.float32)
            self.kf.append(k)
            self.prev.append([0, 0, 0])
            self.lp_xy.append(_LowPass(2))
            self.lp_z.append(_LowPass(1))
            self.lp_h.append(_LowPass(1))

    def predict_location(self, objects):
        now = self.clock()
        dt = now - self.prev_time
        self.prev_time = now
        out, chosen = [], [-1] * self.n
        for d in range(self.n):
            rows = [i for i, o in enumerate(objects) if o["droneIndex"] == d]
            if not rows:
                continue
            cands = [objects[i]["pos"] for i in rows]
            k = self.kf[d]
            T = k.transitionMatrix
            T[:3, 3:6] = dt * np.eye(3)
            T[3:6, 6:9] = dt * np.eye(3)
            T[:3, 6:9] = 0.5 * dt ** 2 * np.eye(3)
            if all(k.statePost == 0):
                x = k.statePost
                x[0:3] = cands[0].reshape((3, 1))
                k.statePost = x
                k.statePre = x
            pred = k.predict()[:3].T[0]
            j = int(np.argmin(np.sqrt(np.sum((cands - pred) ** 2, axis=1))))
            p = cands[j].astype(np.float32)
            v = ((p - self.prev[d]) / dt).astype(np.float32)
            self.prev[d] = p
            k.correct(np.concatenate((p, v)))
            state = k.statePre[:6].T[0]
            heading = self.lp_h[d].filter(objects[rows[j]]["heading"])[0]
            vel = state[3:6].copy()
            vel[0:2] = self.lp_xy[d].filter(vel[0:2])
            vel[2] = self.lp_z[d].filter(vel[2])[0]
            out.append({"pos": state[:3].copy(), "vel": vel, "heading": heading, "droneIndex": d})
            chosen[d] = rows[j]
        return out, chosen

    def reset(self):
        self.prev_time = self.clock() - 20
        for d, k in enumerate(self.kf):
            k.statePost = np.zeros((9, 1), dtype=np.float32)
            self.prev[d] = np.array([0, 0, 0])


def records_to_arrays(records, D):
    """One call's list of records -> pos f32 [D, 3], vel f32 [D, 3], heading f64 [D], present uint8 [D] (0 where absent)."""
    pos = np.zeros((D, 3), np.float32); vel = np.zeros((D, 3), np.float32)
    head = np.zeros(D); pres = np.zeros(D, np.uint8)
    for r in records:
        d = r["droneIndex"]
        pos[d], vel[d], head[d], pres[d] = r["pos"], r["vel"], r["heading"], 1
    return pos, vel, head, pres


def run_oracle(stream, D):
    """The oracle over a whole stream: dict pos, vel, heading, present, chosen, per frame-set and drone."""
    now = [0.0]
    kf = OracleKalmanFilter(D, lambda: now[0])
    B = len(stream["t"])
    out = dict(pos=np.zeros((B, D, 3), np.float32), vel=np.zeros((B, D, 3), np.float32), heading=np.zeros((B, D)),
               present=np.zeros((B, D), np.uint8), chosen=np.full((B, D), -1, np.int32))
    for s in range(B):
        if s == stream["reset_at"]:
            now[0] = stream["reset_time"]
            kf.reset()
        now[0] = float(stream["t"][s])
        rec, ch = kf.predict_location(objects_of(stream, s))
        out["pos"][s], out["vel"][s], out["heading"][s], out["present"][s] = records_to_arrays(rec, D)
        out["chosen"][s] = ch
    return out


# ---------------------------------------------------------------------------------------------- host build
class HostTracker:
    """The host build with the interface of api.Tracker, on numpy arrays."""

    def __init__(self, lib, D):
        self.lib, self.D = lib, D
        self.h = lib.hc_track_new(D)

    def __del__(self):
        self.lib.hc_track_free(self.h)

    def reset(self, prev_time):
        self.lib.hc_track_reset(self.h, float(prev_time))

    def track(self, objects, drone_index, n, t):
        objects = np.ascontiguousarray(objects, np.float64); drone_index = np.ascontiguousarray(drone_index, np.int32)
        n = np.ascontiguousarray(n, np.int32); t = np.ascontiguousarray(t, np.float64)
        B, M = drone_index.shape
        out = dict(pos=np.zeros((B, self.D, 3), np.float32), vel=np.zeros((B, self.D, 3), np.float32),
                   heading=np.zeros((B, self.D)), present=np.zeros((B, self.D), np.uint8), chosen=np.zeros((B, self.D), np.int32))
        self.lib.hc_track(self.h, ptr(objects), ptr(drone_index), ptr(n), M, ptr(t), B, ptr(out["pos"]), ptr(out["vel"]),
                          ptr(out["heading"]), ptr(out["present"]), ptr(out["chosen"]))
        return out


def run_batches(tracker, stream, sizes, track):
    """Run a stream through `tracker` in consecutive batches of the given sizes (the rest in one last batch), calling
    tracker.reset before the batch that starts at reset_at (so reset_at must start a batch).  track(tracker, stream
    slice) -> dict of numpy arrays.  Returns the outputs concatenated."""
    B = len(stream["t"])
    cuts = [0]
    for k in sizes:
        if cuts[-1] + k < B:
            cuts.append(cuts[-1] + k)
    if stream["reset_at"] >= 0 and stream["reset_at"] not in cuts:
        cuts = sorted(cuts + [stream["reset_at"]])
    cuts.append(B)
    parts = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        if a == stream["reset_at"]:
            tracker.reset(stream["reset_time"] - 20)
        sl = {k: stream[k][a:b] for k in ("objects", "drone_index", "n", "t")}
        parts.append(track(tracker, sl))
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def host_run(lib, stream, D, sizes=()):
    return run_batches(HostTracker(lib, D), stream, sizes,
                       lambda tr, sl: tr.track(sl["objects"], sl["drone_index"], sl["n"], sl["t"]))

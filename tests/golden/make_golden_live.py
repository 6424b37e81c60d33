"""Writes tests/golden/live_loop.npz by running the REAL reference's Cameras._camera_read (computer_code/api/helpers.py of
a jyjblrd/Low-Cost-Mocap checkout, imported unmodified through oracle/ref_harness) over a scripted session:

    MOCAP_REFERENCE_DIR=<checkout> python tests/golden/make_golden_live.py

The driver stub's read() returns the raw frames tests/live_util.render_read renders from the seed; socketio and the
serial port record what they receive; helpers' time.sleep is a no-op and KalmanFilter.py's time.time returns the
read's timestamp (both of its reads in a call).  The world matrix comes from the reference's own acquire-floor and
set-origin handlers (index.py:158-210) on recorded floor points, the session switches through index.py's
triangulate-points and locate-objects handlers.  Stored per read: mode, timestamp, the events (name + JSON payload) and
the serial bytes; plus what a replay needs to set up the same state (poses, world matrices, filter generations).
"""
import importlib
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_harness import load_reference_index  # noqa: E402
from tests.live_util import (DIST, GOLDEN, IN_H, IN_W, K, LOCATE, encode_events, encode_serial, floor_points, make_scene,  # noqa: E402
                             render_read, session_script, timestamp, world_of)

SEED = 6
NUM_OBJECTS = 2


class Recorder:
    def __init__(self):
        self.events = []

    def emit(self, name, payload=None, **kw):
        self.events.append((name, json.loads(json.dumps(payload))))


class Serial:
    def __init__(self):
        self.lines = []

    def write(self, b):
        self.lines.append(bytes(b))


def main():
    index, helpers, cams = load_reference_index(4, K)
    kf_mod = importlib.import_module("KalmanFilter")
    now = [0.0]
    kf_mod.time = types.SimpleNamespace(time=lambda: now[0])
    helpers.time = types.SimpleNamespace(sleep=lambda s: None, time=lambda: now[0])
    sio, ser = Recorder(), Serial()
    index.socketio = sio
    cams.camera_params = [{"intrinsic_matrix": K.tolist(), "distortion_coef": DIST.tolist(), "rotation": r} for r in (0, 2, 0, 2)]
    cams.num_cameras = 4
    cams.set_socketio(sio)
    cams.set_ser(ser)
    cams.set_serialLock(__import__("threading").Lock())
    cams.set_num_objects(NUM_OBJECTS)
    cams.is_capturing_points = cams.is_triangulating_points = cams.is_locating_objects = False

    # the world matrix from the reference's handlers: acquire-floor on recorded floor points, then set-origin
    index.acquire_floor({"objectPoints": floor_points(SEED)})
    m_floor = np.array(cams.to_world_coords_matrix)
    index.set_origin({"objectPoint": world_of([0.0, 0.6, 0.0], m_floor).tolist(), "toWorldCoordsMatrix": m_floor.tolist()})
    m0 = np.array(cams.to_world_coords_matrix)
    scene = make_scene(SEED, m0)
    poses = [{"R": p["R"].tolist(), "t": p["t"].tolist()} for p in scene["poses"]]

    script = session_script()
    cur = {"frames": None}
    cams.cameras = types.SimpleNamespace(read=lambda: ([f.copy() for f in cur["frames"]], None))
    worlds = [m0]
    modes, stamps, events, serial, gens, widx = [], [], [], [], [], []
    gen = 0
    for k, (mode, dark, filt, wi) in enumerate(script):
        if mode & 2 and not cams.is_triangulating_points:
            index.live_mocap({"startOrStop": "start", "cameraPoses": poses, "toWorldCoordsMatrix": worlds[wi].tolist()})
            gen = filt
        if mode & LOCATE and not cams.is_locating_objects:
            index.start_or_stop_locating_objects({"startOrStop": "start"})
            cams.drone_armed = [True, False]
        if wi == 1 and len(worlds) == 1:
            # set-origin moves the origin; then triangulation is stopped and started again: a new filter
            index.set_origin({"objectPoint": world_of([0.1, 0.6, -0.05], m0).tolist(), "toWorldCoordsMatrix": m0.tolist()})
            worlds.append(np.array(cams.to_world_coords_matrix))
            index.live_mocap({"startOrStop": "stop", "cameraPoses": poses, "toWorldCoordsMatrix": worlds[1].tolist()})
            cams.is_capturing_points = True        # stop_trangulating_points also stops capturing; the UI's start restores it
            index.live_mocap({"startOrStop": "start", "cameraPoses": poses, "toWorldCoordsMatrix": worlds[1].tolist()})
            gen = filt
        if not mode & 2:
            cams.is_capturing_points = True
        cur["frames"] = list(render_read(scene, k, dark))
        now[0] = timestamp(k)
        sio.events, ser.lines = [], []
        cams._camera_read()
        modes.append(mode); stamps.append(now[0]); gens.append(gen); widx.append(wi)
        events.append(encode_events(sio.events)); serial.append(encode_serial(ser.lines))
    loc = [json.loads(e) for m, e in zip(modes, events) if m & LOCATE]
    both = sum(1 for e in loc if e and {o["droneIndex"] for o in e[0][1]["objects"]} >= {0, 1})
    lines = sum(len(json.loads(s)) for s in serial)
    print(f"live_loop: {len(script)} reads, {len(loc)} locating, {both} find both drones, {lines} serial lines")
    assert both >= 0.75 * len(loc), both
    assert lines > 0
    np.savez_compressed(GOLDEN, seed=SEED, num_objects=NUM_OBJECTS, mode=np.array(modes, np.int32), t=np.array(stamps),
                        dark=np.array([d for _, d, _, _ in script]), filter_gen=np.array(gens, np.int32),
                        world_index=np.array(widx, np.int32), worlds=np.stack(worlds), R=np.stack([p["R"] for p in scene["poses"]]),
                        tvec=np.stack([p["t"] for p in scene["poses"]]), rotations=np.array(scene["rotations"], np.int32),
                        drone_armed=np.array([1, 0], np.uint8), events=np.array(events), serial=np.array(serial),
                        in_size=np.array([IN_W, IN_H]))


if __name__ == "__main__":
    main()

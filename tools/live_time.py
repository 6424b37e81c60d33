"""Wall time per read of the live loop, 4 cameras at 320 x 240 in locate mode, three ways:
  (a) the oracle chain on the CPU (cv2 preprocessing, find_dot, matcher, world transform, locate_objects, Kalman filter);
  (b) the per-stage drop-ins (what install_into(helpers, tracker=True) gives _camera_read): cv2 preprocessing, then
      api.find_dot per camera, api.find_point_correspondance_and_object_points, the Python world transform,
      api.locate_objects and api.KalmanFilter.predict_location;
  (c) api.camera_read (install_into(helpers, live=True));
then the device time of one read from CUDA events and the replay rate of MocapContext.live at B = 1000 reads.

    python tools/live_time.py [--reads 300] [--out live_time.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pct(ts):
    ts = np.asarray(ts) * 1e3
    return {"p50_ms": float(np.percentile(ts, 50)), "p99_ms": float(np.percentile(ts, 99))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import importlib
    api = importlib.import_module("low-cost-mocap_b200.api")
    from oracle.ref_port import RefPort
    from tests.live_util import (CAPTURE, DIST, K, LOCATE, TRIANGULATE, StandinCameras, load_golden, make_scene, oracle_read,
                                 render_read, timestamp, world_of)
    from tests.track_util import OracleKalmanFilter
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    g = load_golden()
    M = g["worlds"][0]
    scene = make_scene(6, M)
    N = args.reads
    raws = [render_read(scene, k) for k in range(N)]
    FULL = CAPTURE | TRIANGULATE | LOCATE
    res = {"gpu": gpu, "reads": N}

    # (a) oracle chain
    port = RefPort([K] * 4)
    now = [0.0]
    kf = OracleKalmanFilter(2, lambda: now[0])
    ta = []
    for k in range(N):
        now[0] = timestamp(k)
        t0 = time.perf_counter()
        oracle_read(port, scene, raws[k], FULL, M, kf, now)
        ta.append(time.perf_counter() - t0)
    res["a_oracle_cpu"] = pct(ta)

    # (b) per-stage drop-ins
    session = api.MocapSession([K] * 4, 320, 320)
    # find_dot's single-camera context first: a context created later sets the kernels' shared-memory limits
    api.find_dot(port.preprocess(raws[0][0], 0, DIST, scene["rotations"][0]), session)
    kfb = api.KalmanFilter(2, session, clock=lambda: now[0])
    poses = scene["poses"]
    tb = []
    for k in range(N + 20):
        now[0] = timestamp(k)
        t0 = time.perf_counter()
        frames = [port.preprocess(raws[k % N][c], c, DIST, scene["rotations"][c]) for c in range(4)]
        pts = []
        for c in range(4):
            frames[c], p = api.find_dot(frames[c], session)
            pts.append(p)
        if any(p[0] != [None, None] for p in pts):
            err, obj, _ = api.find_point_correspondance_and_object_points(pts, poses, frames, session)
            obj = np.array([world_of(p, M) for p in obj])
            objects = api.locate_objects(obj, err, session)
            kfb.predict_location(objects)
        if k >= 20:
            tb.append(time.perf_counter() - t0)
    res["b_stage_dropins"] = pct(tb)

    # (c) camera_read
    cams = StandinCameras(g, scene)
    cams.set_read(len(g["mode"]) - 1)
    tc = []
    for k in range(N + 20):
        cams.frames = list(raws[k % N])
        cams.events, cams.lines = [], []
        t0 = time.perf_counter()
        api.camera_read(cams, session, clock=lambda k=k: timestamp(k))
        if k >= 20:
            tc.append(time.perf_counter() - t0)
    res["c_camera_read"] = pct(tc)

    # device time of one read, and the replay rate at B = 1000
    ctx = api.MocapContext(4, 320, 320, **api.MIRROR_LIMITS)
    ctx.set_preprocess(320, 240, scene["rotations"], [K] * 4, [DIST] * 4)
    ctx.set_cameras([K] * 4, poses)
    ctx.set_world_transform(M)
    tr = ctx.tracker(2)
    dev = ctx.torch_device
    B = 1000
    raw_d = torch.from_numpy(np.stack([raws[k % N] for k in range(B)])).to(dev)
    ts_d = torch.from_numpy(np.array([timestamp(k) for k in range(B)])).to(dev)
    for _ in range(3):
        ctx.live(raw_d[:1], FULL, ts_d[:1], tr)
        ctx.live(raw_d, FULL, ts_d, tr)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    one = []
    for k in range(200):
        e0.record()
        ctx.live(raw_d[k:k + 1], FULL, ts_d[k:k + 1], tr)
        e1.record()
        e1.synchronize()
        one.append(e0.elapsed_time(e1))
    res["device_one_read_ms"] = {"p50": float(np.percentile(one, 50)), "p99": float(np.percentile(one, 99))}
    rates = []
    for _ in range(5):
        e0.record()
        ctx.live(raw_d, FULL, ts_d, tr)
        e1.record()
        e1.synchronize()
        rates.append(B / (e0.elapsed_time(e1) / 1e3))
    res["replay_reads_per_s_B1000"] = float(np.median(rates))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

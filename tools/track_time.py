#!/usr/bin/env python
"""Time of the drone tracker: both kernels of one batch (k_track_scan + k_track_lowpass, CUDA events around
MocapContext.tracker(2).track_dev over many consecutive batches of one stream) at B = 1000 and 4000 frame-sets with 2
drones; the per-call latency of the drop-in api.KalmanFilter.predict_location (a batch of one, host clock, the call
copies its result back); and beside them the per-call CPU time of the oracle (tests/track_util.OracleKalmanFilter:
the reference's cv2.KalmanFilter + lfilter code path) on the same objects.  Prints one JSON document (GPU name and
power limit included); --out also writes it to a file."""
import argparse, importlib, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from tests.track_util import OracleKalmanFilter, make_stream, objects_of
pkg = importlib.import_module("low-cost-mocap_b200")


def batch_ms(B, reps, warmup):
    ctx = pkg.MocapContext(2, 640, 480)
    tr = ctx.tracker(2)
    st = make_stream(B * (reps + warmup), 2, seed=B)
    loc = {k: torch.from_numpy(st[k]).cuda() for k in ("objects", "drone_index", "n")}
    ts = torch.from_numpy(st["t"]).cuda()
    sl = lambda i: ({k: v[i * B:(i + 1) * B] for k, v in loc.items()}, ts[i * B:(i + 1) * B])
    for i in range(warmup):
        tr.track_dev(*sl(i))
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(warmup, warmup + reps):
        tr.track_dev(*sl(i))
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / reps


def per_call_us(fn, stream, calls):
    objs = [objects_of(stream, s) for s in range(calls)]
    t0 = time.perf_counter()
    for s in range(calls):
        fn(s, objs[s])
    return 1e6 * (time.perf_counter() - t0) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--out")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)}
    for B in (1000, 4000):
        ms = batch_ms(B, a.reps, 3)
        res[f"batch_ms_B{B}"] = round(ms, 4)
        res[f"us_per_frame_set_B{B}"] = round(1e3 * ms / B, 4)
    st = make_stream(a.calls + 100, 2, seed=7)
    now = [0.0]
    kf = pkg.KalmanFilter(2, session=pkg.MocapSession([np.eye(3)] * 2), clock=lambda: now[0])
    ok = OracleKalmanFilter(2, lambda: now[0])

    def step(f):
        def run(s, objs):
            now[0] = float(st["t"][s])
            f(objs)
        return run
    for s in range(100):                       # warm-up of both
        now[0] = float(st["t"][s]); kf.predict_location(objects_of(st, s)); ok.predict_location(objects_of(st, s))
    res["drop_in_us_per_call"] = round(per_call_us(step(kf.predict_location), st, a.calls), 1)
    now[0] = 0.0
    ok = OracleKalmanFilter(2, lambda: now[0])
    res["oracle_cpu_us_per_call"] = round(per_call_us(step(ok.predict_location), st, a.calls), 1)
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()

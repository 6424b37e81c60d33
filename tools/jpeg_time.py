"""The camera stream's JPEG on the device, timed, 4 cameras at 320 x 240 in locate mode (the golden scene's frames):
  (a) wall time per read of mocap_live_jpeg_host (MocapContext.live_host(jpeg=True)), against
  (b) mocap_live_host with the frames copied back, np.hstack and cv2.imencode('.jpg') -- the stream as index.py:55-56
      does it after install_into(helpers, live=True);
the two alternated read by read, after warm-up; then the encoder's kernel time (CUDA events) on a batch of 1000 reads'
frames (320 x 1280 x 3 each), with the input bytes per second.  Prints the card and its power limit from the same run.

    python tools/jpeg_time.py [--reads 1000] [--out jpeg_time.json]
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
    return {"p50_ms": float(np.percentile(ts, 50)), "p99_ms": float(np.percentile(ts, 99)), "n": int(ts.size)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    import importlib
    api = importlib.import_module("low-cost-mocap_b200.api")
    from tests.live_util import CAPTURE, DIST, K, LOCATE, TRIANGULATE, golden_scene, load_golden, render_read, timestamp
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    g = load_golden()
    scene = golden_scene(g)
    M = g["worlds"][0]
    FULL = CAPTURE | TRIANGULATE | LOCATE
    n_raw = len(g["mode"])
    raws = [render_read(scene, k, bool(g["dark"][k])) for k in range(n_raw)]
    res = {"gpu": gpu, "reads": args.reads, "cv2": cv2.__version__}

    def make():
        c = api.MocapContext(4, 320, 320, **api.MIRROR_LIMITS)
        c.set_preprocess(320, 240, scene["rotations"], [K] * 4, [DIST] * 4)
        c.set_cameras([K] * 4, scene["poses"])
        c.set_world_transform(M)
        return c, c.tracker(2)
    a, ta = make()
    b, tb = make()
    stride = 1 << 20
    warm, N = 50, args.reads
    t_a, t_b, sizes = [], [], []
    for k in range(warm + N):
        raw = raws[k % n_raw][None]
        ts = [timestamp(k)]
        t0 = time.perf_counter()
        ra = a.live_host(raw, FULL, ts, ta, jpeg=True, jpeg_stride=stride)
        t1 = time.perf_counter()
        rb = b.live_host(raw, FULL, ts, tb, want_frames=True)
        jb = cv2.imencode(".jpg", np.hstack(list(rb["frames"][0])))[1]
        t2 = time.perf_counter()
        if k >= warm:
            t_a.append(t1 - t0)
            t_b.append(t2 - t1)
            sizes.append(int(ra["jpeg_len"][0]))
        if k % 97 == 0:
            assert np.array_equal(ra["jpeg"][0, :ra["jpeg_len"][0]], jb), k
    res["a_live_jpeg_host"] = pct(t_a)
    res["b_live_host_hstack_cv2"] = pct(t_b)
    res["jpeg_bytes_mean"] = float(np.mean(sizes))

    # the encoder alone on 1000 reads' frames
    dev = a.torch_device
    B = 1000
    raw_d = torch.from_numpy(np.stack([raws[k % n_raw] for k in range(B)])).to(dev)
    frames = a.live(raw_d, CAPTURE, want_frames=True)["frames"]
    out = torch.empty((B, 256 << 10), dtype=torch.uint8, device=dev)
    ln = torch.empty((B,), dtype=torch.int32, device=dev)
    import ctypes
    lib = a.lib

    def enc():
        a.use_current_stream()
        st = lib.mocap_encode_jpeg_dev(a.h, ctypes.c_void_p(frames.data_ptr()), B, 4, 320, 320, 95, ctypes.c_void_p(out.data_ptr()),
                                       out.shape[1], ctypes.c_void_p(ln.data_ptr()))
        assert st == 0
    for _ in range(3):
        enc()
    torch.cuda.synchronize()
    assert int(ln.min()) > 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(10):
        e0.record()
        enc()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    t = float(np.median(ms))
    in_bytes = B * 4 * 320 * 320 * 3
    res["encode_B1000_ms"] = {"median": t, "min": float(np.min(ms)), "max": float(np.max(ms))}
    res["encode_input_GB_per_s"] = in_bytes / (t / 1e3) / 1e9
    res["encode_images_per_s"] = B / (t / 1e3)
    print(json.dumps(res, indent=1))
    if args.out:
        d = os.path.dirname(args.out)
        if d:
            os.makedirs(d, exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

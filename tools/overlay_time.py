"""Time the detection overlay adds to a live read (MocapContext.set_overlay): ctx.live in capture mode and in
capture + triangulate mode (the epipolar lines) with the processed frames, overlay off and on alternated, CUDA events
around many calls, at 4 cameras x 320 x 320 and at 8.
Prints one JSON line per shape with the GPU's name and power limit.  Needs the H100; there is no CPU fallback.

    python tools/overlay_time.py [--reps 200] [--batches 1,64]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tests.live_util import CAPTURE, DIST, IN_H, IN_W, K, TRIANGULATE, make_scene, render_read  # noqa: E402

api = importlib.import_module("low-cost-mocap_b200.api")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def time_calls(ctx, raw, mode, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        ctx.live(raw, mode, want_frames=True)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--batches", default="1,64")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "overlay_time needs the GPU"
    info = gpu_info()
    for C in (4, 8):
        scene = make_scene(3, np.eye(4), C=C, rotations=[0, 2] * (C // 2))
        ctx = api.MocapContext(C, 320, 320, **api.MIRROR_LIMITS)
        ctx.set_preprocess(IN_W, IN_H, scene["rotations"], [K] * C, [DIST] * C)
        ctx.set_cameras([K] * C, scene["poses"])
        for mode, B in ((m, int(b)) for m in (CAPTURE, CAPTURE | TRIANGULATE) for b in args.batches.split(",")):
            raw = torch.from_numpy(np.stack([render_read(scene, k) for k in range(B)])).to(ctx.torch_device)
            ms = {False: [], True: []}
            for on in (False, True) * 2:                        # warm-up of both shapes
                ctx.set_overlay(on)
                time_calls(ctx, raw, mode, 5)
            for rnd in range(6):                                # alternated rounds
                for on in ((False, True) if rnd % 2 == 0 else (True, False)):
                    ctx.set_overlay(on)
                    ms[on].append(time_calls(ctx, raw, mode, args.reps))
            off, on_ = float(np.median(ms[False])), float(np.median(ms[True]))
            print(json.dumps({"gpu": info, "cameras": C, "size": 320, "mode": "capture+triangulate" if mode & TRIANGULATE else "capture",
                              "reads_per_call": B,
                              "ms_per_read_off": off / B, "ms_per_read_on": on_ / B, "added_ms_per_read": (on_ - off) / B,
                              "spread_off_ms": [min(ms[False]) / B, max(ms[False]) / B],
                              "spread_on_ms": [min(ms[True]) / B, max(ms[True]) / B]}), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()

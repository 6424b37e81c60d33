"""Time of S1's full-size reduction (k_blob_reduce) on holed images, with and without the whole-image window of the
RETR_TREE slow path (mocap_set_large_holes): one large ring, a frame around the whole image, a 130-px spiral
(84 turns: near the most that 4096 runs per image allow), 16 and 28 nested frames, and the same shapes at sizes the
64 x 64 window takes.  A batch holds one copy of the image per SM, so each CTA reduces one image and the kernel time
is the time of one image.  Device time from torch.profiler (CUDA activity), averaged over --reps detect calls after a warm-up.  Prints one JSON line per case and
the GPU's name and power limit.

    python tools/holes_time.py [--reps 20] [--out holes_time.json]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def cases(H=480, W=640):
    import cv2
    from tests.large_holes_util import nested_frames, spiral

    def new():
        return np.zeros((H, W), np.uint8)
    out = []
    img = new(); cv2.circle(img, (320, 240), 100, 255, 2); out.append(("ring_200px", img, True))
    img = new(); cv2.rectangle(img, (0, 0), (W - 1, H - 1), 255, 1); out.append(("frame_whole_image", img, True))
    img = new(); spiral(img, 300, 200, 429, 329); out.append(("spiral_130px_84_turns", img, True))
    img = new(); nested_frames(img, 200, 100, 16, gap=4); out.append(("nested16_129px", img, True))
    img = new(); nested_frames(img, 200, 100, 28, gap=2); out.append(("nested28_113px", img, True))
    img = new(); cv2.circle(img, (320, 240), 29, 255, 2); out.append(("ring_60px", img, False))
    img = new(); cv2.rectangle(img, (100, 100), (159, 159), 255, 1); out.append(("frame_60px", img, False))
    img = new(); spiral(img, 100, 100, 160, 160); out.append(("spiral_61px", img, False))
    img = new(); nested_frames(img, 200, 100, 15, gap=2); out.append(("nested15_61px", img, False))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from tests.util import retr_tree_blobs
    pkg = importlib.import_module("low-cost-mocap_b200")
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    rows = []
    ctxs = {}
    for on in (False, True):
        ctxs[on] = pkg.MocapContext(1, 640, 480, max_blobs=64, max_segments=4096)
        if on:
            ctxs[on].set_large_holes(True)
    for name, img, large in cases():
        items = retr_tree_blobs(img > 0)[0]
        batch = torch.from_numpy(np.repeat(img[None], n_sm, axis=0)).cuda()
        for on in ((True,) if large else (False, True)):
            ctx = ctxs[on]
            d = ctx.detect(batch, want_moments=True)
            torch.cuda.synchronize()
            flags = int(d["flags"][0])
            n = int(d["n"][0])
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    ctx.detect(batch, want_moments=True)
                torch.cuda.synchronize()
            us = [e.device_time_total / e.count for e in prof.key_averages() if e.key.startswith("void k_blob_reduce<")]
            row = dict(case=name, window="whole-image" if on else "64x64", blob_reduce_us=round(us[0], 2) if us else None,
                       images_per_launch=n_sm, contours=n, cv2_contours=len(items), flags=flags, gpu=smi)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""S4: how does one solve scale with the number of CTAs (MOCAP_BA_GRID), and do two half-grid solves of two contexts on two
streams run side by side?  8 cameras x 18 800 points (the config-3 solve).  Last, the four solves of a config-3 step three
ways, alternated in one run: in turn on one context, four contexts x SMs/4 CTAs on four streams, and one batched launch
(mocap_bundle_adjust_batch_dev) of 4 x SMs/4."""
import importlib, json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth
C, F = 8, 18800
obs_obj, poses, K, pts = synth.make_tracks(C, F, seed=9, missing_frac=0.1)
start = synth.perturb_poses(poses, seed=10)
obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
d_obs, d_mask = torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda()
R0 = torch.from_numpy(np.stack([p["R"] for p in start])).cuda().contiguous()
t0 = torch.from_numpy(np.stack([np.asarray(p["t"]).reshape(3) for p in start])).cuda().contiguous()
res = {}


def make(grid):
    os.environ["MOCAP_BA_GRID"] = str(grid)
    ctx = pkg.MocapContext(C)
    ctx.set_cameras([K] * C, start)
    return ctx


def timed(fn, reps=5):
    ms = []
    for _ in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms[1:]))


SMS = torch.cuda.get_device_properties(0).multi_processor_count
for grid in (SMS // 4, SMS // 2, 3 * SMS // 4, SMS):
    ctx = make(grid)
    Rs = [R0.clone() for _ in range(4)]; ts = [t0.clone() for _ in range(4)]
    def four():
        for i in range(4):
            Rs[i].copy_(R0); ts[i].copy_(t0)
            ctx.bundle_adjust_dev(d_obs, d_mask, Rs[i], ts[i])
    ms4 = timed(four)
    rep = ctx.decode_ba_report(ctx.bundle_adjust_dev(d_obs, d_mask, Rs[0].copy_(R0), ts[0].copy_(t0)))
    torch.cuda.synchronize()
    res[f"grid {grid}: 4 solves one after the other"] = {"ms": ms4, "per_solve": ms4 / 4, "cost_final": rep["cost_final"], "status": rep["status"]}
    print(grid, ms4 / 4, rep["cost_final"], flush=True)
    del ctx

for k in (2, 3):
    grid = SMS // k
    ctxs = [make(grid) for _ in range(k)]
    streams = [torch.cuda.Stream() for _ in range(k)]
    Rs = [R0.clone() for _ in range(12)]; ts = [t0.clone() for _ in range(12)]
    n_solves = 4 if k == 2 else 6
    def side_by_side():
        cur = torch.cuda.current_stream()
        for s in streams: s.wait_stream(cur)
        for i in range(n_solves):
            with torch.cuda.stream(streams[i % k]):
                Rs[i].copy_(R0); ts[i].copy_(t0)
                ctxs[i % k].bundle_adjust_dev(d_obs, d_mask, Rs[i], ts[i])
        for s in streams: cur.wait_stream(s)
    ms = timed(side_by_side)
    res[f"{k} contexts x grid {grid} on {k} streams: {n_solves} solves"] = {"ms": ms, "per_solve": ms / n_solves,
                                                                           "poses_equal_across_contexts": bool(torch.equal(Rs[0], Rs[1]) and torch.equal(ts[0], ts[1]))}
    print(k, grid, ms / n_solves, flush=True)
    del ctxs
# config-3: four solves three ways, alternated
os.environ.pop("MOCAP_BA_GRID", None)
one = pkg.MocapContext(C); one.set_cameras([K] * C, start)
quad = [pkg.MocapContext(C) for _ in range(4)]
for c_ in quad:
    c_.set_cameras([K] * C, start); c_.set_ba_grid(SMS // 4)
bat = pkg.MocapContext(C); bat.set_cameras([K] * C, start); bat.set_ba_grid(4 * (SMS // 4))
streams = [torch.cuda.Stream() for _ in range(4)]
Rs = [R0.clone() for _ in range(4)]; ts = [t0.clone() for _ in range(4)]
probs = [{"obs": d_obs, "mask": d_mask, "R": Rs[i], "t": ts[i]} for i in range(4)]
def in_turn():
    for i in range(4):
        Rs[i].copy_(R0); ts[i].copy_(t0)
        one.bundle_adjust_dev(d_obs, d_mask, Rs[i], ts[i])
def four_contexts():
    cur = torch.cuda.current_stream()
    for s in streams: s.wait_stream(cur)
    for i in range(4):
        with torch.cuda.stream(streams[i]):
            Rs[i].copy_(R0); ts[i].copy_(t0)
            quad[i].bundle_adjust_dev(d_obs, d_mask, Rs[i], ts[i])
    for s in streams: cur.wait_stream(s)
def batched():
    for i in range(4):
        Rs[i].copy_(R0); ts[i].copy_(t0)
    bat.bundle_adjust_batch_dev(probs)
legs = {"4 solves in turn, one context, grid %d" % SMS: in_turn,
        "4 contexts x grid %d on 4 streams" % (SMS // 4): four_contexts,
        "1 batched launch of 4 x %d" % (SMS // 4): batched}
ms = {k: [] for k in legs}
for k, fn in legs.items():                                   # warm-up
    timed(fn, reps=1)
for _ in range(10):
    for k, fn in legs.items():
        ms[k].append(timed(fn, reps=1))
for k in legs:
    res["config-3 step, " + k] = {"ms_median": float(np.median(ms[k])), "ms_min": float(np.min(ms[k])), "ms_max": float(np.max(ms[k]))}
    print(k, np.median(ms[k]), np.min(ms[k]), np.max(ms[k]), flush=True)
import subprocess
res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True).stdout.strip()
print(res["gpu"])
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "profiles", "ba_grid_probe.json"), "w"), indent=1)

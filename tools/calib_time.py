#!/usr/bin/env python
"""Wall time of the cold-start calibration: calibrate_init with the 8-point and the RANSAC estimator, the RANSAC stage
alone (fundamental_ransac: three kernels for all pairs), and calculate_camera_poses(robust=True), at 4, 8 and 16
cameras x 6400 points (16 x 6400 is BASELINE config 5: 64 markers x 100 frames), 10 % of each camera's observations
mismatched; calculate_camera_poses(robust=True, reject_px=REJECT_PX) beside it, and at 16 cameras the screen kernel
alone (CUDA events over many launches, each with its stats reset) and one bundle-adjustment solve of the screened
tracks.  The pose-graph initialiser (calibrate_init(method="graph"), calculate_camera_poses(init="graph", reject_px))
beside the chain, and at 16 cameras its device time per kernel (torch.profiler over one call).  Beside them the CPU time of cv2.findFundamentalMat(FM_RANSAC, 1 px, 0.99999) over the same pairs, the
reference handler's estimator.  Every entry point synchronises before it returns, so a host clock around each call
measures it; the variants are alternated and medians reported.  Prints one JSON document (GPU name and power limit
included); --out also writes it to a file."""
import argparse, importlib, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cv2
import torch
pkg = importlib.import_module("low-cost-mocap_b200")
synth = pkg.synth
REJECT_PX = 8.0      # the value INTEGRATION.md recommends for calculate_camera_poses(reject_px=...)


def tracks(C, n, frac=0.1, seed=3):
    obs_obj, poses, K, _ = synth.make_tracks(C, n, seed=seed, missing_frac=0.1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    rng = np.random.default_rng(seed + 1)
    for c in range(C):
        seen = np.flatnonzero(mask[:, c])
        pick = rng.choice(seen, int(round(frac * len(seen))), replace=False)
        obs[pick, c] = np.floor(rng.uniform([0, 0], [synth.WIDTH, synth.HEIGHT], size=(len(pick), 2)))
    image_points = [[[int(obs[f, c, 0]), int(obs[f, c, 1])] if mask[f, c] else [None, None] for c in range(C)] for f in range(n)]
    return obs, mask, image_points, K


def cv2_pairs(obs, mask):
    for c in range(obs.shape[1] - 1):
        both = (mask[:, c] & mask[:, c + 1]).astype(bool)
        cv2.findFundamentalMat(obs[both, c].astype(np.float32), obs[both, c + 1].astype(np.float32), cv2.FM_RANSAC, 1, 0.99999)


def screen_kernel_ms(obs, mask, K, launches=200, solves=10):
    """Device time of k_screen_observations alone (CUDA events around `launches` back-to-back launches) at the poses
    of the robust chain's first bundle adjustment, and of one k_ba_solve from the same poses for scale."""
    C = obs.shape[1]
    ctx = pkg.MocapContext(C)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    chain = ctx.calibrate_init(obs, mask, method="ransac")[0]
    ctx.set_cameras([K] * C, chain)
    first, _ = ctx.bundle_adjust(obs, mask, chain)
    dev = ctx.torch_device
    d_obs, d_mask = torch.from_numpy(obs).to(dev), torch.from_numpy(mask).to(dev)
    R0 = torch.from_numpy(np.stack([p["R"] for p in first])).to(dev)
    t0 = torch.from_numpy(np.stack([p["t"] for p in first])).to(dev)
    out = ctx.screen_observations_dev(d_obs, d_mask, R0, t0, REJECT_PX)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        ctx.screen_observations_dev(d_obs, d_mask, R0, t0, REJECT_PX, out=out)
    e1.record()
    torch.cuda.synchronize()
    screen = e0.elapsed_time(e1) / launches
    R, t = R0.clone(), t0.clone()
    solve = []
    for _ in range(solves):
        R.copy_(R0); t.copy_(t0)
        e0.record()
        ctx.bundle_adjust_dev(d_obs, out["mask"], R, t)
        e1.record()
        torch.cuda.synchronize()
        solve.append(e0.elapsed_time(e1))
    return {"screen_kernel_ms": screen, "launches": launches, "stats": out["stats"].cpu().tolist(),
            "ba_solve_after_screen_ms_median": float(np.median(solve))}


def graph_kernel_ms(obs, mask, K, calls=3):
    """Device time per kernel of calibrate_init(method="graph"), summed over its launches and averaged over `calls`
    calls (torch.profiler, CUDA activity), with the number of launches per call."""
    from torch.profiler import ProfilerActivity, profile
    C = obs.shape[1]
    ctx = pkg.MocapContext(C)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    ctx.calibrate_init(obs, mask, method="graph")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ctx.calibrate_init(obs, mask, method="graph")
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.key.startswith("k_"):
            dev_us = getattr(ev, "device_time_total", None)
            if dev_us is None:
                dev_us = ev.cuda_time_total
            out[ev.key] = {"ms_per_call": dev_us / 1e3 / calls, "launches_per_call": ev.count / calls}
    return out


def case(C, n, reps):
    obs, mask, image_points, K = tracks(C, n)
    ctx = pkg.MocapContext(C)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    session = pkg.MocapSession([K] * C)
    variants = {
        "calibrate_init_8point": lambda: ctx.calibrate_init(obs, mask),
        "calibrate_init_ransac": lambda: ctx.calibrate_init(obs, mask, method="ransac"),
        "ransac_stage": lambda: ctx.fundamental_ransac(obs, mask),
        "calculate_camera_poses_robust": lambda: pkg.calculate_camera_poses(image_points, session=session, robust=True),
        "calculate_camera_poses_robust_screened": lambda: pkg.calculate_camera_poses(image_points, session=session, robust=True,
                                                                                      reject_px=REJECT_PX),
        "calibrate_init_graph": lambda: ctx.calibrate_init(obs, mask, method="graph"),
        "calculate_camera_poses_graph_screened": lambda: pkg.calculate_camera_poses(image_points, session=session, init="graph",
                                                                                     reject_px=REJECT_PX),
        "cv2_fm_ransac_cpu": lambda: cv2_pairs(obs, mask),
    }
    ms = {k: [] for k in variants}
    for k, fn in variants.items():      # warm-up: module load, scratch allocation
        fn()
    torch.cuda.synchronize()
    for _ in range(reps):
        for k, fn in variants.items():
            t0 = time.perf_counter()
            fn()
            ms[k].append((time.perf_counter() - t0) * 1e3)
    return {"cameras": C, "points": n, "reps": reps, "reject_px": REJECT_PX,
            **{k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))} for k, v in ms.items()},
            **({"screen": screen_kernel_ms(obs, mask, K), "graph_kernels": graph_kernel_ms(obs, mask, K)} if C == 16 else {})}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("calib_time.py needs an H100")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    doc = {"gpu": q.stdout.strip(), "cases": [case(C, 6400, a.reps) for C in (4, 8, 16)]}
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)

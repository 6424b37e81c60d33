#!/usr/bin/env python
"""What threshold should calculate_camera_poses(reject_px=...) use?  On contaminated calibration tracks (a fraction
of each camera's observations replaced by uniform random pixels), at the poses the FIRST screen sees -- the bundle
adjustment of the robust chain, on every view or on the views that are RANSAC inliers with a neighbouring camera (what
calculate_camera_poses uses) -- this measures:
  * the pixel error of every good view against the point triangulated from its track's good views (percentiles), and
    of every mismatched view against that point (low percentiles);
  * for a range of thresholds, the share of good and of mismatched views the screen drops there, and after
    bundle_adjust_screened(rounds=2) the share dropped at the final poses and the largest point error after a
    similarity alignment (the bar of the clean-track test is 0.03).
Prints one JSON document with the GPU's name and power limit."""
import argparse, importlib, json, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from tests.screen_util import contaminated_tracks
pkg = importlib.import_module("low-cost-mocap_b200")

THRESHOLDS = (1.5, 2.0, 3.0, 4.0, 6.0, 8.0, 12.0, 16.0, 24.0)


def view_errors(obs, clean, poses, K):
    """pixel error of every observation against the DLT point of its track's good views, at `poses`"""
    C = obs.shape[1]
    ctx = pkg.MocapContext(C)
    ctx.set_cameras([K] * C, poses)
    keep = clean.sum(axis=1) >= 2
    X, _, _ = ctx.triangulate(obs[keep], clean[keep])
    err = np.full(clean.shape, np.nan)
    for c in range(C):
        pc = X @ np.asarray(poses[c]["R"]).T + np.asarray(poses[c]["t"]).reshape(1, 3)
        uv = pc @ K.T
        err[keep, c] = np.hypot(*(obs[keep, c] - uv[:, :2] / uv[:, 2:3]).T)
    return err


def aligned_error(ctx, obs, clean, pts, rig, K):
    C = obs.shape[1]
    keep = clean.sum(axis=1) >= 2
    ctx.set_cameras([K] * C, rig)
    X, _, _ = ctx.triangulate(obs[keep], clean[keep])
    A = X - X.mean(0); Bm = pts[keep] - pts[keep].mean(0)
    A *= np.linalg.norm(Bm) / np.linalg.norm(A)
    U, _, Vt = np.linalg.svd(A.T @ Bm)
    return float(np.abs(A @ (U @ Vt) - Bm).max())


def ransac_first_mask(mask, inl):
    """the views that are RANSAC inliers with a neighbouring camera (what calculate_camera_poses' first solve sees)"""
    inl = inl.astype(bool)
    near = np.zeros(mask.shape, dtype=bool)
    near[:, :-1] |= inl
    near[:, 1:] |= inl
    return (mask.astype(bool) & near).astype(np.uint8)


def probe(C, n, frac, seed):
    obs, mask, _, bad, poses, K, pts = contaminated_tracks(C, n, frac, seed)
    seen = mask.astype(bool)
    clean = (seen & ~bad).astype(np.uint8)
    ctx = pkg.MocapContext(C)
    ctx.set_cameras([K] * C, [{"R": np.eye(3), "t": np.zeros(3)}] * C)
    chain, _, _, inl = ctx.calibrate_init(obs, mask, method="ransac")
    out = {"cameras": C, "points": n, "mismatched": frac, "seed": seed}
    for name, first_mask in (("first_solve_all_views", mask), ("first_solve_ransac_inliers", ransac_first_mask(mask, inl))):
        ctx.set_cameras([K] * C, chain)
        first, _ = ctx.bundle_adjust(obs, first_mask, chain)
        err = view_errors(obs, clean, first, K)
        good_e, bad_e = err[clean.astype(bool)], err[seen & bad]
        good_e, bad_e = good_e[np.isfinite(good_e)], bad_e[np.isfinite(bad_e)]
        r = {"first_mask_good_views": float((first_mask.astype(bool) & clean.astype(bool)).sum() / clean.sum()),
             "first_mask_mismatched_views": float((first_mask.astype(bool) & bad).sum() / max(1, bad.sum())),
             "point_error_after_first_solve": aligned_error(ctx, obs, clean, pts, first, K),
             "good_view_error_px_at_first_screen": {q: float(np.percentile(good_e, p)) for q, p in
                                                   (("p50", 50), ("p99", 99), ("p99.9", 99.9), ("max", 100))},
             "mismatched_view_error_px_at_first_screen": {q: float(np.percentile(bad_e, p)) if len(bad_e) else None for q, p in
                                                         (("min", 0), ("p0.1", 0.1), ("p1", 1), ("p5", 5))},
             "thresholds": []}
        for thr in THRESHOLDS:
            m1 = ctx.screen_observations(obs, mask, first, thr)["mask"].astype(bool)
            ctx.set_cameras([K] * C, chain)
            final, rep, kept = ctx.bundle_adjust_screened(obs, mask, chain, thr, rounds=2, first_mask=first_mask)
            kept = kept.astype(bool)
            r["thresholds"].append({
                "px": thr,
                "first_screen_good_dropped": float((clean.astype(bool) & ~m1).sum() / clean.sum()),
                "first_screen_mismatched_dropped": float((bad & ~m1).sum() / max(1, bad.sum())),
                "final_good_dropped": float((clean.astype(bool) & ~kept).sum() / clean.sum()),
                "final_mismatched_dropped": float((bad & ~kept).sum() / max(1, bad.sum())),
                "final_point_error": aligned_error(ctx, obs, clean, pts, final, K),
                "final_cost": rep["cost_final"]})
        out[name] = r
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("screen_threshold_probe.py needs an H100")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    cases = [(8, 300, f, 108) for f in (0.0, 0.1, 0.2, 0.3, 0.4)] + [(4, 300, 0.2, 104), (16, 300, 0.2, 116), (16, 6400, 0.1, 3)]
    doc = {"gpu": q.stdout.strip(), "cases": [probe(*c) for c in cases]}
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)

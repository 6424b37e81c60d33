"""Helpers shared by the CPU and GPU tests of the per-view screen (csrc/screen.cuh) and tools/screen_threshold_probe.py:
contaminated calibration tracks, the host build's screen and the inputs both test tiers use."""
import importlib

import numpy as np

from tests.hostbuild import ptr

synth = importlib.import_module("low-cost-mocap_b200.synth")


def contaminated_tracks(C, n, frac, seed):
    """synth.make_tracks with, in each camera, a fraction `frac` of its observations replaced by uniform random
    pixels (a stray reflection recorded instead of the marker).  Returns (obs, mask, obs_obj, bad [n, C], poses, K,
    true points).  The same tracks as tests/test_gpu_calib_ransac.py's helper of that name."""
    obs_obj, poses, K, pts = synth.make_tracks(C, n, seed=seed, missing_frac=0.1)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    rng = np.random.default_rng(seed + 7919)
    bad = np.zeros(mask.shape, dtype=bool)
    for c in range(C):
        seen = np.flatnonzero(mask[:, c])
        pick = rng.choice(seen, int(round(frac * len(seen))), replace=False)
        bad[pick, c] = True
        obs[pick, c] = np.floor(rng.uniform([0, 0], [synth.WIDTH, synth.HEIGHT], size=(len(pick), 2)))
    out = np.empty(obs_obj.shape, dtype=object)
    for f in range(n):
        for c in range(C):
            out[f, c] = [int(obs[f, c, 0]), int(obs[f, c, 1])] if mask[f, c] else [None, None]
    return obs, mask, out, bad, poses, K, pts


def poses_arrays(poses):
    R = np.ascontiguousarray(np.stack([np.asarray(p["R"], dtype=np.float64).reshape(3, 3) for p in poses]))
    t = np.ascontiguousarray(np.stack([np.asarray(p["t"], dtype=np.float64).reshape(3) for p in poses]))
    return R, t


def host_screen(lib, obs, mask, Ks, poses, thr):
    """The host build of the screen: (mask_out uint8 [n, C], stats int32 [4])."""
    obs = np.ascontiguousarray(obs, dtype=np.float64)
    mask = np.ascontiguousarray(mask, dtype=np.uint8)
    n, C = mask.shape
    K = np.ascontiguousarray(np.stack([np.asarray(k, dtype=np.float64).reshape(3, 3) for k in Ks]))
    R, t = poses_arrays(poses)
    out = np.zeros_like(mask)
    stats = np.zeros(4, dtype=np.int32)
    lib.hc_screen(ptr(obs), ptr(mask), n, C, ptr(K), ptr(R), ptr(t), float(thr), ptr(out), ptr(stats))
    return out, stats


def screen_inputs():
    """The inputs both tiers of the screen's tests use: contaminated_tracks at 4 / 8 / 16 cameras and 0-40 %
    mismatched views, at the true poses and at synth.perturb_poses of them.  Yields (name, obs, mask, K, poses)."""
    for C, n in ((4, 120), (8, 80), (16, 40)):
        for frac in (0.0, 0.1, 0.2, 0.3, 0.4):
            obs, mask, _, _, poses, K, _ = contaminated_tracks(C, n, frac, seed=300 + C + int(100 * frac))
            yield f"C{C}_f{frac}_true", obs, mask, K, poses
            yield f"C{C}_f{frac}_perturbed", obs, mask, K, synth.perturb_poses(poses, seed=C, rot_sigma=0.003, t_sigma=0.005)

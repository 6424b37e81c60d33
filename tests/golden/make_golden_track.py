"""Writes tests/golden/track_live.npz by running the REAL reference's KalmanFilter (computer_code/api/KalmanFilter.py
and LowPassFilter.py of a jyjblrd/Low-Cost-Mocap checkout, imported unmodified) on a seeded stream of located
frame-sets, with its clock replaced by the stream's timestamps:

    MOCAP_REFERENCE_DIR=<checkout> python tests/golden/make_golden_track.py

The stream (tests/track_util.make_stream): 1200 calls at about 90 Hz with +-30 % jitter from an epoch-sized
timestamp, 2 drones with drop-outs and a 100-call absence of drone 1, clutter objects with a wrong droneIndex,
frame-sets without objects and one reset().  The inputs are stored in the layout mocap_locate_objects_dev writes;
the outputs are copied per call (the reference's "pos" is a live view into its filter state).
"""
import importlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_harness import REFERENCE_API_DIR, reference_available  # noqa: E402
from tests.track_util import GOLDEN, make_stream, objects_of, records_to_arrays  # noqa: E402

B, D = 1200, 2
RESET_AT = 900


def main():
    if not reference_available():
        raise RuntimeError(f"reference not found at {REFERENCE_API_DIR} (set MOCAP_REFERENCE_DIR to a Low-Cost-Mocap checkout)")
    if REFERENCE_API_DIR not in sys.path:
        sys.path.insert(0, REFERENCE_API_DIR)
    kf_mod = importlib.import_module("KalmanFilter")       # the reference module, unmodified
    now = [0.0]
    kf_mod.time = types.SimpleNamespace(time=lambda: now[0])   # both clock reads of a call see its timestamp
    st = make_stream(B, D, seed=2026, absence=(1, 400, 100), reset_at=RESET_AT)
    kf = kf_mod.KalmanFilter(D)
    pos = np.zeros((B, D, 3), np.float32); vel = np.zeros((B, D, 3), np.float32)
    head = np.zeros((B, D)); pres = np.zeros((B, D), np.uint8)
    for s in range(B):
        if s == RESET_AT:
            now[0] = st["reset_time"]
            kf.reset()
        now[0] = float(st["t"][s])
        rec = [{k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()} for r in kf.predict_location(objects_of(st, s))]
        pos[s], vel[s], head[s], pres[s] = records_to_arrays(rec, D)
    np.savez_compressed(GOLDEN, objects=st["objects"], drone_index=st["drone_index"], n=st["n"], t=st["t"],
                        reset_at=st["reset_at"], reset_time=st["reset_time"], num_objects=D,
                        pos=pos, vel=vel, heading=head, present=pres)
    print("track_live: calls", B, "present per drone", pres.sum(0).tolist(), "empty frame-sets", int((st["n"] == 0).sum()))


if __name__ == "__main__":
    main()

"""Writes tests/golden/locate_edge.npz by running the REAL reference's locate_objects (computer_code/api/helpers.py of
a jyjblrd/Low-Cost-Mocap checkout, imported unmodified) on the scenes of tests/locate_util.py that the locator's tests
run: every named edge scene (crowded rigs, shared markers, tolerance edges, heading folds, the drone-index edge,
non-finite rows) and a 300-scene sample of the random fuzz:

    MOCAP_REFERENCE_DIR=<checkout> python tests/golden/make_golden_locate.py

Stored per scene: the point count and, for the named scenes, the points and errors themselves; for the fuzz sample a
SHA-256 of them (the seeded builder regenerates them; the digest shows if it ever drifts).  Then the reference's
records, concatenated over the scenes: count, pos, heading, error, droneIndex.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_harness import load_reference  # noqa: E402
from tests.locate_util import GOLDEN, edge_scenes, golden_fuzz_scenes  # noqa: E402


def digest(pts, errs):
    return hashlib.sha256(pts.tobytes() + errs.tobytes()).hexdigest()


def main():
    helpers, _ = load_reference(2)
    named = edge_scenes()
    scenes = list(named.values()) + golden_fuzz_scenes()
    counts, rec, di = [], [], []
    for pts, errs in scenes:
        with np.errstate(invalid="ignore"):
            found = helpers.locate_objects(pts.copy(), errs.copy())
        counts.append(len(found))
        for o in found:
            rec.append([*o["pos"], o["heading"], o["error"]])
            di.append(o["droneIndex"])
    edge = list(named.values())
    np.savez_compressed(
        GOLDEN, names=np.array(list(named)), n_points=np.array([len(p) for p, _ in scenes], np.int32),
        edge_points=np.concatenate([p for p, _ in edge]), edge_errors=np.concatenate([e for _, e in edge]),
        fuzz_sha256=np.array([digest(p, e) for p, e in scenes[len(edge):]]),
        n_objects=np.array(counts, np.int32), records=np.array(rec, np.float64).reshape(-1, 5), drone_index=np.array(di, np.int8))
    print("locate_edge:", len(edge), "named scenes,", len(scenes) - len(edge), "fuzz scenes,", sum(counts), "objects,",
          os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    main()

"""The pose-graph cold start's arithmetic (csrc/calib_graph.cuh), compiled for the host with g++: the per-track
elimination and the per-pair cheirality equal numpy restatements, the host rotation averaging and translation stage
recover the true rig from noise-free tracks, and on a 16-camera rig where the reference's chain twists a pair the
pair-frame cheirality picks the true motion of every pair."""
import ctypes
import importlib
import os
import subprocess

import cv2
import numpy as np
import pytest

from oracle.ref_port import RefPort

synth = importlib.import_module("low-cost-mocap_b200.synth")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("calib_graph")), "libcalib_graph_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "calib_graph_host.cpp"), "-lm"])
    lib = ctypes.CDLL(out)
    lib.hc_track_block.argtypes = [P, P, P, P, ctypes.c_int, P]
    lib.hc_track_block.restype = ctypes.c_int
    lib.hc_cheirality.argtypes = [P, P, P, P] + [ctypes.c_double] * 4 + [P]
    lib.hc_cheirality.restype = ctypes.c_double
    lib.hc_motion_from_essential.argtypes = [P, P, P]
    lib.hc_motion_from_essential.restype = None
    lib.hc_rotation_average.argtypes = [ctypes.c_int, ctypes.c_int, P, P, P, P, ctypes.c_double, P, P, P]
    lib.hc_rotation_average.restype = ctypes.c_int
    lib.hc_translations.argtypes = [P, P, ctypes.c_int, ctypes.c_int, P, P, P, ctypes.c_int, ctypes.c_double, P, P]
    lib.hc_translations.restype = ctypes.c_int
    return lib


def p(a):
    return a.ctypes.data_as(P)


def c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def float_tracks(C, n=300, seed=5):
    obs_obj, poses, K, pts = synth.make_tracks(C, n, seed=seed, missing_frac=0.1, round_to_int=False)
    obs = np.array([[[0.0 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    return obs, mask, poses, K, pts


def skew(x):
    return np.array([[0, -x[2], x[1]], [x[2], 0, -x[0]], [-x[1], x[0], 0]])


def restate_block(obs, w, K, R):
    """The Schur complement of the track's point in the normal equations of sqrt(w_c) [x_c]_x (R_c X + t_c) = 0."""
    C = len(w)
    rows = []
    for c in range(C):
        if w[c] <= 0:
            continue
        x = np.linalg.solve(K, [obs[c, 0], obs[c, 1], 1.0])
        x /= np.linalg.norm(x)
        S = np.sqrt(w[c]) * skew(x)
        A = np.zeros((3, 3 + 3 * C))
        A[:, :3] = S @ R[c]
        A[:, 3 + 3 * c:6 + 3 * c] = S
        rows.append(A)
    A = np.vstack(rows)
    N = A.T @ A
    Hxx, Hxt, Htt = N[:3, :3], N[:3, 3:], N[3:, 3:]
    return Htt - Hxt.T @ np.linalg.solve(Hxx, Hxt)


@pytest.mark.parametrize("C", [4, 8, 16])
def test_track_elimination_equals_numpy(lib, C):
    obs, mask, poses, K, _ = float_tracks(C)
    Kinv = c64(np.stack([np.linalg.inv(K)] * C))
    R = c64(np.stack([p_["R"] for p_ in poses]))
    rng = np.random.default_rng(C)
    for f in range(40):
        w = c64(mask[f] * rng.uniform(0.2, 1.0, size=C))
        H = np.zeros((3 * C, 3 * C))
        ok = lib.hc_track_block(p(c64(obs[f])), p(w), p(Kinv), p(R), C, p(H))
        assert ok == (mask[f].sum() >= 2)
        if ok:
            want = restate_block(obs[f], w, K, R)
            assert np.abs(H - want).max() <= 1e-10 * max(1.0, np.abs(want).max())


def dlt(Pa, Pb, xa, xb):
    A = np.array([xa[1] * Pa[2] - Pa[1], Pa[0] - xa[0] * Pa[2], xb[1] * Pb[2] - Pb[1], Pb[0] - xb[0] * Pb[2]])
    X = np.linalg.svd(A)[2][-1]
    return X[:3] / X[3]


@pytest.mark.parametrize("C", [4, 8, 16])
def test_pair_cheirality_equals_numpy(lib, C):
    """Every candidate of E for a few pairs: front flag and triangulation angle as the restatement gives them."""
    obs, mask, poses, K, _ = float_tracks(C)
    for a, b in [(0, 1), (0, C // 2), (1, C - 1)]:
        Rab = poses[b]["R"] @ poses[a]["R"].T
        tab = poses[b]["t"] - Rab @ poses[a]["t"]
        E = c64(skew(tab) @ Rab)
        Rs, ts = np.zeros((4, 9)), np.zeros((4, 3))
        lib.hc_motion_from_essential(p(E), p(Rs), p(ts))
        both = np.flatnonzero(mask[:, a] & mask[:, b])[:30]
        for q in range(4):
            Rq, tq = Rs[q].reshape(3, 3), ts[q]
            Pa, Pb = K @ np.hstack([np.eye(3), np.zeros((3, 1))]), K @ np.hstack([Rq, tq[:, None]])
            for f in both:
                fr = ctypes.c_int(0)
                got = lib.hc_cheirality(p(c64(K)), p(c64(K)), p(c64(Rq)), p(c64(tq)), *obs[f, a], *obs[f, b], ctypes.byref(fr))
                X = dlt(Pa, Pb, obs[f, a], obs[f, b])
                cb = -Rq.T @ tq
                front = X[2] > 0 and (Rq @ X + tq)[2] > 0
                u, v = X, X - cb
                ang = np.degrees(np.arccos(np.clip(u @ v / np.linalg.norm(u) / np.linalg.norm(v), -1, 1)))
                assert bool(fr.value) == front
                assert abs(got - ang) < 1e-6


def eight_point(x1, x2):
    """Hartley-normalised 8-point F in double precision (x2^T F x1 = 0), rank 2"""
    def norm(x):
        c = x.mean(0)
        s = np.sqrt(2.0) / np.linalg.norm(x - c, axis=1).mean()
        return np.array([[s, 0, -s * c[0]], [0, s, -s * c[1]], [0, 0, 1.0]])
    T1, T2 = norm(x1), norm(x2)
    h1 = np.c_[x1, np.ones(len(x1))] @ T1.T
    h2 = np.c_[x2, np.ones(len(x2))] @ T2.T
    A = np.einsum("ni,nj->nij", h2, h1).reshape(len(x1), 9)
    F = np.linalg.svd(A)[2][-1].reshape(3, 3)
    U, S, Vt = np.linalg.svd(F)
    return T2.T @ (U @ np.diag([S[0], S[1], 0.0]) @ Vt) @ T1


def pair_motions(lib, obs, mask, K, pairs):
    """Per pair: the 8-point F of the common observations (noise-free), E = K^T F K, and the candidate with the most
    correspondences in front of both cameras in the pair's own frame."""
    out = []
    for a, b in pairs:
        both = np.flatnonzero(mask[:, a] & mask[:, b])
        F = eight_point(obs[both, a], obs[both, b])
        E = c64(K.T @ F @ K)
        Rs, ts = np.zeros((4, 9)), np.zeros((4, 3))
        lib.hc_motion_from_essential(p(E), p(Rs), p(ts))
        counts = []
        for q in range(4):
            n = 0
            for f in both:
                fr = ctypes.c_int(0)
                lib.hc_cheirality(p(c64(K)), p(c64(K)), p(c64(Rs[q])), p(c64(ts[q])), *obs[f, a], *obs[f, b], ctypes.byref(fr))
                n += fr.value
            counts.append(n)
        q = int(np.argmax(counts))
        out.append((Rs[q].reshape(3, 3), ts[q], counts[q]))
    return out


@pytest.mark.parametrize("C", [4, 8, 16])
def test_host_stages_recover_the_true_rig(lib, C):
    """Noise-free float tracks: rotation averaging over every pair's motion and the translation stage give the true rig
    (in the gauge |t_1| = 1) to 1e-9, and every view keeps full weight."""
    obs, mask, poses, K, _ = float_tracks(C)
    pairs = [(a, b) for a in range(C) for b in range(a + 1, C) if (mask[:, a] & mask[:, b]).sum() >= 30]
    mot = pair_motions(lib, obs, mask, K, pairs)
    a = np.array([x for x, _ in pairs], dtype=np.int32)
    b = np.array([y for _, y in pairs], dtype=np.int32)
    Rab = c64(np.stack([m[0] for m in mot]))
    w = c64([m[2] for m in mot])
    use = np.ones(len(pairs), dtype=np.uint8)
    R = np.zeros((C, 3, 3)); resid = np.zeros(len(pairs))
    assert lib.hc_rotation_average(C, len(pairs), p(a), p(b), p(Rab), p(w), 5.0, p(use), p(R), p(resid)) == 1
    assert use.all() and resid.max() < 1e-4          # degrees through acos: ~1e-6 is its rounding floor near 0
    for c in range(C):
        assert np.abs(R[c] - poses[c]["R"]).max() < 1e-9
    Kinv = c64(np.stack([np.linalg.inv(K)] * C))
    t = np.zeros((C, 3)); wf = np.zeros(mask.shape)
    f = c64([K[0, 0]] * C)
    init = np.ascontiguousarray(mask, dtype=np.uint8)
    assert lib.hc_translations(p(c64(obs)), p(init), len(obs), C, p(Kinv), p(c64(R)), p(f), 4, 4.0, p(t), p(wf)) == 1
    true_t = np.stack([np.asarray(p_["t"]).reshape(3) for p_ in poses])
    true_t = true_t / np.linalg.norm(true_t[1])
    assert np.abs(t - true_t).max() < 1e-9
    assert (wf[mask.astype(bool)] > 1 - 1e-12).all()


def test_rotation_average_drops_a_wrong_pair(lib):
    """One pair's motion rotated by 30 degrees: it is marked unused and the rig is still exact."""
    C = 8
    _, poses, _, _ = synth.make_tracks(C, 10, seed=1)
    pairs = [(x, y) for x in range(C) for y in range(x + 1, C)]
    Rab = np.stack([poses[y]["R"] @ poses[x]["R"].T for x, y in pairs])
    bad = pairs.index((2, 5))
    Rab[bad] = cv2.Rodrigues(np.array([0.0, np.radians(30.0), 0.0]))[0] @ Rab[bad]
    a = np.array([x for x, _ in pairs], dtype=np.int32)
    b = np.array([y for _, y in pairs], dtype=np.int32)
    use = np.ones(len(pairs), dtype=np.uint8)
    R = np.zeros((C, 3, 3)); resid = np.zeros(len(pairs))
    assert lib.hc_rotation_average(C, len(pairs), p(a), p(b), p(c64(Rab)), p(c64(np.full(len(pairs), 100.0))), 5.0, p(use), p(R),
                                   p(resid)) == 1
    assert use.sum() == len(pairs) - 1 and not use[bad]
    assert abs(resid[bad] - 30.0) < 1e-6
    for c in range(C):
        assert np.abs(R[c] - poses[c]["R"]).max() < 1e-9
    # a pair graph that the remaining pairs do not connect is refused
    only = np.zeros(len(pairs), dtype=np.uint8)
    only[pairs.index((0, 1))] = 1
    assert lib.hc_rotation_average(C, len(pairs), p(a), p(b), p(c64(Rab)), p(c64(np.full(len(pairs), 100.0))), 5.0, p(only), p(R),
                                   p(resid)) == 0


def _angle(Ra, Rb):
    return np.degrees(np.arccos(np.clip((np.trace(np.asarray(Ra).T @ np.asarray(Rb)) - 1) / 2, -1, 1)))


def test_pair_frame_cheirality_on_a_rig_the_chain_twists(lib):
    """16-camera arc, integer pixels: the reference chain (RefPort.calibrate_init) gets an adjacent rotation 2 degrees
    or more wrong; the pair-frame cheirality on the same pairs' F picks the true motion of every adjacent pair."""
    C = 16
    for seed in range(116, 140):
        obs_obj, poses, K, _ = synth.make_tracks(C, 300, seed=seed, missing_frac=0.1)
        chain = RefPort([K] * C).calibrate_init(obs_obj.tolist(), rng_seed=0)
        rel = [_angle(poses[c + 1]["R"] @ poses[c]["R"].T, np.asarray(chain[c + 1]["R"]) @ np.asarray(chain[c]["R"]).T) for c in range(C - 1)]
        if max(rel) >= 2.0:
            break
    else:
        pytest.fail("no seed in 116..139 on which the reference chain twists a pair")
    obs = np.array([[[0.0 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    mot = pair_motions(lib, obs, mask, K, [(c, c + 1) for c in range(C - 1)])
    for c, (Rq, tq, _) in enumerate(mot):
        Rt = poses[c + 1]["R"] @ poses[c]["R"].T
        tt = poses[c + 1]["t"] - Rt @ poses[c]["t"]
        assert _angle(Rt, Rq) < 2.0, (seed, c)
        assert tq @ tt / np.linalg.norm(tt) > 0.99, (seed, c)

"""Host model of the cold-start calibration's device paths, shared by the CPU and GPU tests: the adjacent-pair chain of
csrc/calib_init.cu (8-point and RANSAC starts) and the pose graph of csrc/calib_graph.cu, stage by stage.  Where the
product's stage is host code (eigen problems, motion from E, rotation averaging, the translation solve) the model
calls the same code through the g++ builds in tests/hostcheck; where it is a kernel, the model is a g++ build of the
kernel's header (RANSAC, the pair-frame cheirality, the translation stage) or numpy (the 8-point normal matrix, the
Sampson selections, the chain's cheirality vote).

Every thresholded decision is returned with its relative margin in float64, so that a test can tell a decision the
device takes differently because of rounding (nvcc contracts to fused multiply-adds, the g++ builds use
-ffp-contract=off) from a wrong one."""
import ctypes
import importlib

import numpy as np

from tests import hostbuild
from tests.hostbuild import ptr

synth = importlib.import_module("low-cost-mocap_b200.synth")
SCALE_PX = 4.0          # CG_SCALE_PX: the Cauchy scale of the graph's translation weights


def c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Libs:
    """The host builds the model calls: rs of csrc/calib_ransac.cuh, cg of csrc/calib_graph.cuh and calib_pose.h."""
    def __init__(self):
        self.rs, self.cg = hostbuild.load("calib_ransac"), hostbuild.load("calib_graph")


# ------------------------------------------------------------------------------------------------------------ inputs
def float_tracks(C, n, seed, missing_frac=0.1):
    """Noise-free tracks (synth.make_tracks(..., round_to_int=False)): (obs [n, C, 2] float64, mask uint8, poses, K)."""
    obs_obj, poses, K, _ = synth.make_tracks(C, n, seed=seed, missing_frac=missing_frac, round_to_int=False)
    obs = np.array([[[0.0 if v is None else v for v in cam] for cam in fr] for fr in obs_obj], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in obs_obj], dtype=np.uint8)
    return obs, mask, poses, K


def chain_pairs(mask):
    """The chain's pairs (c, c+1) with their common frames, in frame order."""
    C = mask.shape[1]
    m = mask.astype(bool)
    return [(c, c + 1, np.flatnonzero(m[:, c] & m[:, c + 1])) for c in range(C - 1)]


def graph_pairs(mask, min_common):
    """mocap_calibrate_graph_host's pair table: every (a < b) in lexicographic order with >= min_common common frames."""
    C = mask.shape[1]
    m = mask.astype(bool)
    out = []
    for a in range(C):
        for b in range(a + 1, C):
            f = np.flatnonzero(m[:, a] & m[:, b])
            if len(f) >= min_common:
                out.append((a, b, f))
    return out


def pair_points(obs, a, b, frames):
    """{x1, y1, x2, y2} float32, as the device gathers them (the reference casts the common observations to float32)."""
    return np.ascontiguousarray(np.c_[obs[frames, a], obs[frames, b]].astype(np.float32))


# ------------------------------------------------------------------------------------------------------------ RANSAC
def ransac_margin(F, pts, thr):
    """Relative distance of every point's rs_is_inlier decision from its threshold, in float64."""
    F = np.asarray(F, dtype=np.float64).ravel()
    x1, y1, x2, y2 = (pts[:, k].astype(np.float64) for k in range(4))
    a = F[0] * x1 + F[1] * y1 + F[2]
    b = F[3] * x1 + F[4] * y1 + F[5]
    c = F[6] * x1 + F[7] * y1 + F[8]
    d = x2 * a + y2 * b + c
    a1 = F[0] * x2 + F[3] * y2 + F[6]
    b1 = F[1] * x2 + F[4] * y2 + F[7]
    rhs = thr * thr * np.minimum(a * a + b * b, a1 * a1 + b1 * b1)
    return np.abs(d * d - rhs) / np.maximum(rhs, 1e-300)


def host_ransac(libs, pts, pair, H, seed, thr):
    """hc_ransac_select over one pair: dict(ok, F [3, 3], mask bool [m], count, margin [m])."""
    m = len(pts)
    F = np.zeros(9)
    mask = np.zeros(m, dtype=np.uint8)
    cnt = ctypes.c_int(0)
    ok = libs.rs.hc_ransac_select(ptr(pts), m, pair, H, seed, thr, ptr(F), ptr(mask), ctypes.byref(cnt)) == 1
    return {"ok": ok, "F": F.reshape(3, 3), "mask": mask.astype(bool), "count": cnt.value if ok else 0,
            "margin": ransac_margin(F, pts, thr) if ok else np.full(m, np.inf)}


def ransac_models(libs, pts, pair, H, seed, thr):
    """Every (hypothesis, root) model of the scan: (n_models [H], counts [H, 3] with -1 past the models, F [H, 3, 3, 3])."""
    n = np.zeros(H, dtype=np.int32)
    counts = np.zeros((H, 3), dtype=np.int32)
    F = np.zeros((H, 3, 3, 3))
    libs.rs.hc_ransac_models(ptr(pts), len(pts), pair, H, seed, thr, ptr(n), ptr(counts), ptr(F))
    return n, counts, F


# ------------------------------------------------------------------------------------------------------------ 8-point
def hartley(q, inl):
    """(s, tx, ty) of the Hartley normalisation of q [m, 2] over the set inl, as calib_pose::hartley forms it."""
    h = q[inl]
    cx, cy = h[:, 0].sum() / len(h), h[:, 1].sum() / len(h)
    md = np.sqrt((h[:, 0] - cx) ** 2 + (h[:, 1] - cy) ** 2).sum() / len(h)
    s = np.sqrt(2.0) / md if md > 0 else 1.0
    return np.array([s, -s * cx, -s * cy])


def normal45(x1, x2, inl, T):
    """Upper triangle (45 entries, row-major) of the 9x9 normal matrix of rows kron(x2n, x1n) over inl, in float64."""
    a1 = x1[inl] * T[0] + T[1:3]
    a2 = x2[inl] * T[3] + T[4:6]
    one = np.ones(len(a1))
    A = np.c_[a2[:, :1] * a1, a2[:, :1], a2[:, 1:] * a1, a2[:, 1:], a1, one]
    N = A.T @ A
    return c64(N[np.triu_indices(9)])


def fit_numpy(x1, x2, inl, T):
    """Normalised 8-point F in numpy: smallest eigenvector, rank 2, de-normalised, unit norm (sign arbitrary)."""
    up = normal45(x1, x2, inl, T)
    N = np.zeros((9, 9))
    N[np.triu_indices(9)] = up
    N = N + np.triu(N, 1).T
    Fn = np.linalg.eigh(N)[1][:, 0].reshape(3, 3)
    U, s, Vt = np.linalg.svd(Fn)
    T1 = np.array([[T[0], 0, T[1]], [0, T[0], T[2]], [0, 0, 1]])
    T2 = np.array([[T[3], 0, T[4]], [0, T[3], T[5]], [0, 0, 1]])
    F = T2.T @ (U @ np.diag([s[0], s[1], 0]) @ Vt) @ T1
    return F / np.linalg.norm(F)


def fit_product(libs):
    """The product's host fit (hc_fit_from_normal calls calib_pose::fit_from_normal: trf::sym_eig and svd3, the
    product's sign) on the numpy normal matrix."""
    def fit(x1, x2, inl, T):
        F = np.zeros(9)
        assert libs.cg.hc_fit_from_normal(ptr(normal45(x1, x2, inl, T)), ptr(c64(T)), ptr(F)) == 1
        return F.reshape(3, 3)
    return fit


def sampson(F, x1, x2):
    """Sampson distance^2 of k_sampson_pairs, in float64."""
    F = np.asarray(F).ravel()
    l0 = F[0] * x1[:, 0] + F[1] * x1[:, 1] + F[2]
    l1 = F[3] * x1[:, 0] + F[4] * x1[:, 1] + F[5]
    l2 = F[6] * x1[:, 0] + F[7] * x1[:, 1] + F[8]
    m0 = F[0] * x2[:, 0] + F[3] * x2[:, 1] + F[6]
    m1 = F[1] * x2[:, 0] + F[4] * x2[:, 1] + F[7]
    e = x2[:, 0] * l0 + x2[:, 1] * l1 + l2
    return e * e / (l0 * l0 + l1 * l1 + m0 * m0 + m1 * m1)


def chain_refit(x1, x2, inl0, thr2, fit=fit_numpy):
    """calibrate_chain's estimator (calib_init.cu) for one pair from the fit set inl0 (None: all points; a set of fewer
    than 8 falls back to all): three fits, each but the last followed by a Sampson selection at thr2 that becomes the
    next fit set (all points when it holds fewer than 8); a selection of every point after the second fit ends the
    pair's rounds.  Returns (F, final set, smallest relative Sampson margin)."""
    n = len(x1)
    inl = np.ones(n, dtype=bool)
    if inl0 is not None and inl0.sum() >= 8:
        inl = inl0.astype(bool).copy()
    margin = np.inf
    for rnd in range(3):
        T = np.r_[hartley(x1, inl), hartley(x2, inl)]
        F = fit(x1, x2, inl, T)
        if rnd == 2:
            break
        d2 = sampson(F, x1, x2)
        margin = min(margin, (np.abs(d2 - thr2) / thr2).min())
        inl = d2 <= thr2
        cnt = inl.sum()
        if cnt < 8:
            inl[:] = True
        if cnt == n and rnd > 0:
            break
    return F, inl, margin


def eight_point_refit(x1, x2, inl0, thr=1.0):
    """numpy restatement of calibrate_chain's estimator (calib_init.cu) started from a given fit set: normalised 8-point,
    rank 2, then re-fits on the Sampson inliers, three fits in all.  F up to sign."""
    return chain_refit(np.asarray(x1, dtype=np.float64), np.asarray(x2, dtype=np.float64), np.asarray(inl0, dtype=bool), thr * thr)[0]


# ------------------------------------------------------------------------------------------------------------ chain
def dlt(Pa, Pb, xa, xb):
    A = np.array([xa[1] * Pa[2] - Pa[1], Pa[0] - xa[0] * Pa[2], xb[1] * Pb[2] - Pb[1], Pb[0] - xb[0] * Pb[2]])
    X = np.linalg.svd(A)[2][-1]
    return X[:3] / X[3]


def motions(libs, E):
    Rs, ts = np.zeros((4, 9)), np.zeros((4, 3))
    libs.cg.hc_motion_from_essential(ptr(c64(E)), ptr(Rs), ptr(ts))
    return Rs.reshape(4, 3, 3), ts


def chain_vote(libs, x1, x2, F, K0, K1, R_prev, t_prev):
    """k_cheirality's vote (index.py:253-262): candidate q of E = K1^T F K0 counts X_z > 0 plus (R_q^T X)_z > 0 for the
    DLT point X of P1 = K0 [R_prev | t_prev] and P2 = K1 [R_q | t_q] -- camera c's accumulated pose on one side, the
    relative candidate on the other.  Returns (votes [4], Rs, ts, smallest relative margin of the front tests)."""
    Rs, ts = motions(libs, K1.T @ F @ K0)
    P1 = K0 @ np.c_[R_prev, t_prev]
    votes = np.zeros(4, dtype=np.int64)
    margin = np.inf
    for q in range(4):
        P2 = K1 @ np.c_[Rs[q], ts[q]]
        for i in range(len(x1)):
            X = dlt(P1, P2, x1[i], x2[i])
            zc = Rs[q][:, 2] @ X
            votes[q] += int(X[2] > 0) + int(zc > 0)
            margin = min(margin, min(abs(X[2]), abs(zc)) / np.linalg.norm(X))
    return votes, Rs, ts, margin


def chain_model(libs, obs, mask, Ks, method="8point", H=2048, seed=0, thr=1.0):
    """The chain of calibrate_init(method="8point" | "ransac") on the host.  Returns dict(R [C,3,3], t [C,3], F [C-1,3,3],
    votes [C-1,4], inliers [n, C-1] (the final Sampson set, "ransac" only), ransac (per pair, "ransac" only), margins)."""
    n, C = mask.shape
    Ks = [np.asarray(k, dtype=np.float64) for k in Ks]
    K0, K1 = Ks[0], Ks[1]                          # the reference's intrinsics of cameras 0 and 1, for every pair
    R = [np.eye(3)]
    t = [np.zeros(3)]
    Fs, votes, rs_out = [], [], []
    inl_out = np.zeros((n, C - 1), dtype=np.uint8)
    margins = []
    for p_, (a, b, frames) in enumerate(chain_pairs(mask)):
        pts = pair_points(obs, a, b, frames)
        x1, x2 = pts[:, :2].astype(np.float64), pts[:, 2:].astype(np.float64)
        init = None
        if method == "ransac":
            r = host_ransac(libs, pts, p_, H, seed, thr)
            rs_out.append(r)
            init = r["mask"]
        F, inl, m_sampson = chain_refit(x1, x2, init, thr * thr, fit_product(libs))
        inl_out[frames, p_] = inl
        v, Rs, ts, m_front = chain_vote(libs, x1, x2, F, K0, K1, R[-1], t[-1])
        q = int(np.argmax(v))                      # strict >, first maximum
        assert v[q] > 0
        R.append(Rs[q] @ R[-1])
        t.append(t[-1] + R[-2] @ ts[q])
        Fs.append(F)
        votes.append(v)
        margins.append({"sampson": m_sampson, "front": m_front})
    out = {"R": np.stack(R), "t": np.stack(t), "F": np.stack(Fs), "votes": np.stack(votes), "margins": margins}
    if method == "ransac":
        out["inliers"] = inl_out
        out["ransac"] = rs_out
    return out


# ------------------------------------------------------------------------------------------------------------ graph
def inv3(K):
    """calib_graph.cu's inv3: the adjugate over the determinant, in its order of operations."""
    K = np.asarray(K, dtype=np.float64).ravel().tolist()
    det = K[0] * (K[4] * K[8] - K[5] * K[7]) - K[1] * (K[3] * K[8] - K[5] * K[6]) + K[2] * (K[3] * K[7] - K[4] * K[6])
    return np.array([(K[4] * K[8] - K[5] * K[7]) / det, (K[2] * K[7] - K[1] * K[8]) / det, (K[1] * K[5] - K[2] * K[4]) / det,
                     (K[5] * K[6] - K[3] * K[8]) / det, (K[0] * K[8] - K[2] * K[6]) / det, (K[2] * K[3] - K[0] * K[5]) / det,
                     (K[3] * K[7] - K[4] * K[6]) / det, (K[1] * K[6] - K[0] * K[7]) / det, (K[0] * K[4] - K[1] * K[3]) / det])


GRAPH_DEFAULTS = {"min_common": 30, "min_inliers": 30, "min_angle_deg": 2.0, "rot_outlier_deg": 5.0, "irls_rounds": 4}


def graph_model(libs, obs, mask, Ks, H=2048, seed=0, thr=1.0, **options):
    """mocap_calibrate_graph_host on the host, stage by stage (calib_graph.cu).  Returns dict(R [C,3,3], t [C,3] in the
    |t_1| = 1 gauge, pairs (the report's fields), support uint8 [n, C], weights [n, C], ransac (per pair), margins (per
    pair: the smallest relative margin of its RANSAC, Sampson and front decisions), weight_margin (the smallest
    |w - 0.5| / 0.5 of the final weights))."""
    o = dict(GRAPH_DEFAULTS, **options)
    n, C = mask.shape
    Ks = [np.asarray(k, dtype=np.float64) for k in Ks]
    table = graph_pairs(mask, o["min_common"])
    thr2 = thr * thr
    pairs, margins, rs_out = [], [], []
    Rab = np.zeros((len(table), 3, 3))
    wrot = np.zeros(len(table))
    use = np.zeros(len(table), dtype=np.uint8)
    sets = []
    for p_, (a, b, frames) in enumerate(table):
        pts = pair_points(obs, a, b, frames)
        x1, x2 = pts[:, :2].astype(np.float64), pts[:, 2:].astype(np.float64)
        r = host_ransac(libs, pts, p_, H, seed, thr)
        rs_out.append(r)
        mg = {"ransac": r["margin"].min(), "sampson": np.inf, "front": np.inf}
        # re-fits: three fit + Sampson rounds; a selection under 8 points keeps the previous set
        inl = r["mask"].copy() if r["mask"].sum() >= 8 else np.ones(len(pts), dtype=bool)
        for _ in range(3):
            T = np.r_[hartley(x1, inl), hartley(x2, inl)]
            F = fit_product(libs)(x1, x2, inl, T)
            d2 = sampson(F, x1, x2)
            mg["sampson"] = min(mg["sampson"], (np.abs(d2 - thr2) / thr2).min())
            sel = d2 <= thr2
            if sel.sum() >= 8:
                inl = sel
        sets.append(inl)
        # cheirality in the pair's own frame
        Rs, ts = motions(libs, Ks[b].T @ F @ Ks[a])
        counts = np.zeros(4, dtype=np.int64)
        angs = []
        inl8 = np.ascontiguousarray(inl, dtype=np.uint8)
        for q in range(4):
            front = np.zeros(len(pts), dtype=np.uint8)
            ang, marg = np.zeros(len(pts)), np.zeros(len(pts))
            libs.cg.hc_cheirality_pair(ptr(c64(Ks[a])), ptr(c64(Ks[b])), ptr(c64(Rs[q])), ptr(c64(ts[q])), ptr(pts), ptr(inl8), len(pts),
                                       ptr(front), ptr(ang), ptr(marg))
            counts[q] = front.sum()
            angs.append(ang)
            mg["front"] = min(mg["front"], marg.min())
        best, bc = -1, 0
        for q in range(4):
            if counts[q] > bc:
                best, bc = q, int(counts[q])
        rep = {"a": a, "b": b, "common": len(frames), "inliers": int(inl.sum()), "candidate": best if r["ok"] else -1,
               "in_front": bc if r["ok"] else 0, "median_angle_deg": np.nan, "rot_residual_deg": np.nan, "used": 0}
        if rep["candidate"] >= 0:
            av = np.sort(angs[best][angs[best] >= 0.0])
            h = len(av)
            rep["median_angle_deg"] = (av[h // 2] if h % 2 else 0.5 * (av[h // 2 - 1] + av[h // 2])) if h else 0.0
            Rab[p_] = Rs[best]
            wrot[p_] = bc
            use[p_] = 1 if bc >= o["min_inliers"] and rep["median_angle_deg"] >= o["min_angle_deg"] else 0
        pairs.append(rep)
        margins.append(mg)
    # rotation averaging
    ia = np.array([x[0] for x in table], dtype=np.int32)
    ib = np.array([x[1] for x in table], dtype=np.int32)
    R = np.zeros((C, 3, 3))
    resid = np.zeros(len(table))
    assert libs.cg.hc_rotation_average(C, len(table), ptr(ia), ptr(ib), ptr(c64(Rab)), ptr(c64(wrot)), o["rot_outlier_deg"], ptr(use), ptr(R),
                                       ptr(resid)) == 1
    for p_, rep in enumerate(pairs):
        rep["used"] = int(use[p_])
        if rep["candidate"] >= 0:
            rep["rot_residual_deg"] = resid[p_]
    # translations: a view enters if it is an inlier of >= 2 used pairs (>= 1 for a camera with one used pair)
    npairs = np.zeros(C, dtype=np.int64)
    hits = np.zeros((n, C), dtype=np.int64)
    for p_, (a, b, frames) in enumerate(table):
        if not use[p_]:
            continue
        npairs[a] += 1
        npairs[b] += 1
        hits[frames[sets[p_]], a] += 1
        hits[frames[sets[p_]], b] += 1
    init = np.ascontiguousarray(mask.astype(bool) & (hits >= np.where(npairs >= 2, 2, 1)[None, :]), dtype=np.uint8)
    Kinv = c64(np.stack([inv3(k) for k in Ks]))
    f = c64([k[0, 0] for k in Ks])
    t = np.zeros((C, 3))
    w = np.zeros((n, C))
    assert libs.cg.hc_translations(ptr(c64(obs)), ptr(init), n, C, ptr(Kinv), ptr(c64(R)), ptr(f), o["irls_rounds"], SCALE_PX, ptr(t), ptr(w)) == 1
    keep = (w >= 0.5).sum(1) >= 2
    support = ((w >= 0.5) & keep[:, None]).astype(np.uint8)
    wm = np.abs(w[init.astype(bool)] - 0.5) / 0.5
    return {"R": R, "t": t, "pairs": pairs, "support": support, "weights": w, "init": init, "ransac": rs_out, "margins": margins,
            "weight_margin": wm.min() if wm.size else np.inf}

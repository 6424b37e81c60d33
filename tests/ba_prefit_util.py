"""A float64 model of S4's Levenberg-Marquardt prefit, written from the algorithm and not from the kernels.

Both engines run the same prefit before the polish: engine 0 in k_ba_solve (ba_prefit_accumulate / ba_prefit_backsub,
csrc/ba_device.cuh), engine 1 in k_sba + prefit() (csrc/ba.cu).  This module states what they compute:

* unknowns: the poses of cameras 1..C-1, updated as R' = Exp(w) R, t' = t + dt, and one 3D point per valid point (a
  point with >= 2 views); camera 0 is pinned;
* start: the DLT point of every valid point at the start poses (helpers.py's triangulate_point);
* objective: 0.5 * sum of squared pinhole pixel residuals over the present views.  View number k of a point (its k-th
  PRESENT view) uses the intrinsics K[k], as the reference indexes them (helpers.py:305-307), not K[camera];
* Jacobians: complex-step derivatives of that residual function (exact to rounding, no hand-written derivative);
* damping: Marquardt, every diagonal entry of the camera and point blocks times (1 + lambda).  A point whose damped 3x3
  block is not positive definite stays where it is; a camera parameter whose undamped diagonal is zero (a camera that
  sees no point) is held fixed, so the other cameras are fitted as if that camera were absent;
* lambda: 1e-3 at the start; a step is taken when the cost drops and is finite, then lambda <- max(0.3 lambda, 1e-12),
  and the prefit stops once the relative drop is below BA_PREFIT_REL_STOP; a rejected step or a system that is not
  positive definite gives lambda <- 10 lambda, and the prefit stops once lambda > 1e12; at most max_iter iterations.

Small problems are solved as one dense system over poses and points; large ones in the Schur form, vectorised over the
points.  Both forms are the same linear algebra (tests check them against each other)."""
import os

import numpy as np
from scipy.spatial.transform import Rotation

REL_STOP = 1e-7              # BA_PREFIT_REL_STOP
LAMBDA0, LAMBDA_MIN, LAMBDA_MAX = 1e-3, 1e-12, 1e12
DENSE_MAX = 1500             # unknowns up to which the dense form is used
_H = 1e-30                   # complex step


def dlt_point(Ps, uv):
    """The reference's DLT: smallest right singular vector of A^T A, A = rows v P2 - P1, P0 - u P2."""
    A = []
    for P, (u, v) in zip(Ps, uv):
        A.append(v * P[2] - P[1])
        A.append(P[0] - u * P[2])
    A = np.asarray(A)
    _, _, Vh = np.linalg.svd(A.T @ A)
    return Vh[3, :3] / Vh[3, 3]


def _exp_series(w):
    """Exp of the skew matrix of w by its power series: analytic, so complex steps go through it (|w| << 1 only)."""
    W = np.zeros(w.shape[:-1] + (3, 3), dtype=w.dtype)
    W[..., 0, 1], W[..., 0, 2], W[..., 1, 2] = -w[..., 2], w[..., 1], -w[..., 0]
    W[..., 1, 0], W[..., 2, 0], W[..., 2, 1] = w[..., 2], -w[..., 1], w[..., 0]
    E = np.broadcast_to(np.eye(3), W.shape).astype(w.dtype)
    term = E.copy()
    for k in range(1, 6):
        term = term @ W / k
        E = E + term
    return E


class Problem:
    """obs [m, C, 2], mask [m, C], K [C, 3, 3] (K[k] for the k-th present view of a point)."""

    def __init__(self, obs, mask, K):
        self.obs = np.asarray(obs, np.float64)
        self.mask = np.asarray(mask).astype(bool)
        self.K = np.asarray(K, np.float64)
        m, C = self.mask.shape
        self.C, self.n = C, 6 * (C - 1)
        self.valid = self.mask.sum(1) >= 2
        self.pts = np.flatnonzero(self.valid)                       # model point j = problem point pts[j]
        vp, vc = np.nonzero(self.mask[self.pts])                    # views of the valid points, point-major
        rank = np.cumsum(self.mask[self.pts], axis=1) - 1           # k of each present view
        self.v_pt, self.v_cam, self.v_k = vp, vc, rank[vp, vc]
        self.v_uv = self.obs[self.pts[vp], vc]
        Kv = self.K[self.v_k]
        self.v_f = np.stack([Kv[:, 0, 0], Kv[:, 1, 1]], 1)
        self.v_c = np.stack([Kv[:, 0, 2], Kv[:, 1, 2]], 1)

    def dlt_points(self, R, t):
        X = np.empty((len(self.pts), 3))
        for j, p in enumerate(self.pts):
            cams = np.flatnonzero(self.mask[p])
            Ps = [self.K[k] @ np.c_[R[c], t[c]] for k, c in enumerate(cams)]
            X[j] = dlt_point(Ps, self.obs[p, cams])
        return X

    def residuals(self, R, t, X, w=None, dt=None, dX=None):
        """Pixel residuals [V, 2] of every view; w, dt, dX [V, 3] are per-view perturbations (complex allowed)."""
        RX = np.einsum("vij,vj->vi", R[self.v_cam], X[self.v_pt] if dX is None else X[self.v_pt] + dX)
        if w is not None:
            RX = np.einsum("vij,vj->vi", _exp_series(w), RX)
        Xc = RX + t[self.v_cam] + (0 if dt is None else dt)
        return self.v_f * Xc[:, :2] / Xc[:, 2:3] + self.v_c - self.v_uv

    def cost(self, R, t, X):
        e = self.residuals(R, t, X)
        return 0.5 * float(np.sum(e * e))

    def jacobians(self, R, t, X):
        """e [V, 2], Jc [V, 2, 6] wrt (w, dt) of the view's camera, Jp [V, 2, 3] wrt its point: complex step."""
        V = len(self.v_pt)
        e = self.residuals(R, t, X)
        J = np.empty((V, 2, 9))
        for j in range(9):
            d = np.zeros((V, 9), complex)
            d[:, j] = 1j * _H
            J[:, :, j] = self.residuals(R, t, X, d[:, :3], d[:, 3:6], d[:, 6:]).imag / _H
        return e, J[:, :, :6], J[:, :, 6:]

    def system(self, R, t, X):
        """Undamped normal equations: U [n, n] (block diagonal), gc [n], W [np, n, 3], V [np, 3, 3], gp [np, 3]."""
        e, Jc, Jp = self.jacobians(R, t, X)
        n, npt = self.n, len(self.pts)
        U, gc = np.zeros((n, n)), np.zeros(n)
        W = np.zeros((npt, n, 3))
        V = np.einsum("vai,vaj->vij", Jp, Jp)
        V = np.add.reduceat(V, np.r_[0, np.flatnonzero(np.diff(self.v_pt)) + 1], axis=0) if len(V) else V
        gp = np.zeros((npt, 3))
        np.add.at(gp, self.v_pt, np.einsum("vai,va->vi", Jp, e))
        for c in range(1, self.C):
            s = self.v_cam == c
            b = slice(6 * (c - 1), 6 * c)
            U[b, b] = np.einsum("vai,vaj->ij", Jc[s], Jc[s])
            gc[b] = np.einsum("vai,va->i", Jc[s], e[s])
            W[self.v_pt[s], b, :] = np.einsum("vai,vaj->vij", Jc[s], Jp[s])
        return U, gc, W, V, gp

    def step(self, sysm, lam, dense=None):
        """The damped step (dc [n], dp [np, 3]) or None when the reduced system is not positive definite."""
        U, gc, W, V, gp = sysm
        n, npt = self.n, len(self.pts)
        Ud = U + lam * np.diag(np.diag(U))
        held = np.diag(U) == 0.0                                     # parameters of a camera that sees nothing
        Ud[held, :] = 0.0
        Ud[:, held] = 0.0
        Ud[held, held] = 1.0
        rc = np.where(held, 0.0, gc)
        Vd = V * (1.0 + lam * np.eye(3))
        ok = np.array([_is_pd(v) for v in Vd], bool)                 # points whose damped block is singular stay put
        if dense is None:
            dense = n + 3 * int(ok.sum()) <= DENSE_MAX
        if dense:
            act = np.flatnonzero(ok)
            N = n + 3 * len(act)
            H, g = np.zeros((N, N)), np.zeros(N)
            H[:n, :n], g[:n] = Ud, rc
            for q, j in enumerate(act):
                b = slice(n + 3 * q, n + 3 * q + 3)
                H[:n, b] = W[j]
                H[b, :n] = W[j].T
                H[b, b] = Vd[j]
                g[b] = gp[j]
            try:
                L = np.linalg.cholesky(H)
            except np.linalg.LinAlgError:
                return None
            d = -np.linalg.solve(L.T, np.linalg.solve(L, g))
            dp = np.zeros((npt, 3))
            dp[act] = d[n:].reshape(-1, 3)
            return d[:n], dp
        Vi = np.zeros_like(Vd)
        Vi[ok] = np.linalg.inv(Vd[ok])
        WVi = np.einsum("pia,pab->pib", W, Vi)
        S = Ud - np.einsum("pib,pjb->ij", WVi, W)
        r = rc - np.einsum("pib,pb->i", WVi, gp)
        try:
            L = np.linalg.cholesky(S)
        except np.linalg.LinAlgError:
            return None
        dc = -np.linalg.solve(L.T, np.linalg.solve(L, r))
        dp = -np.einsum("pab,pb->pa", Vi, gp + np.einsum("pia,i->pa", W, dc))
        return dc, dp

    def apply(self, R, t, dc):
        R2, t2 = R.copy(), t.copy()
        for c in range(1, self.C):
            d = dc[6 * (c - 1):6 * c]
            R2[c] = Rotation.from_rotvec(d[:3]).as_matrix() @ R[c]
            t2[c] = t[c] + d[3:]
        return R2, t2


def _is_pd(A):
    try:
        np.linalg.cholesky(A)
        return True
    except np.linalg.LinAlgError:
        return False


def prefit(obs, mask, K, R, t, max_iter=50, dense=None):
    """Run the prefit from the poses (R [C, 3, 3], t [C, 3]).  K: one 3x3 matrix or [C, 3, 3].  Returns a dict:
    cost_initial, cost_final (the cost of the last accepted state), iterations, R, t, X (valid points only), and
    `trace`, one dict per iteration: lam (the damping it used), accepted, pd (the system was positive definite),
    cost, R, t (the state after it)."""
    K = np.asarray(K, np.float64)
    C = np.asarray(mask).shape[1]
    if K.ndim == 2:
        K = np.stack([K] * C)
    pb = Problem(obs, mask, K)
    R, t = np.array(R, np.float64), np.array(t, np.float64).reshape(C, 3)
    X = pb.dlt_points(R, t)
    cost = pb.cost(R, t, X)
    out = {"cost_initial": cost, "trace": []}
    lam, go, it = LAMBDA0, True, 0
    while it < max_iter and go:
        sysm = pb.system(R, t, X)
        st = pb.step(sysm, lam, dense)
        accepted = False
        if st is not None:
            dc, dp = st
            R2, t2 = pb.apply(R, t, dc)
            X2 = X + dp
            c2 = pb.cost(R2, t2, X2)
            accepted = bool(c2 < cost and np.isfinite(c2))
        used = lam
        if accepted:
            rel = (cost - c2) / max(cost, 1e-300)
            R, t, X, cost = R2, t2, X2, c2
            lam = max(lam * 0.3, LAMBDA_MIN)
            go = rel >= REL_STOP
        else:
            lam *= 10.0
            go = lam <= LAMBDA_MAX
        it += 1
        out["trace"].append({"lam": used, "accepted": accepted, "pd": st is not None, "cost": cost, "R": R.copy(), "t": t.copy()})
    out.update(cost_final=cost, iterations=it, R=R, t=t, X=X)
    return out


def rotvec_round_trip(R):
    """What the engines return after the prefit: every pose goes through its rotation vector (helpers.py:278-285)."""
    return Rotation.from_rotvec(Rotation.from_matrix(R).as_rotvec()).as_matrix()


def scale_free(t):
    """Translations up to the free global scale (camera 0 is pinned, so only the scale of the rig is free)."""
    t = np.asarray(t, np.float64)
    return t / np.linalg.norm(t)


# ---- cases shared by the host and the GPU tests --------------------------------------------------------------------
def golden_case(root, name):
    """(obs, mask, K, R_start, t_start) of an S4 golden of the real reference."""
    z = np.load(os.path.join(root, "tests", "golden", name + ".npz"))
    return z["obs"], z["mask"], z["K"], z["R_start"], z["t_start"]


def tracks_case(synth, C, F, seed, rot=0.03, tsig=0.05, missing=0.1):
    """Known-correspondence tracks of a synthetic rig and a perturbed start (rot: rad, tsig: pose units)."""
    o, poses, K, _ = synth.make_tracks(C, F, seed=seed, missing_frac=missing)
    st = synth.perturb_poses(poses, seed=seed + 1, rot_sigma=rot, t_sigma=tsig)
    obs = np.array([[[-1 if v is None else v for v in cam] for cam in fr] for fr in o], dtype=np.float64)
    mask = np.array([[cam[0] is not None for cam in fr] for fr in o], dtype=np.uint8)
    return obs, mask, K, np.stack([p["R"] for p in st]), np.stack([np.asarray(p["t"]).reshape(3) for p in st])


def unseen(case, cam):
    """The case with every view of camera `cam` masked out (points left with one view are not valid and take no part)."""
    obs, mask, K, R0, t0 = case
    mask = mask.copy()
    mask[:, cam] = 0
    return obs, mask, K, R0, t0


def without(case, cam):
    """The same data as a rig without camera `cam` (cam > 0)."""
    obs, mask, K, R0, t0 = case
    keep = [c for c in range(mask.shape[1]) if c != cam]
    K = np.asarray(K)
    return (np.ascontiguousarray(obs[:, keep]), np.ascontiguousarray(mask[:, keep]), K if K.ndim == 2 else K[keep],
            R0[keep], t0[keep])


# the engines against the model: same iteration count, prefit costs to 1e-10 relative, poses to 1e-9 after a few
# iterations (the model sums in another order and takes its DLT points from an SVD), and at the end of the prefit
# rotations to 1e-8 and translations to 1e-8 up to the free global scale of the rig
COST_RTOL, POSE_TOL, END_TOL = 1e-10, 1e-9, 1e-8


def assert_iteration(M, k, R, t, rep, loose=1.0):
    """Poses and report of an engine run with prefit_max_iter = k, max_nfev = 1 against iteration k of the model.
    loose: factor on the tolerances."""
    tr = M["trace"][k - 1]
    assert rep["prefit_iterations"] == k
    assert abs(rep["prefit_cost_initial"] - M["cost_initial"]) <= COST_RTOL * M["cost_initial"]
    assert abs(rep["prefit_cost_final"] - tr["cost"]) <= loose * COST_RTOL * tr["cost"], (k, rep["prefit_cost_final"], tr["cost"])
    assert np.abs(R - rotvec_round_trip(tr["R"])).max() < loose * POSE_TOL, (k, np.abs(R - rotvec_round_trip(tr["R"])).max())
    assert np.abs(t - tr["t"]).max() < loose * POSE_TOL, (k, np.abs(t - tr["t"]).max())


def assert_prefit(M, R, t, rep, loose=1.0):
    """Poses and report of an engine run with max_nfev = 1 against the model's whole prefit."""
    assert rep["prefit_iterations"] == M["iterations"], (rep["prefit_iterations"], M["iterations"])
    assert abs(rep["prefit_cost_final"] - M["cost_final"]) <= loose * COST_RTOL * max(M["cost_final"], 1.0)
    assert np.abs(R - rotvec_round_trip(M["R"])).max() < loose * END_TOL
    assert np.abs(scale_free(t) - scale_free(M["t"])).max() < loose * END_TOL

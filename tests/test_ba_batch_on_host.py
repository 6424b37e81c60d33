"""A batched launch of the device-resident bundle adjustment (csrc/ba_device.cuh), run unchanged on the host through
the SIMT emulation: several problems on sub-grids of one launch, each with its own barrier and workspace.  Every
problem must give the same bits (poses and report) as the single-solve hook on a grid of its own CTA count."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from tests.util import ROOT

HC = os.path.join(ROOT, "tests", "hostcheck")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
_P = ctypes.c_void_p
KEYS = ["cost_initial", "cost_final", "optimality", "n_iterations", "n_fev", "status", "n_residuals", "prefit_cost_initial",
        "prefit_cost_final", "prefit_iterations", "smem", "n_tr_solves", "n_tr_newton"]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    d = tmp_path_factory.mktemp("ba_batch_emu")
    libs = {}
    for name, src in (("single", "ba_dev_emu_host.cpp"), ("batch", "ba_batch_emu_host.cpp")):
        out = str(d / f"lib{name}.so")
        subprocess.check_call(["g++", "-std=c++20", "-O2", "-shared", "-fPIC", "-pthread", "-I" + CUDA_INC, "-Wno-attributes",
                               "-Wno-unknown-pragmas", "-fno-strict-aliasing", "-o", out, os.path.join(HC, src)])
        libs[name] = ctypes.CDLL(out)
    libs["single"].hc_ba_solve_dev.argtypes = [_P] * 2 + [ctypes.c_int] * 2 + [_P] * 3 + [ctypes.c_double] + [ctypes.c_int] * 6 + [_P]
    libs["batch"].hc_ba_solve_batch.argtypes = [ctypes.c_int, _P, _P, _P, ctypes.c_int, _P, _P, _P, ctypes.c_double] + \
        [ctypes.c_int] * 4 + [_P, ctypes.c_int, _P]
    return libs


def _p(a):
    return a.ctypes.data_as(_P)


def _single(emu, prob, K, prefit, n_ctas, n_threads, jac_mode=1):
    obs, mask, R, t = prob
    C = mask.shape[1]
    Ks = np.ascontiguousarray(np.stack([K] * C))
    R, t = R.copy(), t.copy()
    rep = np.zeros(13)
    assert emu["single"].hc_ba_solve_dev(_p(obs), _p(mask), obs.shape[0], C, _p(Ks), _p(R), _p(t), 1e-2, 0, jac_mode, int(prefit), 50,
                                         n_ctas, n_threads, _p(rep)) == 0
    return R, t, rep


def _batch(emu, probs, K, prefit, ctas, n_threads, jac_mode=1):
    n = len(probs)
    C = probs[0][1].shape[1]
    Ks = np.ascontiguousarray(np.stack([K] * C))
    keep = [np.ascontiguousarray(a) for pr in probs for a in pr[:2]]
    Rs = [p[2].copy() for p in probs]
    ts = [p[3].copy() for p in probs]
    reps = [np.zeros(13) for _ in probs]
    arr = lambda xs: (ctypes.c_void_p * n)(*[x.ctypes.data for x in xs])
    m = np.array([p[0].shape[0] for p in probs], dtype=np.int32)
    c = np.array(ctas, dtype=np.int32)
    assert emu["batch"].hc_ba_solve_batch(n, arr(keep[0::2]), arr(keep[1::2]), _p(m), C, _p(Ks), arr(Rs), arr(ts), 1e-2, 0, jac_mode,
                                          int(prefit), 50, _p(c), n_threads, arr(reps)) == 0
    return list(zip(Rs, ts, reps))


def _perturbed(R, t, seed):
    rng = np.random.default_rng(seed)
    R2, t2 = R.copy(), t.copy()
    for c in range(1, R.shape[0]):
        R2[c] = Rotation.from_rotvec(rng.normal(scale=0.01, size=3)).as_matrix() @ R[c]
        t2[c] = t[c] + rng.normal(scale=0.02, size=3)
    return np.ascontiguousarray(R2), np.ascontiguousarray(t2)


@pytest.fixture(scope="module")
def problems():
    """The ba_c4 golden and two smaller problems on the same rig (subsets of its points, other starting poses)."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "ba_c4.npz"))
    obs, mask = np.ascontiguousarray(z["obs"], np.float64), np.ascontiguousarray(z["mask"], np.uint8)
    R0, t0 = np.ascontiguousarray(z["R_start"], np.float64), np.ascontiguousarray(z["t_start"], np.float64)
    golden = (obs, mask, R0, t0)
    small1 = (np.ascontiguousarray(obs[:24]), np.ascontiguousarray(mask[:24])) + _perturbed(R0, t0, 1)
    small2 = (np.ascontiguousarray(obs[10:26]), np.ascontiguousarray(mask[10:26])) + _perturbed(R0, t0, 2)
    return z["K"], [golden, small1, small2]


def _assert_same(a, b):
    Ra, ta, ra = a
    Rb, tb, rb = b
    assert np.array_equal(Ra, Rb) and np.array_equal(ta, tb)
    assert np.array_equal(ra, rb), dict(zip(KEYS, zip(ra, rb)))


@pytest.mark.parametrize("prefit", [True, False])
def test_batch_problems_equal_their_single_solves(emu, problems, prefit):
    """3 problems on sub-grids of 2 + 1 + 1 CTAs x 64 threads: each equals the single solve on a grid of its size, bit
    for bit, with the prefit on and off."""
    K, probs = problems
    ctas = [2, 1, 1]
    out = _batch(emu, probs, K, prefit, ctas, 64)
    for prob, g, got in zip(probs, ctas, out):
        ref = _single(emu, prob, K, prefit, g, 64)
        _assert_same(got, ref)
        assert got[2][5] in (0, 1, 2, 3, 4) and got[2][6] == prob[0].shape[0]


def test_batch_empty_problem_beside_a_normal_one(emu, problems):
    """A problem without points reports status -3 and keeps its poses; the problem beside it equals its single solve."""
    K, probs = problems
    obs, mask, R, t = probs[1]
    empty = (np.zeros((0, mask.shape[1], 2)), np.zeros((0, mask.shape[1]), np.uint8), R, t)
    out = _batch(emu, [empty, probs[1]], K, True, [1, 2], 64)
    Re, te, re = out[0]
    assert re[5] == -3 and re[6] == 0 and np.array_equal(Re, R) and np.array_equal(te, t)
    _assert_same(out[1], _single(emu, probs[1], K, True, 2, 64))
    # one view per point: no point has two views
    one = mask.copy()
    one[:, 1:] = 0
    out = _batch(emu, [probs[2], (obs, np.ascontiguousarray(one), R, t)], K, True, [1, 1], 64)
    assert out[1][2][5] == -3 and np.array_equal(out[1][0], R) and np.array_equal(out[1][1], t)
    _assert_same(out[0], _single(emu, probs[2], K, True, 1, 64))

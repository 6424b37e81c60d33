"""S4's Levenberg-Marquardt prefit on the H100, held to the float64 model of tests/ba_prefit_util.py through every entry
point: engine 0 (the one-launch solve k_ba_solve, behind bundle_adjust and bundle_adjust_dev), engine 1 (the
host-stepped k_sba + prefit() of ba.cu) and the batched launch bundle_adjust_batch_dev.  prefit_max_iter = k with
max_nfev = 1 returns the poses after k prefit iterations.  Every shape is also run with a camera that sees no point:
that camera is held, and the others are fitted as if the rig did not have it."""
import importlib

import numpy as np
import pytest

from tests import ba_prefit_util as bu
from tests.util import ROOT, synth

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
UNSEEN_COST_RTOL = 1e-6      # final robust cost of the masked rig against the rig without that camera


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _ctx(case):
    obs, mask, K, R0, t0 = case
    C = mask.shape[1]
    K = np.asarray(K)
    ctx = pkg.MocapContext(C, 640, 480)
    ctx.set_cameras(list(K) if K.ndim == 3 else [K] * C, [{"R": R0[c], "t": t0[c]} for c in range(C)])
    return ctx


def _poses(case):
    _, _, _, R0, t0 = case
    return [{"R": R0[c], "t": t0[c]} for c in range(len(R0))]


def run_host(ctx, case, engine, **kw):
    """bundle_adjust (engine 0: one launch of k_ba_solve; engine 1: the host-stepped solve) -> R, t, report"""
    obs, mask = case[:2]
    out, rep = ctx.bundle_adjust(obs, mask, _poses(case), engine=engine, **kw)
    return np.stack([p["R"] for p in out]), np.stack([p["t"] for p in out]), rep


def run_dev(torch, ctx, case, **kw):
    """bundle_adjust_dev on device tensors -> R, t, report"""
    obs, mask, _, R0, t0 = case
    R = torch.from_numpy(np.ascontiguousarray(R0)).cuda()
    t = torch.from_numpy(np.ascontiguousarray(t0)).cuda()
    rep = ctx.bundle_adjust_dev(torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), R, t, **kw)
    torch.cuda.synchronize()
    return R.cpu().numpy(), t.cpu().numpy(), ctx.decode_ba_report(rep)


def _runner(torch, entry):
    if entry == "dev":
        return lambda ctx, case, **kw: run_dev(torch, ctx, case, **kw)
    return lambda ctx, case, **kw: run_host(ctx, case, int(entry[-1]), **kw)


def check_against_model(run, ctx, case, ks=(1, 2, 3), M=None, loose=1.0):
    M = bu.prefit(*case) if M is None else M
    for k in ks:
        if k <= M["iterations"]:
            bu.assert_iteration(M, k, *run(ctx, case, prefit_max_iter=k, max_nfev=1), loose=loose)
    bu.assert_prefit(M, *run(ctx, case, max_nfev=1), loose=loose)
    return M


def _cases():
    far = bu.tracks_case(synth, 4, 40, 10, rot=0.5, tsig=0.3)
    obs, mask, K, R0, t0 = bu.tracks_case(synth, 5, 60, 7)
    Ks = np.stack([K] * 5)
    for c in range(5):
        Ks[c, 0, 0] += 40 * c; Ks[c, 1, 1] -= 25 * c; Ks[c, 0, 2] += 7 * c; Ks[c, 1, 2] -= 5 * c
    rng = np.random.default_rng(8)
    mask[rng.uniform(size=60) < 0.5, 0] = 0
    mask[rng.uniform(size=60) < 0.4, 1] = 0
    return {"ba_c4": bu.golden_case(ROOT, "ba_c4"), "ba_c8": bu.golden_case(ROOT, "ba_c8"),
            "c16_n90": bu.tracks_case(synth, 16, 90, 36), "k_not_c": (obs, mask, Ks, R0, t0), "far_start": far,
            "ba_c4_unseen3": bu.unseen(bu.golden_case(ROOT, "ba_c4"), 3)}


CASES = _cases()
ENTRIES = ["engine0", "dev", "engine1"]


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("name", list(CASES))
def test_prefit_equals_model(torch, entry, name):
    """Iterations 1, 2 and 3 and the whole prefit equal the model: iteration count, prefit costs, poses.  Far from the
    minimum engine 1, which inverts the point blocks by cofactors, keeps 1e-9 of the cost rather than 1e-10."""
    case = CASES[name]
    loose = 100.0 if (name, entry) == ("far_start", "engine1") else 1.0
    M = check_against_model(_runner(torch, entry), _ctx(case), case, loose=loose)
    if name == "far_start":
        assert not all(s["accepted"] for s in M["trace"])


BIG = {"c8_m3000": (8, 3000, 5), "c16_m1600": (16, 1600, 6)}


@pytest.fixture(scope="module", params=list(BIG))
def big(request):
    """Config-sized problems the host build is too slow for, each with its unseen-camera variant (camera C // 2)."""
    C, F, seed = BIG[request.param]
    case = bu.tracks_case(synth, C, F, seed)
    masked = bu.unseen(case, C // 2)
    return case, masked, bu.without(case, C // 2), bu.prefit(*case), bu.prefit(*masked)


@pytest.mark.parametrize("entry", ENTRIES)
def test_config_sized_prefit_equals_model(torch, big, entry):
    run = _runner(torch, entry)
    case, masked, _, Mc, Mm = big
    check_against_model(run, _ctx(case), case, ks=(1, 3), M=Mc)
    M = check_against_model(run, _ctx(masked), masked, ks=(2,), M=Mm)
    C = case[1].shape[1]
    assert np.array_equal(M["R"][C // 2], case[3][C // 2])


@pytest.mark.parametrize("engine", [0, 1])
def test_unseen_camera_full_solve_equals_the_smaller_rig(torch, big, engine):
    """The whole solve, prefit and polish, with camera C // 2 masked out, against the same data as a rig without it:
    that camera comes back where it started, the others as in the smaller rig, at the same final cost."""
    case, masked, small = big[:3]
    C = case[1].shape[1]
    R, t, r = run_host(_ctx(masked), masked, engine)
    Rs, ts, rs = run_host(_ctx(small), small, engine)
    keep = [c for c in range(C) if c != C // 2]
    assert r["status"] in (1, 2, 3, 4) and r["prefit_iterations"] == rs["prefit_iterations"]
    assert abs(r["prefit_cost_final"] - rs["prefit_cost_final"]) <= 1e-9 * rs["prefit_cost_final"]
    assert abs(r["cost_final"] - rs["cost_final"]) <= UNSEEN_COST_RTOL * rs["cost_final"], (r["cost_final"], rs["cost_final"])
    assert np.abs(R[keep] - Rs).max() < 1e-6 and np.abs(t[keep] - ts).max() < 1e-6
    assert np.abs(R[C // 2] - masked[3][C // 2]).max() < 1e-15 and np.array_equal(t[C // 2], masked[4][C // 2])


def test_unseen_camera_on_the_golden_engines_agree(torch):
    """Golden ba_c4 with camera 3 masked out: both engines hold camera 3, report the prefit's cost, and reach the cost
    of the 3-camera rig (before camera 3 was held: 16 prefit iterations, prefit_cost_final 0, final cost 201 against
    0.055)."""
    case = CASES["ba_c4_unseen3"]
    small = bu.without(bu.golden_case(ROOT, "ba_c4"), 3)
    M = bu.prefit(*case)
    for engine in (0, 1):
        R, t, r = run_host(_ctx(case), case, engine)
        _, _, rs = run_host(_ctx(small), small, engine)
        assert r["prefit_iterations"] == M["iterations"] == rs["prefit_iterations"]
        assert abs(r["prefit_cost_final"] - M["cost_final"]) <= bu.COST_RTOL * M["cost_final"]
        assert abs(r["cost_final"] - rs["cost_final"]) <= UNSEEN_COST_RTOL * rs["cost_final"], (engine, r["cost_final"], rs["cost_final"])
        assert np.abs(R[3] - case[3][3]).max() < 1e-15 and np.array_equal(t[3], case[4][3])


def test_prefit_without_a_step_starts_the_polish_as_the_reference(torch):
    """One prefit iteration whose step is rejected: both engines report the initial prefit cost as the final one and run
    the polish as without the prefit (scipy's ||x0|| start radius)."""
    case = bu.tracks_case(synth, 4, 40, 11, rot=0.5, tsig=0.3)
    M = bu.prefit(*case, max_iter=1)
    assert not M["trace"][0]["accepted"]
    for engine in (0, 1):
        ctx = _ctx(case)
        _, _, r = run_host(ctx, case, engine, prefit_max_iter=1)
        _, _, rn = run_host(ctx, case, engine, prefit=False)
        assert r["prefit_iterations"] == 1 and r["prefit_cost_final"] == r["prefit_cost_initial"]
        assert abs(r["prefit_cost_final"] - M["cost_initial"]) <= bu.COST_RTOL * M["cost_initial"]
        assert (r["status"], r["n_fev"], r["n_iterations"]) == (rn["status"], rn["n_fev"], rn["n_iterations"])
        assert abs(r["cost_final"] - rn["cost_final"]) <= 1e-6 * rn["cost_final"]


@pytest.mark.parametrize("grid", ["1", "37", "all"])
def test_prefit_equals_model_on_any_grid(torch, big, grid):
    """set_ba_grid(1 / 37 / every SM): the prefit of engine 0 still equals the model, unseen camera included."""
    run = _runner(torch, "dev")
    case, masked, _, Mc, Mm = big
    for cs, M in ((case, Mc), (masked, Mm)):
        ctx = _ctx(cs)
        ctx.set_ba_grid({"1": 1, "37": 37, "all": 0}[grid])
        bu.assert_iteration(M, 2, *run(ctx, cs, prefit_max_iter=2, max_nfev=1))
        bu.assert_prefit(M, *run(ctx, cs, max_nfev=1))


def test_batch_with_an_unseen_camera_problem(torch):
    """bundle_adjust_batch_dev with a masked-camera problem between two normal ones, on 3 x 10 CTAs: every problem's
    prefit equals the model, and the whole solves equal single solves on 10 CTAs, bit for bit."""
    probs = [bu.tracks_case(synth, 8, 3000, 5), bu.unseen(bu.tracks_case(synth, 8, 500, 9), 2), bu.tracks_case(synth, 8, 40, 12)]

    def dev(p):
        obs, mask, _, R0, t0 = p
        return {"obs": torch.from_numpy(obs).cuda(), "mask": torch.from_numpy(mask).cuda(),
                "R": torch.from_numpy(np.ascontiguousarray(R0)).cuda(), "t": torch.from_numpy(np.ascontiguousarray(t0)).cuda()}
    ctx = _ctx(probs[0])
    ctx.set_ba_grid(30)
    single = _ctx(probs[0])
    single.set_ba_grid(10)
    for max_nfev in (1, 0):
        ds = [dev(p) for p in probs]
        reps = ctx.bundle_adjust_batch_dev(ds, max_nfev=max_nfev)
        torch.cuda.synchronize()
        for p, d, rep in zip(probs, ds, reps):
            r = ctx.decode_ba_report(rep)
            R, t = d["R"].cpu().numpy(), d["t"].cpu().numpy()
            Rs, ts, rs = run_dev(torch, single, p, max_nfev=max_nfev)
            r.pop("phase_ms"); rs.pop("phase_ms")
            assert np.array_equal(R, Rs) and np.array_equal(t, ts) and r == rs
            if max_nfev == 1:
                bu.assert_prefit(bu.prefit(*p), R, t, r)
            else:
                assert r["status"] in (1, 2, 3, 4)
        assert np.abs(ds[1]["R"].cpu().numpy()[2] - probs[1][3][2]).max() < 1e-15
        assert np.array_equal(ds[1]["t"].cpu().numpy()[2], probs[1][4][2])

"""The per-view screen of explicit correspondences (csrc/screen.cuh), compiled for the host with g++: the mask equals a
numpy restatement of the rule built on the oracle's triangulation and cv2's projection, hand-built tracks behave as the
rule says, and at the true poses the screen drops the mismatched views of contaminated tracks and keeps the good ones."""
import importlib

import cv2
import numpy as np
import pytest

from oracle.ref_port import RefPort
from tests import hostbuild
from tests.screen_util import contaminated_tracks, host_screen, screen_inputs

synth = importlib.import_module("low-cost-mocap_b200.synth")
THR = 4.0
NEAR = 1e-6          # px: rows with a compared error this close to the threshold are left out of the comparison


@pytest.fixture(scope="module")
def lib():
    return hostbuild.load("screen")


def restate_row(port, o, m, poses, thr):
    """The rule, restated from its definition: RefPort.triangulate_one (the reference's DLT, K of the k-th present
    view) and cv2.projectPoints on the float32 point with K of the rank the view holds among the triangulated views.
    Returns (kept mask, smallest |error - thr| over every comparison made)."""
    C = len(m)
    S = [c for c in range(C) if m[c]]
    margin = [np.inf]
    if len(S) < 2:
        return np.array(m, dtype=np.uint8), margin[0]

    def point(T):
        views = [[None, None] for _ in range(C)]
        for c in T:
            views[c] = [o[c][0], o[c][1]]
        return port.triangulate_one(views, poses)

    def support(T, Q):
        X32 = np.asarray(point(T), dtype=np.float64).astype(np.float32)[None, :]
        out = []
        for c in Q:
            k = sum(1 for q in T if q < c)
            px = cv2.projectPoints(X32, np.asarray(poses[c]["R"], dtype=np.float64), np.asarray(poses[c]["t"], dtype=np.float64),
                                   port.K[k], np.array([]))[0][0, 0]
            dx, dy = o[c][0] - float(px[0]), o[c][1] - float(px[1])
            d2 = dx * dx + dy * dy
            margin[0] = min(margin[0], abs(np.sqrt(d2) - thr))
            if d2 <= thr * thr:
                out.append(c)
        return out

    best, W = -1, []
    for i in range(len(S)):
        for j in range(i + 1, len(S)):
            sup = support([S[i], S[j]], S)
            if len(sup) > best:
                best, W = len(sup), sup
    kept = []
    if len(W) >= 2:
        Sp = support(W, S)
        if len(Sp) >= 2 and support(Sp, Sp) == Sp:
            kept = Sp
    out = np.zeros(C, dtype=np.uint8)
    out[kept] = 1
    return out, margin[0]


def test_pair_order_is_lexicographic(lib):
    S = 0b1011010010000110                       # views 1 2 7 10 12 13 15
    views = [c for c in range(16) if S >> c & 1]
    want = [(1 << views[i]) | (1 << views[j]) for i in range(len(views)) for j in range(i + 1, len(views))]
    assert [lib.hc_screen_pair(S, p) for p in range(len(want))] == want
    assert lib.hc_screen_pair(S, len(want)) == 0


@pytest.mark.parametrize("case", list(range(30)))
def test_host_build_equals_restatement(lib, case):
    """4 / 8 / 16 cameras, 0-40 % mismatched views, at the true and at perturbed poses: the host build's mask equals
    the restatement's on every row whose compared errors all lie further than 1e-6 px from the threshold."""
    name, obs, mask, K, poses = list(screen_inputs())[case]
    C = mask.shape[1]
    port = RefPort([K] * C)
    got, stats = host_screen(lib, obs, mask, [K] * C, poses, THR)
    compared = 0
    for f in range(len(mask)):
        want, margin = restate_row(port, obs[f].tolist(), mask[f], poses, THR)
        if margin < NEAR:
            continue
        compared += 1
        assert np.array_equal(got[f], want), (name, f, mask[f], got[f], want)
    assert compared >= 0.95 * len(mask), (name, compared)
    nv, nk = mask.astype(bool).sum(axis=1), got.astype(bool).sum(axis=1)
    assert stats.tolist() == [nv.sum(), nk.sum(), nv.sum() - nk.sum(), int(((nv >= 2) & (nk == 0)).sum())]


# ---- hand-built tracks on the 16-camera rig at its true poses ---------------------------------------------------------
def _rig(C=16):
    poses, K = synth.make_rig(C)
    return poses, K


def _views(X, poses, K):
    return np.floor(np.stack([synth.project(X[None, :], p, K)[0] for p in poses]))


def _screen(lib, o, m, poses, K, thr=THR):
    out, _ = host_screen(lib, o[None], np.asarray(m, dtype=np.uint8)[None], [K] * len(poses), poses, thr)
    return out[0]


def test_clean_track_keeps_every_view(lib):
    poses, K = _rig()
    rng = np.random.default_rng(1)
    for _ in range(20):
        X = rng.uniform(-0.5, 0.5, 3) + [0, 0, 3]
        o = _views(X, poses, K)
        m = np.ones(16, dtype=np.uint8)
        assert _screen(lib, o, m, poses, K).tolist() == m.tolist()


@pytest.mark.parametrize("m", list(range(3, 17)))
def test_one_bad_view_is_the_one_removed(lib, m):
    poses, K = _rig()
    rng = np.random.default_rng(m)
    for trial in range(5):
        X = rng.uniform(-0.5, 0.5, 3) + [0, 0, 3]
        o = _views(X, poses, K)
        keep = np.zeros(16, dtype=np.uint8)
        keep[np.sort(rng.choice(16, m, replace=False))] = 1
        bad = rng.choice(np.flatnonzero(keep))
        o[bad] += rng.choice([-1, 1], 2) * rng.uniform(30, 120, 2)
        want = keep.copy()
        want[bad] = 0
        assert _screen(lib, o, keep, poses, K).tolist() == want.tolist(), (trial, bad)


def test_two_bad_views_among_five_are_both_removed(lib):
    poses, K = _rig()
    rng = np.random.default_rng(7)
    for trial in range(20):
        X = rng.uniform(-0.5, 0.5, 3) + [0, 0, 3]
        o = _views(X, poses, K)
        keep = np.zeros(16, dtype=np.uint8)
        keep[rng.choice(16, 5, replace=False)] = 1
        bad = rng.choice(np.flatnonzero(keep), 2, replace=False)
        o[bad] = np.floor(rng.uniform([0, 0], [synth.WIDTH, synth.HEIGHT], size=(2, 2)))
        want = keep.copy()
        want[bad] = 0
        assert _screen(lib, o, keep, poses, K).tolist() == want.tolist(), (trial, bad)


def test_wrong_view_on_the_epipolar_line_of_a_two_view_track_is_kept(lib):
    """Two views only test epipolar consistency: a wrong point of camera b on the epipolar line of camera a's pixel
    (the image of another point on camera a's ray) is indistinguishable from a right one, and the rule keeps it."""
    poses, K = _rig(8)
    X = np.array([0.1, -0.2, 3.0])
    a, b = 0, 1
    centre_a = -np.asarray(poses[a]["R"]).T @ np.asarray(poses[a]["t"])
    Xw = centre_a + 1.25 * (X - centre_a)                      # same pixel in camera a, 60+ px away in camera b
    o = _views(X, poses, K)
    o[b] = _views(Xw, poses, K)[b]
    assert np.abs(o[b] - _views(X, poses, K)[b]).max() > 20
    m = np.zeros(8, dtype=np.uint8)
    m[[a, b]] = 1
    assert _screen(lib, o, m, poses, K).tolist() == m.tolist()


def test_two_view_track_over_the_threshold_is_dropped_whole(lib):
    poses, K = _rig(8)
    o = _views(np.array([0.1, -0.2, 3.0]), poses, K)
    o[3] += [0, 40]
    m = np.zeros(8, dtype=np.uint8)
    m[[2, 3]] = 1
    assert _screen(lib, o, m, poses, K).tolist() == [0] * 8


def test_rows_with_fewer_than_two_views_pass_unchanged(lib):
    poses, K = _rig(8)
    o = np.full((3, 8, 2), 1e4)                                # far off: it must not matter
    m = np.zeros((3, 8), dtype=np.uint8)
    m[1, 5] = 1
    m[2, 0] = 1
    out, stats = host_screen(lib, o, m, [K] * 8, poses, THR)
    assert np.array_equal(out, m)
    assert stats.tolist() == [2, 2, 0, 0]


def test_tie_in_support_keeps_the_earlier_pair(lib):
    """Views 0, 1 see one point, views 2, 3 another: both pairs are supported by two views, the earlier pair wins,
    whichever point it sees."""
    poses, K = _rig(8)
    P, Q = np.array([0.2, 0.1, 2.8]), np.array([-0.3, -0.2, 3.3])
    for first, second in ((P, Q), (Q, P)):
        o = np.concatenate([_views(first, poses, K)[:2], _views(second, poses, K)[2:]])
        m = np.array([1, 1, 1, 1, 0, 0, 0, 0], dtype=np.uint8)
        assert _screen(lib, o, m, poses, K).tolist() == [1, 1, 0, 0, 0, 0, 0, 0]


# ---- the rates of the rule at the true poses --------------------------------------------------------------------------
def screen_rates(lib, C, frac, n=300, seed=108, thr=THR):
    obs, mask, _, bad, poses, K, _ = contaminated_tracks(C, n, frac, seed)
    out, _ = host_screen(lib, obs, mask, [K] * C, poses, thr)
    seen, kept = mask.astype(bool), out.astype(bool)
    drop_bad = (~kept & bad).sum() / max(1, bad.sum())
    drop_good = (seen & ~bad & ~kept).sum() / max(1, (seen & ~bad).sum())
    return drop_bad, drop_good


@pytest.mark.parametrize("C", [8, 16])
@pytest.mark.parametrize("frac", [0.1, 0.2, 0.3, 0.4])
def test_rates_at_true_poses(lib, C, frac):
    """>= 99.5 % of the mismatched views dropped and <= 0.5 % of the good ones at 10-30 %; >= 98 % and <= 1 % at 40 %."""
    drop_bad, drop_good = screen_rates(lib, C, frac)
    lo, hi = (0.98, 0.01) if frac >= 0.4 else (0.995, 0.005)
    assert drop_bad >= lo and drop_good <= hi, (drop_bad, drop_good)

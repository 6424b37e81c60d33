"""The live loop's CPU tier: the host build of csrc/live.cuh (k_live_blobs's step code) against numpy on random blob
lists; the host part of the drop-in _camera_read (api.live_read_events), fed the oracle chain's outputs, against the
real reference's events and serial bytes in tests/golden/live_loop.npz; install_into(live=True)."""
import ctypes
import importlib
import json
import os
import subprocess

import numpy as np
import pytest

from tests.live_util import (CAPTURE, DIST, K, LOCATE, ROOT, TRIANGULATE, encode_events, golden_scene, load_golden,
                             oracle_read, render_read)

api = importlib.import_module("low-cost-mocap_b200.api")
pkg = importlib.import_module("low-cost-mocap_b200")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("live")), "liblive_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-ffp-contract=off", "-std=c++17", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "live_host.cpp")])
    lib = ctypes.CDLL(out)
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.hc_live.restype = None
    lib.hc_live.argtypes = [P, P, P, I, I, I, I, I, I, P, P, P, P, P, P]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


@pytest.mark.parametrize("C,MB,mode,have", [(4, 64, CAPTURE, 1), (2, 8, CAPTURE | TRIANGULATE, 1),
                                            (8, 32, CAPTURE | TRIANGULATE | LOCATE, 1), (3, 16, 0, 0)])
def test_host_build_equals_numpy(lib, C, MB, mode, have):
    """Gate, called, first points, counts, the flag OR (merged with what the matcher left when triangulating) and the
    dots, on random blob lists with empty cameras, empty reads, centres on and off the frame and more blobs than kept."""
    rng = np.random.default_rng(C * 100 + MB)
    n, S = 300, 48
    xy = rng.integers(-3, S + 3, (n, C, MB, 2)).astype(np.int32)
    cnt = rng.integers(0, MB + 3, (n, C)).astype(np.int32)
    cnt[rng.uniform(size=(n, C)) < 0.4] = 0
    cnt[::7] = 0
    fl = np.where(rng.uniform(size=(n, C)) < 0.1, rng.integers(1, 64, (n, C)), 0).astype(np.int32)
    set_fl = rng.integers(0, 32, n).astype(np.int32)
    out = dict(cnt=np.full((n, C), 99, np.int32), first=np.full((n, C, 2), 99, np.int32), gate=np.full(n, 9, np.uint8),
               called=np.full(n, 9, np.uint8), flags=set_fl.copy())
    frames = rng.integers(0, 256, (n, C, S, S, 3), dtype=np.uint8)
    before = frames.copy()
    lib.hc_live(_p(xy), _p(cnt), _p(fl), n, C, MB, S, have, mode, _p(out["cnt"]), _p(out["first"]), _p(out["gate"]), _p(out["called"]),
                _p(out["flags"]), _p(frames))
    eff = cnt if have else np.zeros_like(cnt)
    assert np.array_equal(out["cnt"], eff)
    want_first = np.where(eff[:, :, None] > 0, xy[:, :, 0, :], -1)
    assert np.array_equal(out["first"], want_first)
    gate = (eff > 0).any(1)
    assert np.array_equal(out["gate"], gate.astype(np.uint8))
    assert np.array_equal(out["called"], (gate & bool(mode & LOCATE)).astype(np.uint8))
    want_flags = (set_fl if mode & TRIANGULATE else np.zeros(n, np.int32)) | (np.bitwise_or.reduce(fl, axis=1) if have else 0)
    assert np.array_equal(out["flags"], want_flags)
    want = before.copy()
    if have and mode & CAPTURE:
        for r in range(n):
            for c in range(C):
                for x, y in xy[r, c, :min(cnt[r, c], MB)]:
                    if 0 <= x < S and 0 <= y < S:
                        want[r, c, y, x] = (100, 255, 100)
    assert np.array_equal(frames, want)
    assert not gate.all() and (gate.any() or not have)


def test_emits_of_the_oracle_chain_reproduce_the_reference():
    """live_read_events fed the oracle chain's outputs read by read gives the real reference's events and serial bytes
    exactly, over the whole scripted session: capture-only, triangulating, locating with gated reads, a set-origin
    change and a new filter."""
    from oracle.ref_port import RefPort
    from tests.track_util import OracleKalmanFilter
    g = load_golden()
    scene = golden_scene(g)
    port = RefPort([K] * 4)
    now = [0.0]
    kf, gen = None, 0
    n_serial = 0
    for k in range(len(g["mode"])):
        mode = int(g["mode"][k])
        if int(g["filter_gen"][k]) != gen:
            gen = int(g["filter_gen"][k])
            kf = OracleKalmanFilter(int(g["num_objects"]), lambda: now[0])
        now[0] = float(g["t"][k])
        wi = int(g["world_index"][k])
        res = oracle_read(port, scene, render_read(scene, k, bool(g["dark"][k])), mode, g["worlds"][wi] if wi >= 0 else None, kf, now)
        events, serial = api.live_read_events(res, 0, mode, g["drone_armed"])
        assert json.loads(encode_events(events)) == json.loads(str(g["events"][k])), k
        assert [b.decode("latin-1") for b in serial] == json.loads(str(g["serial"][k])), k
        n_serial += len(serial)
    assert n_serial > 50


def test_emits_raise_on_overflow_and_stay_silent_when_gated():
    res = dict(flags=np.array([api.F_BLOBS, 0], np.int32), gate=np.array([1, 0], np.uint8))
    with pytest.raises(pkg.MocapError):
        api.live_read_events(res, 0, CAPTURE, [])
    assert api.live_read_events(res, 1, CAPTURE | TRIANGULATE | LOCATE, [True]) == ([], [])
    assert api.live_read_events(res, 0, 0, []) == ([], [])


def test_install_into_rebinds_camera_read(monkeypatch):
    """live=True replaces _camera_read on the class behind the Singleton wrapper (where get_frames' self._camera_read
    resolves); the default leaves it.  Without a GPU the replacement fails loudly instead of falling back."""
    import torch
    from tests.test_host_cpu import _reference_like_modules
    api_, helpers, _ = _reference_like_modules(np.array([[600.0, 0, 320], [0, 600, 240], [0, 0, 1]]))
    monkeypatch.setattr(api.MocapSession, "_default", None)
    cams = helpers.Cameras.instance()
    cls = type(cams)
    monkeypatch.setattr(cls, "_camera_read", lambda self: "cpu", raising=False)
    pkg.install_into(helpers)
    assert cams._camera_read() == "cpu"
    pkg.install_into(helpers, live=True)
    assert cls._camera_read.__mocap_b200__ and cams._camera_read.__func__ is cls._camera_read
    assert not hasattr(helpers.Cameras, "_camera_read")
    if not torch.cuda.is_available():
        cams.cameras = type("Drv", (), {"read": lambda s: ([np.zeros((240, 320, 3), np.uint8)] * 4, None)})()
        cams.num_cameras = 4
        cams.is_capturing_points = cams.is_triangulating_points = cams.is_locating_objects = False
        with pytest.raises(pkg.MocapError):
            cams._camera_read()


def test_rotations_other_than_0_and_2_are_refused(monkeypatch):
    from tests.test_host_cpu import _reference_like_modules
    _, helpers, _ = _reference_like_modules(K)
    cams = helpers.Cameras.instance()
    cams.camera_params = [{"intrinsic_matrix": K.tolist(), "distortion_coef": DIST.tolist(), "rotation": r} for r in (0, 1, 0, 2)]
    cams.num_cameras = 4
    s = api.MocapSession.__new__(api.MocapSession)
    s._live, s.device, s.large_holes = {}, 0, False
    with pytest.raises(ValueError, match="rotation"):
        api._live_cameras(cams, s, [np.zeros((240, 320, 3), np.uint8)] * 4)

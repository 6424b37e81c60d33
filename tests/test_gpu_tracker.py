"""The drone tracker on the GPU (csrc/track.cu): bit-equal to the host build of track.cuh, held to the oracle and to
the real reference's records (tests/golden/track_live.npz), invariant to how a stream is split into batches, the
chain pipeline -> locate_objects -> tracker on one stream, the KalmanFilter drop-in, launch accounting,
reproducibility and refusals.  Run with ``-m gpu`` on an H100."""
import ctypes
import importlib

import numpy as np
import pytest

from tests.track_util import (build_track_host, golden_stream, host_run, load_golden, make_stream, objects_of, run_batches,
                              run_oracle)

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
TOL, TOL_AFTER_RESET = 5e-5, 5e-4       # as tests/test_tracker_on_host.py
SPLITS = (1, 7, 299, 301)
EINVAL = -1
K = np.array([[600.0, 0, 320], [0, 600, 240], [0, 0, 1]])


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build_track_host(tmp_path_factory.mktemp("track"))


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def _ctx():
    return pkg.MocapContext(2, 640, 480)


def _located(torch, sl):
    return {"objects": torch.from_numpy(np.ascontiguousarray(sl["objects"])).cuda(),
            "drone_index": torch.from_numpy(np.ascontiguousarray(sl["drone_index"])).cuda(),
            "n": torch.from_numpy(np.ascontiguousarray(sl["n"])).cuda()}


def device_run(torch, stream, D, sizes=(), ctx=None):
    ctx = ctx or _ctx()
    tr = ctx.tracker(D)

    def track(tr, sl):
        r = tr.track_dev(_located(torch, sl), torch.from_numpy(np.ascontiguousarray(sl["t"])).cuda())
        return {k: v.cpu().numpy() for k, v in r.items()}
    out = run_batches(tr, stream, sizes, track)
    tr.close()
    return out


def _equal(a, b):
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_device_equals_host_build_on_the_golden_stream(torch, lib, golden):
    st = golden_stream(golden)
    _equal(device_run(torch, st, 2), host_run(lib, st, 2))


@pytest.mark.parametrize("D,seed", [(1, 21), (2, 22), (8, 23)])
def test_device_equals_host_build_on_synthetic_streams(torch, lib, D, seed):
    st = make_stream(2500, D, seed=seed, absence=(0, 700, 100), reset_at=1800)
    _equal(device_run(torch, st, D, sizes=(1000,)), host_run(lib, st, D, sizes=(1000,)))


def test_device_follows_the_golden_records(torch, golden, capsys):
    """Against the real reference's records: present flags exact, heading bit-exact, pos / vel within 5e-5 before the
    reset and 5e-4 after it (test_tracker_on_host.py says why)."""
    st = golden_stream(golden)
    d = device_run(torch, st, 2)
    assert np.array_equal(d["present"], golden["present"]) and np.array_equal(d["heading"], golden["heading"])
    r = st["reset_at"]
    before = max(np.abs(d[k][:r] - golden[k][:r]).max() for k in ("pos", "vel"))
    after = max(np.abs(d[k][r:] - golden[k][r:]).max() for k in ("pos", "vel"))
    with capsys.disabled():
        print(f"\ngolden stream, device vs reference: max |d| {before:.2e} before reset, {after:.2e} after it")
    assert before <= TOL and after <= TOL_AFTER_RESET
    o = run_oracle(st, 2)
    assert np.array_equal(d["chosen"], o["chosen"])


def test_batch_split_invariance(torch, golden):
    """One batch, and batches of 1, 7, 299, 301 and the rest (crossing the low-pass buffer's 300 / 150 cut and the
    tracker's buffer growth), give identical bits."""
    st = golden_stream(golden)
    _equal(device_run(torch, st, 2), device_run(torch, st, 2, sizes=SPLITS))


def _drone_scenes(B, seed):
    """Marker triplets of two drones flying smooth paths 1 m apart (drone 0 with its third marker on the +y side,
    drone 1 on the -y side, so locate_objects labels them 0 and 1), clutter points, some frame-sets without drone 1."""
    rng = np.random.default_rng(seed)
    half, h = 0.075, np.sqrt(0.095 ** 2 - 0.075 ** 2)
    t = 1.7e9 + np.cumsum(rng.uniform(0.008, 0.014, B))
    scenes = []
    for s in range(B):
        tt = t[s] - t[0]
        pts = []
        for d, side in ((0, 1.0), (1, -1.0)):
            if d == 1 and 200 <= s < 260:
                continue
            centre = np.array([-0.5 + d, 0.3 * np.sin(0.7 * tt + d), 0.5 + 0.2 * np.cos(0.5 * tt)])
            yaw = 0.9 * np.sin(0.3 * tt + 2 * d)
            c, sn = np.cos(yaw), np.sin(yaw)
            local = np.array([[half, 0, 0], [-half, 0, 0], [0, side * h, 0]])
            Rz = np.array([[c, -sn, 0], [sn, c, 0], [0, 0, 1]])
            pts.extend(list(local @ Rz.T + centre + rng.normal(0, 0.002, (3, 3))))
        pts.extend(list(rng.uniform(-2, 2, (int(rng.integers(0, 3)), 3))))
        pts = np.array(pts).reshape(-1, 3)[rng.permutation(len(pts))]
        scenes.append((pts, rng.uniform(0.05, 2.0, len(pts))))
    return t, scenes


def test_full_chain_against_the_oracle(torch, capsys):
    """Drone marker points -> ctx.locate_objects -> tracker on one stream, against RefPort.locate_objects + the oracle
    tracker on the same points: present and chosen exact, pos / vel within 5e-5, heading within the locate_objects
    parity."""
    from oracle.ref_port import RefPort
    B, R, MO = 600, 16, 6
    t, scenes = _drone_scenes(B, seed=31)
    obj = np.zeros((B, R, 3)); err = np.zeros((B, R)); n = np.zeros(B, np.int32)
    for s, (p, e) in enumerate(scenes):
        n[s] = len(p); obj[s, :len(p)] = p; err[s, :len(p)] = e
    ctx = pkg.MocapContext(2, 640, 480, max_roots=R)
    tr = ctx.tracker(2)
    loc = ctx.locate_objects(torch.from_numpy(obj).cuda(), torch.from_numpy(err).cuda(), torch.from_numpy(n).cuda(), max_objects=MO)
    d = {k: v.cpu().numpy() for k, v in tr.track_dev(loc, torch.from_numpy(t).cuda()).items()}
    ref_objects = np.zeros((B, MO, 5)); ref_di = np.full((B, MO), -1, np.int32); ref_n = np.zeros(B, np.int32)
    for s, (p, e) in enumerate(scenes):
        ref = RefPort.locate_objects(p, e)
        ref_n[s] = len(ref)
        for i, o in enumerate(ref):
            ref_objects[s, i, :3], ref_objects[s, i, 3], ref_objects[s, i, 4], ref_di[s, i] = o["pos"], o["heading"], o["error"], o["droneIndex"]
    o = run_oracle(dict(objects=ref_objects, drone_index=ref_di, n=ref_n, t=t, reset_at=-1, reset_time=0.0), 2)
    assert np.array_equal(d["present"], o["present"]) and np.array_equal(d["chosen"], o["chosen"])
    assert o["present"].sum() >= 2 * B - 70
    dp, dv = float(np.abs(d["pos"] - o["pos"]).max()), float(np.abs(d["vel"] - o["vel"]).max())
    dh = float(np.abs(d["heading"] - o["heading"]).max())
    with capsys.disabled():
        print(f"\nchain: max |dpos| {dp:.2e}, |dvel| {dv:.2e}, |dheading| {dh:.2e}")
    assert dp <= TOL and dv <= TOL and dh <= 1e-11


def test_drop_in_equals_the_batched_path(torch, golden):
    """api.KalmanFilter with an injected clock: the batched path's bits, the reference's keys and dtypes, an empty
    object list (time advances, no record) and reset()."""
    st = golden_stream(golden)
    now = [0.0]
    kf = pkg.KalmanFilter(2, session=pkg.MocapSession([K] * 2), clock=lambda: now[0])
    B = 400
    r = st["reset_at"]
    idx = list(range(B)) + list(range(r, r + 60))     # up to 400, then jump to the reset (the same stream's calls)
    st2 = dict(st)
    st2.update({k: st[k][idx] for k in ("objects", "drone_index", "n", "t")})
    st2["reset_at"] = B
    want = device_run(torch, st2, 2)
    saw_empty = False
    for s in range(len(idx)):
        if s == B:
            now[0] = st2["reset_time"]
            kf.reset()
        now[0] = float(st2["t"][s])
        objs = objects_of(st2, s)
        recs = kf.predict_location(objs)
        saw_empty |= not objs
        assert [x["droneIndex"] for x in recs] == [d for d in range(2) if want["present"][s, d]]
        for x in recs:
            d = x["droneIndex"]
            assert set(x) == {"pos", "vel", "heading", "droneIndex"}
            assert x["pos"].dtype == np.float32 and x["pos"].shape == (3,) and x["vel"].dtype == np.float32
            assert isinstance(x["heading"], np.float64) and type(d) is int
            assert np.array_equal(x["pos"], want["pos"][s, d]) and np.array_equal(x["vel"], want["vel"][s, d])
            assert x["heading"] == want["heading"][s, d]
    assert saw_empty
    assert kf.predict_location([]) == []


@pytest.mark.parametrize("D", [1, 2, 5, 8])
def test_two_launches_per_batch(torch, D):
    ctx = _ctx()
    tr = ctx.tracker(D)
    for B in (1, 1000, 5000):
        st = make_stream(B, D, seed=B + D)
        loc = _located(torch, st)
        ts = torch.from_numpy(st["t"]).cuda()
        before = ctx.launch_count()
        tr.track_dev(loc, ts)
        assert ctx.launch_count() - before == 2, (D, B)
    torch.cuda.synchronize()


def test_chain_on_a_side_stream(torch):
    """locate_objects and the tracker enqueued on a non-default stream give the default stream's bits."""
    st = make_stream(800, 2, seed=41, reset_at=500)
    want = device_run(torch, st, 2)
    ctx = _ctx()
    tr = ctx.tracker(2)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        loc = _located(torch, st)
        ts = torch.from_numpy(st["t"]).cuda()
        a = tr.track_dev({k: v[:500] for k, v in loc.items()}, ts[:500])
        tr.reset(st["reset_time"] - 20)
        b = tr.track_dev({k: v[500:] for k, v in loc.items()}, ts[500:])
    side.synchronize()
    for k in want:
        assert np.array_equal(np.concatenate([a[k].cpu().numpy(), b[k].cpu().numpy()]), want[k]), k


def test_reproducible(torch):
    st = make_stream(3000, 2, seed=51, reset_at=2000)
    _equal(device_run(torch, st, 2, sizes=(1500,)), device_run(torch, st, 2, sizes=(1500,)))


def test_refusals_launch_nothing(torch):
    ctx = _ctx()
    lib = ctx.lib
    h = ctypes.c_void_p()
    for D in (0, 9, -1):
        assert lib.mocap_tracker_create(ctx.h, D, ctypes.byref(h)) == EINVAL
    assert lib.mocap_tracker_create(ctx.h, 2, None) == EINVAL
    tr = ctx.tracker(2)
    st = make_stream(4, 2, seed=1)
    loc = _located(torch, st)
    ts = torch.from_numpy(st["t"]).cuda()
    outs = [torch.empty(n, dtype=dt, device="cuda") for n, dt in (((24,), torch.float32), ((24,), torch.float32),
            ((8,), torch.float64), ((8,), torch.uint8), ((8,), torch.int32))]
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    args = [p(loc["objects"]), p(loc["drone_index"]), p(loc["n"]), 8, p(ts), 4] + [p(o) for o in outs]
    before = ctx.launch_count()
    for i in (0, 1, 2, 4, 6, 7, 8, 9, 10):
        bad = list(args)
        bad[i] = ctypes.c_void_p(0)
        assert lib.mocap_track_objects_dev(tr.h, *bad) == EINVAL, i
    for i, v in ((3, 0), (5, 0), (5, -3), (3, -1)):
        bad = list(args)
        bad[i] = v
        assert lib.mocap_track_objects_dev(tr.h, *bad) == EINVAL, i
    assert lib.mocap_track_objects_dev(None, *args) == EINVAL
    assert lib.mocap_tracker_reset(tr.h, float("nan")) == EINVAL
    assert ctx.launch_count() == before
    with pytest.raises(ValueError):
        tr.track_dev(loc, ts[:3])
    assert lib.mocap_track_objects_dev(tr.h, *args) == 0
    assert ctx.launch_count() == before + 2
    torch.cuda.synchronize()

"""The live loop on the H100 (mocap_live_dev / mocap_live_host, api.camera_read): the drop-in _camera_read replaying the
real reference's session (tests/golden/live_loop.npz), every read against the oracle chain at 2, 4 and 8 cameras (and
with large holes), batched replay against single reads, the gated tracker, flags, modes and launch counts."""
import importlib

import numpy as np
import pytest

from tests.live_util import (CAPTURE, DIST, IN_H, IN_W, K, LOCATE, TRIANGULATE, StandinCameras, compare_events,
                             compare_serial, golden_scene, load_golden, make_scene, oracle_read, render_read, timestamp)

pytestmark = pytest.mark.gpu
api = importlib.import_module("low-cost-mocap_b200.api")
pkg = importlib.import_module("low-cost-mocap_b200")
FULL = CAPTURE | TRIANGULATE | LOCATE


def _ctx(scene, large_holes=False, cameras=True, world=None, **kw):
    C = scene["C"]
    ctx = api.MocapContext(C, 320, 320, **(kw or api.MIRROR_LIMITS))
    if large_holes:
        ctx.set_large_holes(True)
    ctx.set_preprocess(IN_W, IN_H, scene["rotations"], [K] * C, [DIST] * C)
    if cameras:
        ctx.set_cameras([K] * C, scene["poses"])
        ctx.set_world_transform(world)
    return ctx


def test_golden_replay_through_the_drop_in(capsys):
    """camera_read on a stand-in Cameras replays the reference's session: event names identical, image-points exact,
    point counts exact, object_points 1e-7, errors rtol 1e-9, objects exact in count and droneIndex with pos 1e-7, error
    rtol 1e-9 and heading 1e-9, filtered drones present exactly as the reference's and within the tracker's bars, serial
    bytes identical up to reported rounding-midpoint cases."""
    g = load_golden()
    scene = golden_scene(g)
    cams = StandinCameras(g, scene)
    session = api.MocapSession([K] * 4, 320, 320)
    bad, notes = [], []
    for k in range(len(g["mode"])):
        cams.set_read(k)
        frames = api.camera_read(cams, session, clock=lambda k=k: timestamp(k))
        assert isinstance(frames, list) and frames[0].shape == (320, 320, 3)
        want = [(n, p) for n, p in __import__("json").loads(str(g["events"][k]))]
        bad += [f"read {k}: {b}" for b in compare_events(cams.events, want)]
        want_serial = [s.encode("latin-1") for s in __import__("json").loads(str(g["serial"][k]))]
        bad += [f"read {k}: {b}" for b in compare_serial(cams.lines, want_serial, want, report=notes.append)]
    with capsys.disabled():
        print(f"\ngolden replay: {len(g['mode'])} reads; rounding-midpoint cases: {len(notes)}")
        for n in notes:
            print("  ", n)
    assert not bad, bad[:10]


@pytest.mark.parametrize("C,large", [(2, False), (4, False), (8, False), (4, True)])
def test_every_read_equals_the_oracle_chain(C, large):
    """live_host per read against RefPort preprocessing -> find_dot -> match + world transform -> locate_objects ->
    OracleKalmanFilter: processed frames with the dots bit-equal, first points, counts and gate exact, points and
    objects within the replay's bars, the drones present as the oracle's.  large: discs of 40-60 px that preprocessing
    turns into rings over 62 px, with large_holes on."""
    from oracle.ref_port import RefPort
    from tests.track_util import OracleKalmanFilter
    g = load_golden()
    M = g["worlds"][0]
    rot = [0, 2, 2, 0, 0, 2, 2, 0][:C]
    scene = make_scene(10 + C, M, C=C, rotations=rot, radius=(20, 30) if large else (2, 4), large=large,
                       drones=1 if large else 2, clutter=0 if large else 1)
    ctx = _ctx(scene, large_holes=large, world=M)
    tr = ctx.tracker(2)
    port = RefPort([K] * C)
    now = [0.0]
    kf = OracleKalmanFilter(2, lambda: now[0])
    n_reads, open_reads, found = 24, 0, 0
    for k in range(n_reads):
        dark = k in (9, 10)
        raw = render_read(scene, k, dark)
        mode = CAPTURE if k < 4 else FULL
        now[0] = timestamp(k)
        got = ctx.live_host(raw[None], mode, [now[0]] if mode & LOCATE else None, tr if mode & LOCATE else None, want_frames=True)
        want = oracle_read(port, scene, raw, mode, M, kf, now)
        assert np.array_equal(got["frames"][0], want["frames"]), k
        for key in ("blob_n", "first", "gate"):
            assert np.array_equal(got[key][0], want[key][0]), (k, key)
        assert got["flags"][0] == 0, k
        open_reads += int(want["gate"][0])
        if mode & LOCATE and want["gate"][0]:
            n = int(want["n"][0])
            assert got["n"][0] == n and got["called"][0] == 1, k
            assert np.allclose(got["obj"][0, :n], want["obj"][0, :n], rtol=1e-7, atol=1e-7), k
            assert np.allclose(got["err"][0, :n], want["err"][0, :n], rtol=1e-9, atol=0), k
            m = int(want["n_objects"][0])
            assert got["n_objects"][0] == m and np.array_equal(got["drone_index"][0, :m], want["drone_index"][0, :m]), k
            assert np.allclose(got["objects"][0, :m], want["objects"][0, :m], rtol=1e-7, atol=1e-7), k
            assert np.array_equal(got["present"][0], want["present"][0]), k
            assert np.allclose(got["pos"][0], want["pos"][0], atol=5e-4) and np.allclose(got["vel"][0], want["vel"][0], atol=5e-4), k
            found += m
        elif mode & LOCATE:
            assert got["called"][0] == 0 and not got["present"][0].any(), k
    assert open_reads >= n_reads - 2 and (found > 0 or large)


def _batch(scene, B, seed=0):
    rng = np.random.default_rng(seed)
    dark = rng.uniform(size=B) < 0.15
    raw = np.stack([render_read(scene, k, bool(dark[k])) for k in range(B)])
    return raw, np.array([timestamp(k) for k in range(B)])


@pytest.mark.parametrize("B", [1, 7, 300])
def test_batched_replay_equals_single_reads(B):
    """live over B reads (gated ones included) equals B live_host reads of one, bit for bit in every computed slice and
    the frames; live_host of the whole batch as well."""
    import torch
    g = load_golden()
    scene = make_scene(6, g["worlds"][0])
    raw, ts = _batch(scene, B, seed=B)
    a, b, c = _ctx(scene, world=g["worlds"][0]), _ctx(scene, world=g["worlds"][0]), _ctx(scene, world=g["worlds"][0])
    ta, tb, tc = a.tracker(2), b.tracker(2), c.tracker(2)
    dev = a.torch_device
    whole = a.live(torch.from_numpy(raw).to(dev), FULL, torch.from_numpy(ts).to(dev), ta, want_frames=True)
    torch.cuda.synchronize()
    whole = {k: v.cpu().numpy() for k, v in whole.items()}
    host = c.live_host(raw, FULL, ts, tc, want_frames=True)
    single = [b.live_host(raw[k:k + 1], FULL, ts[k:k + 1], tb, want_frames=True) for k in range(B)]
    for r, s in enumerate(single):
        for key in ("flags", "gate", "blob_n", "first", "n", "n_objects", "called", "pos", "vel", "heading", "present", "chosen", "frames"):
            assert np.array_equal(whole[key][r], s[key][0]), (r, key)
            assert np.array_equal(host[key][r], s[key][0]), (r, key)
        n, m = int(s["n"][0]), int(s["n_objects"][0])
        for key, cnt in (("obj", n), ("err", n), ("objects", m), ("drone_index", m)):
            assert np.array_equal(whole[key][r, :cnt], s[key][0, :cnt]), (r, key)
    if B == 300:
        assert 0 < whole["called"].sum() < B and whole["present"].any()


def test_gated_tracker_equals_the_tracker_without_the_closed_reads():
    """track_dev(calls=) on a batch equals track_dev on the same batch with the closed frame-sets removed, bit for bit,
    and the closed ones are absent; calls=None is today's track_dev."""
    import torch
    from tests.track_util import make_stream
    st = make_stream(600, 2, seed=31)
    ctx = api.MocapContext(4, 320, 320)
    dev = ctx.torch_device
    calls = (np.random.default_rng(3).uniform(size=600) > 0.2).astype(np.uint8)
    loc = {"objects": torch.from_numpy(st["objects"]).to(dev), "drone_index": torch.from_numpy(st["drone_index"]).to(dev),
           "n": torch.from_numpy(st["n"]).to(dev)}
    keep = np.flatnonzero(calls)
    loc_k = {k: v[torch.from_numpy(keep).to(dev)].contiguous() for k, v in loc.items()}
    t = torch.from_numpy(st["t"]).to(dev)
    gated = ctx.tracker(2).track_dev(loc, t, calls=torch.from_numpy(calls).to(dev))
    plain = ctx.tracker(2).track_dev(loc_k, t[torch.from_numpy(keep).to(dev)].contiguous())
    none_ = ctx.tracker(2).track_dev(loc, t, calls=None)
    ref = ctx.tracker(2).track_dev(loc, t)
    torch.cuda.synchronize()
    for k in gated:
        gv, pv = gated[k].cpu().numpy(), plain[k].cpu().numpy()
        assert np.array_equal(gv[keep], pv), k
        assert np.array_equal(none_[k].cpu().numpy(), ref[k].cpu().numpy()), k
    closed = calls == 0
    assert not gated["present"].cpu().numpy()[closed].any() and (gated["chosen"].cpu().numpy()[closed] == -1).all()
    assert not gated["pos"].cpu().numpy()[closed].any() and not gated["vel"].cpu().numpy()[closed].any()


def test_a_flagged_read_carries_its_flag_and_the_drop_in_raises():
    """A read with more blobs than max_blobs in one image carries MOCAP_F_BLOBS, its neighbours none; the drop-in raises
    MocapError on it and reads the next one normally."""
    g = load_golden()
    scene = make_scene(6, g["worlds"][0])
    raw = np.stack([render_read(scene, k) for k in range(3)])
    yy, xx = np.mgrid[0:IN_H, 0:IN_W]
    speckle = ((yy % 12 == 6) & (xx % 12 == 6) & (yy > 20) & (yy < IN_H - 20))
    raw[1, 2][speckle] = 255
    raw[1, 2] = np.maximum(raw[1, 2], np.roll(raw[1, 2], 1, axis=1))
    ctx = _ctx(scene, world=g["worlds"][0])
    out = ctx.live_host(raw, CAPTURE)
    assert out["flags"][1] & api.F_BLOBS and out["flags"][0] == 0 and out["flags"][2] == 0
    cams = StandinCameras(g, scene)
    session = api.MocapSession([K] * 4, 320, 320)
    cams.set_read(0)
    for k in range(3):
        cams.frames = list(raw[k])
        cams.events = []
        if k == 1:
            with pytest.raises(pkg.MocapError):
                api.camera_read(cams, session)
        else:
            api.camera_read(cams, session)
            assert cams.events and cams.events[0][0] == "image-points"


def test_modes():
    """Invalid combinations return EINVAL before any launch; capture-only runs on a context without cameras;
    triangulating without cameras is a state error; locating needs a tracker and timestamps."""
    g = load_golden()
    scene = make_scene(6, g["worlds"][0])
    ctx = _ctx(scene, cameras=False)
    raw = render_read(scene, 0)[None]
    for mode in (TRIANGULATE, LOCATE, TRIANGULATE | LOCATE, CAPTURE | LOCATE, 8, -1):
        n0 = ctx.launch_count()
        with pytest.raises(pkg.MocapError) as e:
            ctx.live_host(raw, mode, [0.0], ctx.tracker(2))
        assert e.value.status == -1 and ctx.launch_count() == n0, mode
    out = ctx.live_host(raw, CAPTURE, want_frames=True)
    assert out["gate"][0] == 1 and out["blob_n"][0].sum() > 0
    with pytest.raises(pkg.MocapError) as e:
        ctx.live_host(raw, CAPTURE | TRIANGULATE)
    assert e.value.status == -5
    ctx.set_cameras([K] * 4, scene["poses"])
    with pytest.raises(pkg.MocapError) as e:
        ctx.live_host(raw, FULL, [0.0], None)
    assert e.value.status == -1
    zero = ctx.live_host(raw, 0, want_frames=True)
    assert zero["gate"][0] == 0 and zero["blob_n"][0].sum() == 0 and zero["flags"][0] == 0


def test_launch_count_per_read_is_fixed(capsys):
    """Kernels per live read by mode, the same for every read (busy, empty and dark ones)."""
    g = load_golden()
    scene = make_scene(6, g["worlds"][0])
    ctx = _ctx(scene, world=g["worlds"][0])
    tr = ctx.tracker(2)
    counts = {}
    for mode in (0, CAPTURE, CAPTURE | TRIANGULATE, FULL):
        seen = set()
        for k in range(8):
            raw = render_read(scene, k, dark=k % 3 == 1)[None]
            n0 = ctx.launch_count()
            ctx.live_host(raw, mode, [timestamp(k)], tr if mode & LOCATE else None, want_frames=bool(k % 2))
            seen.add(ctx.launch_count() - n0)
        assert len(seen) == 1, (mode, seen)
        counts[mode] = seen.pop()
    with capsys.disabled():
        print(f"\nlaunches per read: {counts}")
    assert counts == {0: 2, CAPTURE: 5, CAPTURE | TRIANGULATE: 7, FULL: 10}

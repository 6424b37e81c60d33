"""The drone locator on the GPU (csrc/locate_kernels.cu): held to the oracle on the scenes of tests/locate_util.py with
the bars of tests/test_locate_on_host.py (counts, record order, droneIndex, pos and error bit-exact, heading within 4
ulp of pi/2) and bit-equal to the host build of locate_device.cuh in everything but the heading; batch sizes around one
128-thread block and 100 000 frame-sets, max_roots 16 / 64 / 128, count limits, truncation with guard rows, streams,
reproducibility, launch accounting, refusals and the drop-in.  Run with ``-m gpu`` on an H100."""
import ctypes
import importlib

import numpy as np
import pytest

from tests import hostbuild
from tests.locate_util import (GUARD, MAX_POINTS, SENTINEL_F, SENTINEL_I, bits, check_guards, compare_to_oracle, count_cases,
                               edge_scenes, equal_but_heading, fold_allowed, fuzz_scenes, guarded_outputs, host_locate_batch,
                               large_scenes, oracle, pack, small_scenes)

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
OK, EINVAL = 0, -1


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


@pytest.fixture(scope="module")
def lib():
    return hostbuild.load("locate")


def _ctx(R):
    return pkg.MocapContext(2, 640, 480, max_roots=R)


def _inputs(torch, obj, err, n):
    return torch.from_numpy(obj).cuda(), torch.from_numpy(err).cuda(), torch.from_numpy(n).cuda()


def _device(torch, ctx, obj, err, n, max_objects):
    d = ctx.locate_objects(*_inputs(torch, obj, err, n), max_objects=max_objects)
    return {k: v.cpu().numpy() for k, v in d.items()}


def _same_bits(a, b):
    """Two device runs: counts and every valid record bit-equal, the heading too."""
    assert np.array_equal(a["n"], b["n"])
    valid = np.arange(a["objects"].shape[1])[None, :] < a["n"][:, None]
    assert np.array_equal(bits(a["objects"][valid]), bits(b["objects"][valid]))
    assert np.array_equal(a["drone_index"][valid], b["drone_index"][valid])


def _fold_sets(names):
    return [s for s, k in enumerate(names) if fold_allowed(k)]


# ---------------------------------------------------------------------------------------------- scenes
@pytest.mark.parametrize("R", [16, 64, MAX_POINTS])
def test_device_equals_the_oracle_and_the_host_build_on_the_edge_scenes(torch, lib, R, capsys):
    named = {k: v for k, v in edge_scenes().items() if len(v[0]) <= R}
    names, scenes = list(named), list(named.values())
    obj, err, n = pack(scenes, R)
    got = _device(torch, _ctx(R), obj, err, n, R)
    total, cut, worst = compare_to_oracle(got, scenes, R, names)
    equal_but_heading(host_locate_batch(lib, obj, err, n, R, R), got, _fold_sets(names))
    with capsys.disabled():
        print(f"\nmax_roots {R}: {len(names)} edge scenes, {total} objects, worst heading difference to the oracle {worst:.2e}")
    assert cut == 0 and total >= {16: 90, 64: 90, MAX_POINTS: 700}[R]


@pytest.mark.parametrize("B", [1, 127, 128, 129])
def test_batch_sizes_around_one_block(torch, lib, B):
    """The edge scenes, the 128-point ones first, repeated to B frame-sets: one thread short of a block, a full block,
    one thread into the next."""
    named = {**large_scenes(), **small_scenes()}
    names = [list(named)[s % len(named)] for s in range(B)]
    scenes = [named[k] for k in names]
    obj, err, n = pack(scenes, MAX_POINTS)
    got = _device(torch, _ctx(MAX_POINTS), obj, err, n, MAX_POINTS)
    compare_to_oracle(got, scenes, MAX_POINTS, names)
    equal_but_heading(host_locate_batch(lib, obj, err, n, MAX_POINTS, MAX_POINTS), got, _fold_sets(names))


def test_100000_frame_sets(torch):
    """782 blocks: the small edge scenes tiled; the first copy equals the oracle and every copy equals the first."""
    named = small_scenes()
    names, scenes = list(named), list(named.values())
    B, R, S = 100_000, 16, len(named)
    obj, err, n = pack(scenes, R)
    idx = np.arange(B) % S
    ctx = _ctx(R)
    got = _device(torch, ctx, obj[idx], err[idx], n[idx], R)
    first = {k: v[:S] for k, v in got.items()}
    compare_to_oracle(first, scenes, R, names)
    _same_bits(got, {k: v[idx] for k, v in first.items()})


@pytest.mark.parametrize("R", [16, 64, MAX_POINTS])
def test_frame_set_counts(torch, lib, R):
    """n_obj of 0, 1, 2, max_roots, max_roots + 5 and -1 over rows that hold valid triplets throughout."""
    seen, (obj, err, n) = count_cases(R)
    assert n.max() == R + 5 and n.min() == -1
    got = _device(torch, _ctx(R), obj, err, n, R)
    compare_to_oracle(got, seen, R)
    assert list(got["n"][[0, 1, 2, 6]]) == [0, 0, 0, 0] and got["n"][4] == 1 and got["n"][5] == 1
    equal_but_heading(host_locate_batch(lib, obj, err, n, R, R), got)


def test_fuzz(torch, lib, capsys):
    """The 2000 seeded scenes of the host test, one object slot per point and 4 slots."""
    scenes = fuzz_scenes()
    obj, err, n = pack(scenes, MAX_POINTS)
    ctx = _ctx(MAX_POINTS)
    got = _device(torch, ctx, obj, err, n, MAX_POINTS)
    total, cut, worst = compare_to_oracle(got, scenes, MAX_POINTS)
    equal_but_heading(host_locate_batch(lib, obj, err, n, MAX_POINTS, MAX_POINTS), got)
    few = _device(torch, ctx, obj, err, n, 4)
    _, cut4, _ = compare_to_oracle(few, scenes, 4)
    with capsys.disabled():
        print(f"\nfuzz: {len(scenes)} scenes, {total} objects, worst heading difference to the oracle {worst:.2e}, "
              f"{cut4} scenes truncated at 4 objects")
    assert cut == 0 and total > 40000 and cut4 > 1200


# ---------------------------------------------------------------------------------------------- truncation, guards
def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize("max_objects", [1, 3, 40])
def test_truncation_writes_nothing_past_its_records(torch, max_objects):
    """Outputs with sentinel rows after every frame-set's records, in one tensor; each frame-set is located into its
    own view of it.  More objects than max_objects: the oracle's first max_objects, n == max_objects; every guard row
    and every slot at or beyond n keeps its sentinel.  Then the whole batch in one call, a guard slab after it."""
    named = edge_scenes()
    names, scenes = list(named), list(named.values())
    B = len(scenes)
    obj, err, n = pack(scenes, MAX_POINTS)
    tobj, terr, tn = _inputs(torch, obj, err, n)
    ctx = _ctx(MAX_POINTS)
    ctx.use_current_stream()
    rec, di, cnt = guarded_outputs(B, max_objects, xp=torch, device="cuda")
    for s in range(B):
        assert ctx.lib.mocap_locate_objects_dev(ctx.h, _p(tobj[s]), _p(terr[s]), _p(tn[s:]), 1, max_objects,
                                                _p(rec[s]), _p(di[s]), _p(cnt[s:])) == OK
    torch.cuda.synchronize()
    rec, di, cnt = rec.cpu().numpy(), di.cpu().numpy(), cnt.cpu().numpy()
    check_guards(rec, di, cnt, B, max_objects)
    got = {"objects": rec[:B, :max_objects], "drone_index": di[:B, :max_objects], "n": cnt[:B]}
    _, cut, _ = compare_to_oracle(got, scenes, max_objects, names)
    assert cut >= (9 if max_objects == 40 else 14)
    assert all(got["n"][s] == max_objects for s, sc in enumerate(scenes) if oracle(*sc)[0] > max_objects)
    # the dense layout: frame-set s at row s * max_objects, sentinel rows for GUARD more frame-sets behind the last
    rec2, di2, cnt2 = guarded_outputs(B + GUARD, max_objects, xp=torch, device="cuda")
    assert ctx.lib.mocap_locate_objects_dev(ctx.h, _p(tobj), _p(terr), _p(tn), B, max_objects, _p(rec2), _p(di2), _p(cnt2)) == OK
    torch.cuda.synchronize()
    flat = rec2.cpu().numpy().reshape(-1, 5); flat_di = di2.cpu().numpy().reshape(-1); cnt2 = cnt2.cpu().numpy()
    dense = {"objects": flat[:B * max_objects].reshape(B, max_objects, 5), "drone_index": flat_di[:B * max_objects].reshape(B, max_objects),
             "n": cnt2[:B]}
    _same_bits(got, dense)
    assert (flat[B * max_objects:] == SENTINEL_F).all() and (flat_di[B * max_objects:] == SENTINEL_I).all()
    assert (cnt2[B:] == SENTINEL_I).all()


# ---------------------------------------------------------------------------------------------- streams, launches
def test_side_stream_and_second_run_give_the_same_bits(torch):
    named = edge_scenes()
    obj, err, n = pack(list(named.values()), MAX_POINTS)
    ctx = _ctx(MAX_POINTS)
    want = _device(torch, ctx, obj, err, n, 64)
    _same_bits(want, _device(torch, ctx, obj, err, n, 64))
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d = ctx.locate_objects(*_inputs(torch, obj, err, n), max_objects=64)
    side.synchronize()
    _same_bits(want, {k: v.cpu().numpy() for k, v in d.items()})
    _same_bits(want, _device(torch, _ctx(MAX_POINTS), obj, err, n, 64))


def test_one_launch_per_call(torch):
    ctx = _ctx(16)
    scenes = list(small_scenes().values())
    for B in (1, 128, 129, 5000):
        obj, err, n = pack([scenes[s % len(scenes)] for s in range(B)], 16)
        args = _inputs(torch, obj, err, n)
        before = ctx.launch_count()
        ctx.locate_objects(*args, max_objects=8)
        assert ctx.launch_count() - before == 1, B
    torch.cuda.synchronize()


def test_refusals_launch_nothing(torch):
    """Null pointers, max_objects < 1 and n_frame_sets < 0 are MOCAP_EINVAL; n_frame_sets == 0 is OK; none launches or
    touches the outputs."""
    ctx = _ctx(16)
    ctx.use_current_stream()
    obj, err, n = pack(list(small_scenes().values())[:4], 16)
    tobj, terr, tn = _inputs(torch, obj, err, n)
    rec, di, cnt = guarded_outputs(4, 8, xp=torch, device="cuda")
    args = [_p(tobj), _p(terr), _p(tn), 4, 8, _p(rec), _p(di), _p(cnt)]
    before = ctx.launch_count()
    for i in (0, 1, 2, 5, 6, 7):
        bad = list(args)
        bad[i] = ctypes.c_void_p(0)
        assert ctx.lib.mocap_locate_objects_dev(ctx.h, *bad) == EINVAL, i
    for i, v in ((4, 0), (4, -1), (3, -1), (3, -100)):
        bad = list(args)
        bad[i] = v
        assert ctx.lib.mocap_locate_objects_dev(ctx.h, *bad) == EINVAL, (i, v)
    assert ctx.lib.mocap_locate_objects_dev(None, *args) == EINVAL
    none = list(args)
    none[3] = 0
    assert ctx.lib.mocap_locate_objects_dev(ctx.h, *none) == OK
    assert ctx.launch_count() == before
    torch.cuda.synchronize()
    sent = guarded_outputs(4, 8)
    for t, s in zip((rec, di, cnt), sent):
        assert np.array_equal(t.cpu().numpy(), s)
    assert ctx.lib.mocap_locate_objects_dev(ctx.h, *args) == OK
    assert ctx.launch_count() == before + 1
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- drop-in
def test_drop_in_on_a_crowded_128_point_scene(torch):
    """pkg.locate_objects sizes its output at one object per point: on 128 crowded points and on the lattice (105
    objects) it returns the oracle's list; 129 points are refused."""
    s = pkg.MocapSession([np.eye(3)] * 2)
    for name in ("crowded_40_full", "lattice_8x16", "straddle_63_64_127"):
        pts, errs = large_scenes()[name]
        got = pkg.locate_objects(pts, errs, session=s)
        k, rec, di = oracle(pts, errs)
        assert len(got) == k >= 55
        for g, r, d in zip(got, rec, di):
            assert set(g) == {"pos", "heading", "error", "droneIndex"} and g["droneIndex"] == d
            assert np.array_equal(bits(g["pos"]), bits(r[:3])) and g["error"] == r[4]
            assert abs(g["heading"] - r[3]) <= 4 * np.spacing(np.pi / 2)
    pts, errs = large_scenes()["crowded_40_full"]
    with pytest.raises(pkg.MocapError):
        pkg.locate_objects(np.vstack([pts, [[0.0, 0.0, 0.0]]]), np.append(errs, 0.1), session=s)
    assert pkg.locate_objects(np.zeros((0, 3)), np.zeros(0), session=s) == []

"""The capture-side preprocessing kernel itself (csrc/preproc.cu k_preprocess, stages in csrc/preproc_tile.cuh)
against the reference's cv2 chain (helpers.py:70-82, restated by oracle.ref_port.RefPort.preprocess), bit for bit:
cameras that share nothing, every regime of frame size, partial frame-sets, the byte-store path, the grey plane S1
reads, the split into several launches, and ordering on a side stream.  tests/test_host_cpu.py steps the same stages
through on the host; this file runs the device code.  Run with ``-m gpu`` on an H100."""
import ctypes as C
import importlib

import numpy as np
import pytest

from tests.preproc_util import FRAME_KINDS, cv2_chain, frame, marker_frames, rig, rig_poses

pytestmark = pytest.mark.gpu

pkg = importlib.import_module("low-cost-mocap_b200")
api = importlib.import_module("low-cost-mocap_b200.api")

CANARY = 0xA5
PP_F = 2                                  # frames of one camera per CTA (preproc_tile.cuh): B = 3 leaves a one-frame group
# square sizes: below one 64-px tile, ragged right / bottom tiles, the common 320, and the largest square a context
# accepts (width * height / 16 <= 65535 rules out 1024); each with its own number of cameras
GEOMETRIES = {48: 8, 80: 5, 208: 3, 320: 3, 336: 8, 496: 5, 1008: 3}
THRESHOLDS = (0, 1, 51, 127, 200, 254)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs an H100 (run with -m gpu)")
    return torch


def _in_heights(S):
    """1 row, an odd height near S / 2, and the tallest frame make_square feathers (8 pad rows above and below): the
    make_square offset (S - in_h) / 2 is odd for the first two and 8 for the last."""
    mid = S // 2 + 1 if (S // 2) % 2 == 0 else S // 2
    return (1, mid, S - 16)


def _same(got, want, case):
    assert got.shape == want.shape, (case, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = got != want
        lead = bad.reshape(bad.shape[0], -1).any(axis=1) if bad.ndim > 1 else bad
        pytest.fail(f"{case}: {int(bad.sum())} of {bad.size} bytes differ (first differing index along axis 0: "
                    f"{int(np.argmax(lead))})")


def _ctx(Cn, S, in_h, Ks, dists, rots, **kw):
    ctx = pkg.MocapContext(Cn, S, S, max_blobs=64, **kw)
    ctx.set_preprocess(S, in_h, rots, Ks, dists)
    return ctx


def _check_maps(ctx, S, Ks, dists, case):
    """undistort_map(c) is cv2.initUndistortRectifyMap(..., CV_16SC2) of camera c's own K and distortion."""
    import cv2
    maps = []
    for c, (K, d) in enumerate(zip(Ks, dists)):
        m1, m2 = ctx.undistort_map(c)
        r1, r2 = cv2.initUndistortRectifyMap(K, np.asarray(d, dtype=np.float64), np.eye(3), K, (S, S), cv2.CV_16SC2)
        _same(m1, r1, (case, "m1 of camera", c))
        _same(m2, r2, (case, "m2 of camera", c))
        maps.append(m1)
    return maps


def _frames(rng, B, Cn, in_h, S):
    """[B, C, in_h, S, 3]: every kind of frame on every camera across the batch."""
    return np.stack([np.stack([frame(rng, FRAME_KINDS[(b + c) % len(FRAME_KINDS)], in_h, S) for c in range(Cn)]) for b in range(B)])


def _preprocess_dev(ctx, raw_ptr, n, out_ptr):
    """mocap_preprocess_dev through the C ABI with raw pointers (any n, any alignment), on torch's current stream."""
    ctx.use_current_stream()
    ctx._check(ctx.lib.mocap_preprocess_dev(ctx.h, C.c_void_p(raw_ptr), int(n), C.c_void_p(out_ptr)))


# ---------------------------------------------------------------------------------------------- cameras, sizes
@pytest.mark.parametrize("Cn", [3, 5, 8])
def test_every_camera_uses_its_own_map_and_rotation(torch, Cn):
    """Every camera its own K, distortion and rotation (8 cameras: one whose map reaches the int16 clamp): the device
    maps equal cv2's, and every processed frame equals the cv2 chain with its own camera's parameters, for B = 3
    (a one-frame last group) and B = 1."""
    S, in_h = 208, 101
    rng = np.random.default_rng(100 + Cn)
    Ks, dists, rots = rig(rng, Cn, S, clamp=Cn == 8)
    ctx = _ctx(Cn, S, in_h, Ks, dists, rots)
    maps = _check_maps(ctx, S, Ks, dists, ("cameras", Cn))
    assert any(((m < 0) | (m >= S)).any() for m in maps)                     # some map leaves the frame
    if Cn == 8:
        assert (maps[-1] == 32767).any() and (maps[-1] == -32768).any()      # and one reaches the clamp
    assert len({(tuple(K.ravel()), tuple(d)) for K, d in zip(Ks, dists)}) == Cn and len(set(rots)) == 2
    raw = _frames(rng, 3, Cn, in_h, S)
    want = cv2_chain(raw, Ks, dists, rots)
    raw_d = torch.from_numpy(raw).cuda()
    for B in (3, 1):
        got = ctx.preprocess(raw_d[:B]).cpu().numpy().reshape(B, Cn, S, S, 3)
        for b in range(B):
            for c in range(Cn):
                _same(got[b, c], want[b, c], ("cameras", Cn, "B", B, "frame", b, "camera", c, "rot", rots[c]))


@pytest.mark.parametrize("S", sorted(GEOMETRIES))
def test_every_frame_size_equals_cv2(torch, S):
    """Each square size with raw heights 1, odd near S / 2 and S - 16; noise, saturated, zero and binary frames on
    cameras that share nothing; B = 3 and B = 1."""
    Cn = GEOMETRIES[S]
    for in_h in _in_heights(S):
        case = ("S", S, "in_h", in_h, "C", Cn)
        rng = np.random.default_rng(S * 1000 + in_h)
        Ks, dists, rots = rig(rng, Cn, S)
        ctx = _ctx(Cn, S, in_h, Ks, dists, rots)
        _check_maps(ctx, S, Ks, dists, case)
        raw = _frames(rng, 3, Cn, in_h, S)
        want = cv2_chain(raw, Ks, dists, rots)
        raw_d = torch.from_numpy(raw).cuda()
        for B in (3, 1):
            got = ctx.preprocess(raw_d[:B]).cpu().numpy().reshape(B, Cn, S, S, 3)
            _same(got, want[:B], case + ("B", B, "rot", rots))
        ctx.close()


# ---------------------------------------------------------------------------------------------- partial sets, stores
@pytest.mark.parametrize("Cn", [3, 5])
def test_partial_frame_sets_leave_the_tail_untouched(torch, Cn):
    """n_images below a whole number of frame-sets (C B - 1, and fewer than one frame-set): the frames below n equal
    cv2, and the output past them -- at least one whole frame -- keeps its canary.  The raw buffer holds whole
    frame-sets, the output buffer whole frame-sets plus one frame, so a kernel that guarded only on the frame-set
    would read and write in bounds, and be caught by the canary."""
    S, in_h, B = 80, 41, 3
    rng = np.random.default_rng(300 + Cn)
    Ks, dists, rots = rig(rng, Cn, S)
    ctx = _ctx(Cn, S, in_h, Ks, dists, rots)
    raw = _frames(rng, B, Cn, in_h, S)
    want = cv2_chain(raw, Ks, dists, rots).reshape(B * Cn, S, S, 3)
    raw_d = torch.from_numpy(raw).cuda()
    frame_bytes = S * S * 3
    out = torch.empty((B * Cn + 1) * frame_bytes, dtype=torch.uint8, device="cuda")
    for n in (Cn * B - 1, Cn + 1, Cn - 1, 1):
        out.fill_(CANARY)
        _preprocess_dev(ctx, raw_d.data_ptr(), n, out.data_ptr())
        got = out.cpu().numpy()
        _same(got[:n * frame_bytes].reshape(n, S, S, 3), want[:n], ("partial", Cn, "n", n))
        tail = got[n * frame_bytes:]
        assert (tail == CANARY).all(), ("partial", Cn, "n", n, "bytes past n written:", int((tail != CANARY).sum()))


@pytest.mark.parametrize("S", [48, 80])
def test_unaligned_output_takes_the_byte_stores(torch, S):
    """Output at data_ptr() + 1 and + 2 (the kernel falls back from word to byte stores) and raw frames at an odd
    offset: the same bytes as the aligned call, those equal cv2, and nothing written outside the output.  The grey
    plane always lives in the context's aligned scratch, so no entry point takes its byte-store path."""
    Cn, B = 3, 3
    in_h = _in_heights(S)[1]
    rng = np.random.default_rng(400 + S)
    Ks, dists, rots = rig(rng, Cn, S)
    ctx = _ctx(Cn, S, in_h, Ks, dists, rots)
    raw = _frames(rng, B, Cn, in_h, S)
    want = cv2_chain(raw, Ks, dists, rots).reshape(-1)
    n = B * Cn
    N = want.size
    raw_d = torch.from_numpy(raw).cuda().reshape(-1)
    aligned = ctx.preprocess(raw_d).cpu().numpy().reshape(-1)
    _same(aligned, want, ("aligned", S))
    raw_odd = torch.empty(raw_d.numel() + 1, dtype=torch.uint8, device="cuda")
    raw_odd[1:] = raw_d
    buf = torch.empty(N + 8, dtype=torch.uint8, device="cuda")
    for raw_off, out_off in ((0, 1), (0, 2), (1, 0), (1, 3)):
        buf.fill_(CANARY)
        src = raw_odd.data_ptr() + 1 if raw_off else raw_d.data_ptr()
        _preprocess_dev(ctx, src, n, buf.data_ptr() + out_off)
        got = buf.cpu().numpy()
        case = ("S", S, "raw offset", raw_off, "output offset", out_off)
        _same(got[out_off:out_off + N], aligned, case)
        outside = np.concatenate([got[:out_off], got[out_off + N:]])
        assert (outside == CANARY).all(), case + ("bytes written outside the output:", int((outside != CANARY).sum()))


# ---------------------------------------------------------------------------------------------- the grey plane
@pytest.mark.parametrize("S", sorted(GEOMETRIES))
def test_grey_plane_feeds_s1_as_cv2_frames_do(torch, S):
    """No entry point returns the grey plane the kernel writes for S1, so it is checked through S1-S3: on marker
    frames (bright spots projected from 3D points through each camera's K, distortion and rotation),
    pipeline_raw(raw, t) equals pipeline(cv2 frames, t) bit for bit in n, flags, obj and err, at every threshold;
    a live(..., CAPTURE) read of the raw frames gives the blob counts and first centres of S1 on the cv2 frames."""
    Cn = GEOMETRIES[S]
    matched = 0
    for in_h in _in_heights(S):
        rng = np.random.default_rng(500 + S * 1000 + in_h)
        Ks, dists, rots = rig(rng, Cn, S)
        poses = rig_poses(Cn)
        B = 3
        raw = marker_frames(rng, B, S, in_h, Ks, dists, rots, poses)
        frames = cv2_chain(raw, Ks, dists, rots)
        # two contexts with the same history, so that the pipeline picks the same kernels for both
        ctx_raw = _ctx(Cn, S, in_h, Ks, dists, rots)
        ctx_ref = _ctx(Cn, S, in_h, Ks, dists, rots)
        for c in (ctx_raw, ctx_ref):
            c.set_cameras(Ks, poses)
        raw_d = torch.from_numpy(raw).cuda()
        frames_d = torch.from_numpy(frames).cuda()
        for t in THRESHOLDS:
            case = ("S", S, "in_h", in_h, "C", Cn, "threshold", t)
            a = ctx_raw.pipeline_raw(raw_d, threshold=t)
            b = ctx_ref.pipeline(frames_d, threshold=t)
            n = a["n"].cpu().numpy()
            _same(n, b["n"].cpu().numpy(), case + ("n",))
            _same(a["flags"].cpu().numpy(), b["flags"].cpu().numpy(), case + ("flags",))
            for key in ("obj", "err"):
                ga, gb = a[key].cpu().numpy(), b[key].cpu().numpy()
                for s in range(B):
                    _same(ga[s, :n[s]].view(np.uint64), gb[s, :n[s]].view(np.uint64), case + (key, "frame-set", s))
            if t == api.THRESHOLD:
                matched += int(n.sum())
        live = ctx_raw.live(raw_d, api.LIVE_CAPTURE)
        det = ctx_ref.detect(frames_d)
        cnt = det["n"].cpu().numpy().reshape(B, Cn)
        first = np.where(cnt[:, :, None] > 0, det["xy"].cpu().numpy()[:, 0].reshape(B, Cn, 2), -1)
        case = ("S", S, "in_h", in_h, "C", Cn, "live")
        _same(live["blob_n"].cpu().numpy(), cnt, case + ("blob_n",))
        _same(live["first"].cpu().numpy(), first, case + ("first",))
        ctx_raw.close(); ctx_ref.close()
    assert matched > 0, ("S", S, "no frame-set triangulated a point: S2 and S3 did not run")


# ---------------------------------------------------------------------------------------------- the launch split
@pytest.mark.parametrize("Cn", [1, 3])
def test_launch_split(torch, Cn):
    """More images than one launch takes ((65535 // C) groups of 2 frames per camera, about 131 000 images of 32 x 16):
    two launches, the second ending in a partial group (and for C = 3 a partial frame-set), then a call of exactly one
    launch's worth.  Each image comes from a pool of 64 distinct noise frames per camera, picked by a hash of its index
    so that nothing repeats with the launch period; every output image equals cv2's processing of its pool frame, and the
    frame past the last image keeps its canary."""
    S, in_w, in_h, P = 32, 32, 16, 64
    rng = np.random.default_rng(600 + Cn)
    Ks, dists, rots = rig(rng, Cn, S)
    ctx = _ctx(Cn, S, in_h, Ks, dists, rots)
    pool = np.stack([np.stack([frame(rng, ("noise", "binary")[p % 2], in_h, in_w) for p in range(P)]) for c in range(Cn)])
    want_pool = np.stack([cv2_chain(pool[c][:, None], [Ks[c]], [dists[c]], [rots[c]])[:, 0] for c in range(Cn)])   # [C, P, S, S, 3]
    per_launch = (65535 // Cn) * PP_F * Cn
    n_split = per_launch + 17 * Cn - (1 if Cn > 1 else 0)                     # 17 frame-sets after the boundary: 9 groups, the
    n_alloc = -(-n_split // Cn) * Cn                                          # last of one frame-set, partial for C = 3
    i = np.arange(n_alloc, dtype=np.uint64)
    entry = torch.from_numpy((((i * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(26)).astype(np.int64)).cuda()
    cam = torch.arange(n_alloc, device="cuda") % Cn
    raw_d = torch.from_numpy(pool).cuda()[cam, entry].contiguous()          # [n_alloc, in_h, in_w, 3]
    want_d = torch.from_numpy(want_pool).cuda()[cam, entry]                 # [n_alloc, S, S, 3]
    out = torch.empty((n_alloc + 1, S, S, 3), dtype=torch.uint8, device="cuda")
    for n, launches in ((n_split, 2), (per_launch, 1)):
        out.fill_(CANARY)
        before = ctx.launch_count()
        _preprocess_dev(ctx, raw_d.data_ptr(), n, out.data_ptr())
        assert ctx.launch_count() - before == launches, ("split", Cn, n)
        bad = (out[:n] != want_d[:n]).reshape(n, -1).any(dim=1).nonzero().flatten().cpu().numpy()
        assert bad.size == 0, ("split", Cn, "n", n, "images differing:", int(bad.size), "first:", bad[:8].tolist())
        tail = int((out[n:] != CANARY).sum())
        assert tail == 0, ("split", Cn, "n", n, "bytes past n written:", tail)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- ordering, reconfiguration
def test_side_stream_after_a_kernel_that_writes_the_raw_frames(torch):
    """The raw frames are written by a kernel on a side stream right before the call (after a spin that keeps that
    stream busy): preprocessing enqueued on the side stream reads them after they are written and gives the default
    stream's bytes."""
    S, in_h, Cn, B = 208, 101, 3, 4
    rng = np.random.default_rng(700)
    Ks, dists, rots = rig(rng, Cn, S)
    ctx = _ctx(Cn, S, in_h, Ks, dists, rots)
    raw = _frames(rng, B, Cn, in_h, S)
    want = ctx.preprocess(torch.from_numpy(raw).cuda()).cpu().numpy()
    _same(want.reshape(B, Cn, S, S, 3), cv2_chain(raw, Ks, dists, rots), ("default stream",))
    masked = torch.from_numpy(raw ^ np.uint8(0x5A)).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)
        raw_side = torch.bitwise_xor(masked, 0x5A)
        got = ctx.preprocess(raw_side)
    side.synchronize()
    _same(got.cpu().numpy(), want, ("side stream",))


def test_set_preprocess_again_leaves_nothing_of_the_first(torch):
    """A second set_preprocess on the same context (other raw height, other rotations, other maps) gives what a fresh
    context with only the second setting gives, and cv2's frames: no map or rotation of the first survives."""
    S, Cn, B = 80, 5, 3
    rng = np.random.default_rng(800)
    first = rig(rng, Cn, S)
    Ks, dists, _ = rig(rng, Cn, S)
    rots = [2 - r for r in first[2]]
    ctx = _ctx(Cn, S, 64, *first)
    ctx.preprocess(torch.from_numpy(_frames(rng, B, Cn, 64, S)).cuda())
    ctx.set_preprocess(S, 41, rots, Ks, dists)
    fresh = _ctx(Cn, S, 41, Ks, dists, rots)
    for c in range(Cn):
        for a, b in zip(ctx.undistort_map(c), fresh.undistort_map(c)):
            _same(a, b, ("map after reconfiguration", c))
    _check_maps(ctx, S, Ks, dists, ("reconfigured",))
    raw = _frames(rng, B, Cn, 41, S)
    raw_d = torch.from_numpy(raw).cuda()
    got = ctx.preprocess(raw_d).cpu().numpy()
    _same(got, fresh.preprocess(raw_d).cpu().numpy(), ("reconfigured vs fresh",))
    _same(got.reshape(B, Cn, S, S, 3), cv2_chain(raw, Ks, dists, rots), ("reconfigured vs cv2", rots))

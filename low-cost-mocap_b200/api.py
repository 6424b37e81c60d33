"""Host-side mirror of the reference's hot-path call surface on top of libmocap_b200.so.

Two layers:

* :class:`MocapContext` -- the batched API the benchmark and the multi-GPU driver use:
  device (torch) tensors in, device tensors out, no synchronisation.
* module-level functions with the reference's own names, arguments and return values
  (computer_code/api/helpers.py), bound to a :class:`MocapSession` that plays the part
  of the reference's ``Cameras`` singleton for this path.  ``install_into(helpers)``
  monkey-patches a loaded reference ``helpers`` module so that ``index.py``, the UI and
  the drone loop run unchanged on the CUDA path (INTEGRATION.md).

torch is used for device memory and streams only.  There is no CPU fallback: every
function raises :class:`MocapError` when the library or the GPU is missing.
"""
from __future__ import annotations

import ctypes as C
import json
import threading
import time

import numpy as np

from . import _lib
from ._lib import MocapError, Config, BAOptions, BAProblem, BAReport, RansacOptions, GraphOptions, GraphPair, LiveLayout, check

THRESHOLD = 51   # cv.threshold(grey, 255*0.2, 255, THRESH_BINARY) on uint8 == pix > 51 (helpers.py:146)

# MOCAP_F_* bits of include/mocap_b200.h
F_SEGMENTS, F_BLOBS, F_ROOTS, F_CANDS, F_GROUPS, F_HOLES = 1, 2, 4, 8, 16, 32
_FLAG_NAMES = {F_SEGMENTS: "max_segments", F_BLOBS: "max_blobs", F_ROOTS: "max_roots", F_CANDS: "max_cands",
               F_GROUPS: "max_groups"}
# mode bits of mocap_live_dev (include/mocap_b200.h): Cameras.is_capturing_points, is_triangulating_points,
# is_locating_objects, as the reference nests them (helpers.py:84-106)
LIVE_CAPTURE, LIVE_TRIANGULATE, LIVE_LOCATE = 1, 2, 4
# cv2's default IMWRITE_JPEG_QUALITY, what index.py's cv.imencode('.jpg', frames) (index.py:56) encodes at
JPEG_QUALITY = 95
# the reference is unbounded; the drop-in mirrors run with the compile-time maxima and raise on overflow
MIRROR_LIMITS = dict(max_blobs=64, max_segments=4096, max_roots=128, max_cands=16, max_groups=1 << 16)


def raise_on_overflow(flags, what):
    """The reference keeps every contour / root / candidate group; a result truncated at a configured
    capacity would differ from it silently, so the mirrors turn any MOCAP_F_* bit into an error."""
    flags = int(flags)
    if flags & F_HOLES:
        raise MocapError(-1, f"{what}: a blob with a hole is too large for the RETR_TREE slow path (wider or taller than 62 pixels, "
                             f"or more than 64 holes in the image); cv.findContours would give each hole a contour of its own "
                             f"and fill the outer one (MOCAP_F_HOLES; large_holes=True lifts the size limit)")
    if flags:
        names = [n for b, n in _FLAG_NAMES.items() if flags & b]
        raise MocapError(-1, f"{what}: capacity overflow ({', '.join(names)}); results would be truncated "
                             f"where the reference is unbounded")


def _torch():
    import torch
    return torch


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _np_ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else C.c_void_p(0)


def _report_dict(rep):
    d = {f: getattr(rep, f) for f, _ in BAReport._fields_}
    d["phase_ms"] = [float(v) for v in rep.phase_ms]
    return d


class MocapContext:
    """One libmocap_b200 context (one CUDA device, one stream, one camera rig)."""

    def __init__(self, n_cam, width=640, height=480, device=0, max_blobs=None, max_segments=None,
                 max_roots=None, max_cands=None, max_groups=None):
        self.lib = _lib.load()
        cfg = Config()
        self.lib.mocap_default_config(C.byref(cfg), n_cam, width, height)
        cfg.device = device
        for k, v in dict(max_blobs=max_blobs, max_segments=max_segments, max_roots=max_roots,
                         max_cands=max_cands, max_groups=max_groups).items():
            if v is not None:
                setattr(cfg, k, v)
        self.cfg = cfg
        h = C.c_void_p()
        check(self.lib.mocap_create(C.byref(h), C.byref(cfg)))
        self.h = h
        self.n_cam, self.width, self.height = n_cam, width, height
        self.device = device
        self._tdev = None
        self._pp_in = None
        self.large_holes = False

    # -- lifetime -------------------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.lib.mocap_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st):
        check(st, self.h)

    @property
    def torch_device(self):
        if self._tdev is None:
            self._tdev = _torch().device("cuda", self.device)
        return self._tdev

    def use_current_stream(self):
        """Enqueue on torch's current stream of this device."""
        s = _torch().cuda.current_stream(self.torch_device)
        self._check(self.lib.mocap_set_stream(self.h, C.c_void_p(s.cuda_stream)))

    # -- session state --------------------------------------------------------------------
    def set_large_holes(self, on=True):
        """Reproduce cv.findContours(RETR_TREE) for holed blobs wider or taller than 62 pixels too (helpers.py:147-158),
        in every S1 entry point of this context: a whole-image window for the slow path, about 166 KB of device memory
        per SM at 640 x 480.  Off (the default) such an image keeps MOCAP_F_HOLES.  ``on=False`` frees the window
        (mocap_set_large_holes, include/mocap_b200.h)."""
        self._check(self.lib.mocap_set_large_holes(self.h, 1 if on else 0))
        self.large_holes = bool(on)

    def set_cameras(self, intrinsics, poses):
        """intrinsics: C 3x3 matrices; poses: list of {"R": 3x3, "t": 3} as the reference passes them."""
        n = self.n_cam
        K = np.ascontiguousarray(np.stack([np.asarray(k, dtype=np.float64).reshape(3, 3) for k in intrinsics]))
        R = np.ascontiguousarray(np.stack([np.asarray(p["R"], dtype=np.float64).reshape(3, 3) for p in poses]))
        t = np.ascontiguousarray(np.stack([np.asarray(p["t"], dtype=np.float64).reshape(3) for p in poses]))
        if K.shape[0] != n or R.shape[0] != n:
            raise ValueError(f"context was created for {n} cameras")
        self._check(self.lib.mocap_set_cameras(self.h, _np_ptr(K), _np_ptr(R), _np_ptr(t)))

    def set_world_transform(self, M):
        if M is None:
            self._check(self.lib.mocap_set_world_transform(self.h, C.c_void_p(0)))
        else:
            M = np.ascontiguousarray(np.asarray(M, dtype=np.float64).reshape(4, 4))
            self._check(self.lib.mocap_set_world_transform(self.h, _np_ptr(M)))

    # -- capture-side preprocessing (helpers.py:70-82) -------------------------------------
    def set_preprocess(self, in_width, in_height, rotations, intrinsics, distortions):
        rot = np.ascontiguousarray(np.asarray(rotations, dtype=np.int32).reshape(self.n_cam))
        K = np.ascontiguousarray(np.stack([np.asarray(k, dtype=np.float64).reshape(3, 3) for k in intrinsics]))
        D = np.ascontiguousarray(np.stack([np.asarray(d, dtype=np.float64).reshape(5) for d in distortions]))
        self._check(self.lib.mocap_set_preprocess(self.h, int(in_width), int(in_height), _np_ptr(rot), _np_ptr(K), _np_ptr(D)))
        self._pp_in = (int(in_height), int(in_width))

    def preprocess(self, raw):
        """raw uint8 cuda tensor [..., in_h, in_w, 3] (whole frame-sets) -> uint8 [N, S, S, 3]."""
        torch = _torch()
        if self._pp_in is None:
            raise MocapError(-5, "mocap_set_preprocess has not been called (MocapContext.set_preprocess)")
        h, w = self._pp_in
        n = raw.numel() // (h * w * 3)
        out = torch.empty((n, self.height, self.width, 3), dtype=torch.uint8, device=raw.device)
        self.use_current_stream()
        self._check(self.lib.mocap_preprocess_dev(self.h, _ptr(raw.contiguous()), n, _ptr(out)))
        return out

    def pipeline_raw(self, raw, threshold=THRESHOLD, want_frames=False):
        """Raw camera frames uint8 cuda [B, C, in_h, in_w, 3] -> tracks (and the processed frames)."""
        torch = _torch()
        if self._pp_in is None:
            raise MocapError(-5, "mocap_set_preprocess has not been called (MocapContext.set_preprocess)")
        h, w = self._pp_in
        B = raw.numel() // (self.n_cam * h * w * 3)
        out = self.alloc_tracks(B, raw.device)
        frames = torch.empty((B, self.n_cam, self.height, self.width, 3), dtype=torch.uint8, device=raw.device) if want_frames else None
        self.use_current_stream()
        self._check(self.lib.mocap_pipeline_raw_dev(self.h, _ptr(raw.contiguous()), B, int(threshold), _ptr(frames),
                                                    _ptr(out["obj"]), _ptr(out["err"]), _ptr(out["n"]), _ptr(out["flags"])))
        if want_frames:
            out["frames"] = frames
        return out

    # -- the live capture loop (helpers.py:68-135) ---------------------------------------------
    def live_layout(self, n_reads, num_objects=0):
        """Byte offsets of the slices of a mocap_live_dev result buffer and its size (``total``)."""
        L = LiveLayout()
        self._check(self.lib.mocap_live_layout(self.h, int(n_reads), int(num_objects), C.byref(L)))
        return L

    def _live_views(self, buf, n_reads, num_objects, frombuffer):
        """The result buffer's slices as arrays of their dtypes and shapes (views, no copy)."""
        B, Cn, RM, D = n_reads, self.n_cam, self.cfg.max_roots, num_objects
        L = self.live_layout(B, D)
        spec = dict(flags=("int32", (B,)), gate=("uint8", (B,)), blob_n=("int32", (B, Cn)), first=("int32", (B, Cn, 2)),
                    n=("int32", (B,)), obj=("float64", (B, RM, 3)), err=("float64", (B, RM)), n_objects=("int32", (B,)),
                    objects=("float64", (B, RM, 5)), drone_index=("int32", (B, RM)), called=("uint8", (B,)),
                    pos=("float32", (B, D, 3)), vel=("float32", (B, D, 3)), heading=("float64", (B, D)),
                    present=("uint8", (B, D)), chosen=("int32", (B, D)))
        return {k: frombuffer(buf, getattr(L, k), dt, shape) for k, (dt, shape) in spec.items()}

    def _live_args(self, raw, mode, timestamps, tracker):
        if self._pp_in is None:
            raise MocapError(-5, "mocap_set_preprocess has not been called (MocapContext.set_preprocess)")
        h, w = self._pp_in
        per = self.n_cam * h * w * 3
        n = raw.numel() if hasattr(raw, "numel") else raw.size
        if n % per:
            raise ValueError(f"raw must hold whole reads of {self.n_cam} x {h} x {w} x 3 bytes")
        B = n // per
        if mode & LIVE_LOCATE and (timestamps is None or len(timestamps) != B):
            raise ValueError("locate mode needs one timestamp per read")
        return B, (tracker.num_objects if tracker is not None else 0)

    def live(self, raw, mode, timestamps=None, tracker=None, want_frames=False):
        """The live capture loop for a batch of reads on the device (mocap_live_dev): raw uint8 cuda [B, C, in_h, in_w, 3],
        mode a set of LIVE_* bits, timestamps f64 cuda [B] (locate mode), tracker a :class:`Tracker` of this context.
        Returns a dict of views into one result buffer (``"buffer"``) -- flags, gate, blob_n, first, n, obj, err,
        n_objects, objects, drone_index, called, pos, vel, heading, present, chosen; slices the mode does not compute
        are undefined -- and ``"frames"`` uint8 [B, C, S, S, 3] with ``want_frames``.  No synchronisation."""
        torch = _torch()
        B, D = self._live_args(raw, mode, timestamps, tracker)
        buf = torch.empty((self.live_layout(B, D).total,), dtype=torch.uint8, device=raw.device)
        frames = torch.empty((B, self.n_cam, self.height, self.width, 3), dtype=torch.uint8, device=raw.device) if want_frames else None
        ts = None if timestamps is None else timestamps.contiguous()
        self.use_current_stream()
        self._check(self.lib.mocap_live_dev(self.h, tracker.h if tracker is not None else None, _ptr(raw.contiguous()), B, int(mode),
                                            _ptr(ts), _ptr(frames), _ptr(buf)))
        out = self._live_views(buf, B, D, lambda b, off, dt, shape: b[off:off + int(np.prod(shape)) * np.dtype(dt).itemsize]
                               .view(getattr(torch, dt)).view(shape))
        out["buffer"] = buf
        if want_frames:
            out["frames"] = frames
        return out

    def live_host(self, raw, mode, timestamps=None, tracker=None, want_frames=False, jpeg=False, quality=JPEG_QUALITY,
                  jpeg_stride=None):
        """The same on host arrays (mocap_live_host): raw uint8 ndarray [B, C, in_h, in_w, 3], timestamps a sequence of B
        floats; one copy in, one copy back of the result (and of the frames), one synchronisation.  Returns numpy views.
        ``jpeg=True`` (mocap_live_jpeg_host): also each read's processed frames side by side as cv2.imencode('.jpg')
        encodes them at ``quality``, encoded on the device -- ``"jpeg"`` uint8 [B, jpeg_stride] (default: the worst
        case) and ``"jpeg_len"`` int32 [B]; two synchronisations.  A JPEG longer than jpeg_stride raises MocapError."""
        raw = np.ascontiguousarray(raw, dtype=np.uint8)
        B, D = self._live_args(raw, mode, timestamps, tracker)
        buf = np.empty((self.live_layout(B, D).total,), dtype=np.uint8)
        frames = np.empty((B, self.n_cam, self.height, self.width, 3), dtype=np.uint8) if want_frames else None
        ts = None if timestamps is None else np.ascontiguousarray(timestamps, dtype=np.float64)
        trh = tracker.h if tracker is not None else None
        if jpeg:
            stride = int(jpeg_stride if jpeg_stride is not None else self.lib.mocap_jpeg_bound(self.n_cam * self.width, self.height))
            jbuf = np.empty((B, stride), dtype=np.uint8)
            jlen = np.empty((B,), dtype=np.int32)
            self._check(self.lib.mocap_live_jpeg_host(self.h, trh, _np_ptr(raw), B, int(mode), _np_ptr(ts), _np_ptr(frames), _np_ptr(buf),
                                                      int(quality), _np_ptr(jbuf), stride, _np_ptr(jlen)))
        else:
            self._check(self.lib.mocap_live_host(self.h, trh, _np_ptr(raw), B, int(mode), _np_ptr(ts), _np_ptr(frames), _np_ptr(buf)))
        out = self._live_views(buf, B, D, lambda b, off, dt, shape: b[off:off + int(np.prod(shape)) * np.dtype(dt).itemsize]
                               .view(dt).reshape(shape))
        out["buffer"] = buf
        if want_frames:
            out["frames"] = frames
        if jpeg:
            out["jpeg"], out["jpeg_len"] = jbuf, jlen
        return out

    # -- JPEG (the camera stream, index.py:55-56) ------------------------------------------------
    def jpeg_bound(self, width, height):
        """Worst-case bytes of the JPEG of one width x height image (mocap_jpeg_bound)."""
        return int(self.lib.mocap_jpeg_bound(int(width), int(height)))

    def encode_jpeg(self, images, tiles=1, quality=JPEG_QUALITY, stride=None):
        """cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality]) of a batch of BGR images on the device, byte for
        byte (mocap_encode_jpeg_dev).  images: contiguous uint8 cuda tensor [..., H, W, 3], or with ``tiles`` > 1
        [..., tiles, H, w, 3] -- each image is its ``tiles`` frames side by side (np.hstack), e.g. the frames of
        ``live(..., want_frames=True)`` with tiles = C.  Returns {"jpeg": uint8 [n, stride], "len": int32 [n]} on the
        device: image i is jpeg[i, :len[i]], len -1 where it did not fit ``stride`` (default: the worst case).  No
        synchronisation."""
        torch = _torch()
        if images.dtype != torch.uint8 or not images.is_cuda or not images.is_contiguous() or images.dim() < 3 or images.shape[-1] != 3:
            raise ValueError("encode_jpeg: images must be a contiguous uint8 cuda tensor [..., H, W, 3]")
        tiles = int(tiles)
        if tiles > 1 and (images.dim() < 4 or images.shape[-4] != tiles):
            raise ValueError(f"encode_jpeg: with tiles={tiles} images must be [..., {tiles}, H, w, 3]")
        th, tw = int(images.shape[-3]), int(images.shape[-2])
        per = max(1, tiles) * th * tw * 3
        n = images.numel() // per if per else 0
        if stride is None:
            stride = self.jpeg_bound(max(1, tiles) * tw, th)
        jbuf = torch.empty((n, int(stride)), dtype=torch.uint8, device=images.device)
        jlen = torch.empty((n,), dtype=torch.int32, device=images.device)
        self.use_current_stream()
        self._check(self.lib.mocap_encode_jpeg_dev(self.h, _ptr(images), n, tiles, tw, th, int(quality), _ptr(jbuf), int(stride), _ptr(jlen)))
        return {"jpeg": jbuf, "len": jlen}

    def undistort_map(self, cam):
        m1 = np.empty((self.height, self.width, 2), dtype=np.int16)
        m2 = np.empty((self.height, self.width), dtype=np.uint16)
        self._check(self.lib.mocap_get_undistort_map(self.h, int(cam), _np_ptr(m1), _np_ptr(m2)))
        return m1, m2

    # -- batched device API ---------------------------------------------------------------
    def detect(self, frames, threshold=THRESHOLD, want_moments=False):
        """frames: uint8 cuda tensor [..., H, W] or [..., H, W, 3].  Returns dict of cuda tensors:
        xy int32 [N, max_blobs, 2], n int32 [N], flags int32 [N], (mom int64 [N, max_blobs, 4])."""
        torch = _torch()
        ch = 3 if (frames.dim() >= 3 and frames.shape[-1] == 3 and frames.shape[-2] == self.width) else 1
        per = self.width * self.height * ch
        if not frames.is_contiguous() or frames.dtype != torch.uint8 or frames.numel() % per:
            raise ValueError("frames must be a contiguous uint8 tensor of whole images")
        n = frames.numel() // per
        dev = frames.device
        xy = torch.empty((n, self.cfg.max_blobs, 2), dtype=torch.int32, device=dev)
        cnt = torch.empty((n,), dtype=torch.int32, device=dev)
        flags = torch.empty((n,), dtype=torch.int32, device=dev)
        mom = torch.empty((n, self.cfg.max_blobs, 4), dtype=torch.int64, device=dev) if want_moments else None
        self.use_current_stream()
        self._check(self.lib.mocap_detect_dev(self.h, _ptr(frames), n, ch, int(threshold), _ptr(xy), _ptr(cnt), _ptr(mom), _ptr(flags)))
        out = {"xy": xy, "n": cnt, "flags": flags}
        if want_moments:
            out["mom"] = mom
        return out

    def match_triangulate(self, xy, n, want_chosen=False):
        """xy int32 [B*C, max_blobs, 2], n int32 [B*C] (output of detect).  Returns dict: obj f64
        [B, max_roots, 3], err f64 [B, max_roots], n int32 [B], flags int32 [B], (chosen int32 [B, max_roots, C])."""
        torch = _torch()
        B = n.numel() // self.n_cam
        dev = xy.device
        R = self.cfg.max_roots
        obj = torch.empty((B, R, 3), dtype=torch.float64, device=dev)
        err = torch.empty((B, R), dtype=torch.float64, device=dev)
        cnt = torch.empty((B,), dtype=torch.int32, device=dev)
        flags = torch.empty((B,), dtype=torch.int32, device=dev)
        chosen = torch.empty((B, R, self.n_cam), dtype=torch.int32, device=dev) if want_chosen else None
        self.use_current_stream()
        self._check(self.lib.mocap_match_triangulate_dev(self.h, _ptr(xy), _ptr(n), B, _ptr(obj), _ptr(err), _ptr(cnt), _ptr(flags), _ptr(chosen)))
        out = {"obj": obj, "err": err, "n": cnt, "flags": flags}
        if want_chosen:
            out["chosen"] = chosen
        return out

    def tracks_to_observations(self, xy, n_obj, chosen):
        """Matcher output -> explicit correspondences for S4 (BASELINE config 3: bundle adjustment on the
        tracks of a batch).  xy int32 [B*C, max_blobs, 2] (detect), n_obj int32 [B], chosen int32
        [B, max_roots, C] (match_triangulate(want_chosen=True)).  Returns host arrays obs f64 [P, C, 2],
        mask uint8 [P, C] with one row per triangulated point, in frame order."""
        torch = _torch()
        B, R, Cn = chosen.shape
        MB = xy.shape[1]
        keep = torch.arange(R, device=chosen.device)[None, :] < n_obj[:, None].to(torch.int64)      # [B, R]
        ch = chosen[keep].to(torch.int64)                                                          # [P, C]
        set_idx = torch.arange(B, device=chosen.device)[:, None].expand(B, R)[keep]                # [P]
        img = set_idx[:, None] * Cn + torch.arange(Cn, device=chosen.device)[None, :]              # [P, C]
        mask = ch >= 0
        pts = xy.view(-1, MB, 2)[img, ch.clamp(min=0)]                                             # [P, C, 2]
        obs = torch.where(mask[:, :, None], pts.to(torch.float64), torch.zeros((), dtype=torch.float64, device=pts.device))
        return obs.cpu().numpy(), mask.to(torch.uint8).cpu().numpy()

    def alloc_tracks(self, n_sets, device=None):
        torch = _torch()
        dev = device or self.torch_device
        R = self.cfg.max_roots
        return {"obj": torch.empty((n_sets, R, 3), dtype=torch.float64, device=dev),
                "err": torch.empty((n_sets, R), dtype=torch.float64, device=dev),
                "n": torch.empty((n_sets,), dtype=torch.int32, device=dev),
                "flags": torch.empty((n_sets,), dtype=torch.int32, device=dev)}

    def pipeline(self, frames, threshold=THRESHOLD, out=None, want_tracks=False):
        """S1+S2+S3 on a device tensor of frame-sets [B, C, H, W] (or [B, C, H, W, 3]).  want_tracks (or an ``out``
        that holds "track_xy"): also the winners' pixels per camera, int32 [B, max_roots, C, 2], (-1, -1) = no view."""
        torch = _torch()
        ch = 3 if (frames.shape[-1] == 3 and frames.shape[-2] == self.width) else 1
        B = frames.numel() // (self.n_cam * self.width * self.height * ch)
        if out is None:
            out = self.alloc_tracks(B, frames.device)
        if want_tracks and "track_xy" not in out:
            out["track_xy"] = torch.empty((B, self.cfg.max_roots, self.n_cam, 2), dtype=torch.int32, device=frames.device)
        self.use_current_stream()
        self._check(self.lib.mocap_pipeline_tracks_dev(self.h, _ptr(frames), B, ch, int(threshold), _ptr(out["obj"]), _ptr(out["err"]),
                                                       _ptr(out["n"]), _ptr(out["flags"]), _ptr(out.get("track_xy"))))
        return out

    def tracks_to_observations_dev(self, tracks, max_err=0.0, capacity=None, out=None):
        """Matcher output of a batch (``pipeline(..., want_tracks=True)``) -> the explicit correspondences S4 consumes,
        on the device, no synchronisation: dict obs f64 [capacity, C, 2], mask uint8 [capacity, C], n int32 [1]."""
        torch = _torch()
        B = tracks["n"].numel()
        dev = tracks["n"].device
        cap = int(capacity or B * self.cfg.max_roots)
        if out is None:
            out = {"obs": torch.empty((cap, self.n_cam, 2), dtype=torch.float64, device=dev),
                   "mask": torch.empty((cap, self.n_cam), dtype=torch.uint8, device=dev),
                   "n": torch.zeros((1,), dtype=torch.int32, device=dev)}
        self.use_current_stream()
        self._check(self.lib.mocap_tracks_to_observations_dev(self.h, _ptr(tracks["track_xy"]), _ptr(tracks["n"]), _ptr(tracks["err"]), B,
                                                              float(max_err), _ptr(out["obs"]), _ptr(out["mask"]), _ptr(out["n"]), cap))
        return out

    def set_ba_grid(self, n_ctas=0):
        """CTA budget G of the device-resident bundle adjustment of this context (0: one per SM).  A single solve runs on G
        CTAs, a batch of K (``bundle_adjust_batch_dev``) splits them, G // K + (k < G % K) for problem k.  Independent
        solves finish sooner side by side: in one batched call, or as K contexts on K streams with SMs // K CTAs each
        (mocap_set_ba_grid, include/mocap_b200.h)."""
        self._check(self.lib.mocap_set_ba_grid(self.h, int(n_ctas)))

    def bundle_adjust_dev(self, obs, mask, R, t, n_points=None, report=None, ftol=1e-2, max_nfev=0, prefit=True, jacobian=1,
                          prefit_max_iter=50):
        """S4 wholly on the device (mocap_bundle_adjust_dev): obs f64 [P, C, 2], mask uint8 [P, C], R f64 [C, 3, 3] and
        t f64 [C, 3] cuda tensors (R, t updated in place), n_points an int32 cuda tensor [1] or None.  One cooperative
        launch, no synchronisation.  Returns the report as a uint8 cuda tensor (decode with ``decode_ba_report``)."""
        torch = _torch()
        opt = BAOptions()
        self.lib.mocap_ba_default_options(C.byref(opt))
        opt.ftol, opt.max_nfev, opt.prefit, opt.jacobian, opt.prefit_max_iter = ftol, max_nfev, 1 if prefit else 0, jacobian, prefit_max_iter
        if report is None:
            report = torch.zeros((C.sizeof(BAReport),), dtype=torch.uint8, device=obs.device)
        self.use_current_stream()
        self._check(self.lib.mocap_bundle_adjust_dev(self.h, _ptr(obs), _ptr(mask), obs.shape[0], _ptr(n_points), _ptr(R), _ptr(t),
                                                     C.byref(opt), _ptr(report)))
        return report

    def bundle_adjust_batch_dev(self, problems, ftol=1e-2, max_nfev=0, prefit=True, jacobian=1, prefit_max_iter=50):
        """Several independent S4 solves in ONE cooperative launch (mocap_bundle_adjust_batch_dev): problems is a list of
        dicts with the tensors ``bundle_adjust_dev`` takes -- "obs", "mask", "R", "t" and optionally "n" (int32 cuda [1])
        and "report" -- sharing this context's cameras and one set of options.  Problem k runs on G // K + (k < G % K) of
        the context's G CTAs (``set_ba_grid``) and gives the bits ``bundle_adjust_dev`` gives on that many.  No
        synchronisation.  Returns one report tensor per problem (decode with ``decode_ba_report``)."""
        torch = _torch()
        opt = BAOptions()
        self.lib.mocap_ba_default_options(C.byref(opt))
        opt.ftol, opt.max_nfev, opt.prefit, opt.jacobian, opt.prefit_max_iter = ftol, max_nfev, 1 if prefit else 0, jacobian, prefit_max_iter
        reports = []
        arr = (BAProblem * max(1, len(problems)))()
        for k, p in enumerate(problems):
            obs = p.get("obs")
            rep = p.get("report")
            if rep is None:
                rep = torch.zeros((C.sizeof(BAReport),), dtype=torch.uint8, device=f"cuda:{self.cfg.device}")
            reports.append(rep)
            arr[k] = BAProblem(_ptr(obs), _ptr(p.get("mask")), 0 if obs is None else int(obs.shape[0]), _ptr(p.get("n")),
                               _ptr(p.get("R")), _ptr(p.get("t")), _ptr(rep))
        self.use_current_stream()
        self._check(self.lib.mocap_bundle_adjust_batch_dev(self.h, arr, len(problems), C.byref(opt)))
        return reports

    def screen_observations_dev(self, obs, mask, R, t, threshold_px, n_points=None, out=None):
        """Per-view screen of explicit correspondences against the current poses (mocap_screen_observations_dev, rule in
        DESIGN section 5): obs f64 [P, C, 2], mask uint8 [P, C] (the caller's ORIGINAL mask), R f64 [C, 3, 3], t f64
        [C, 3] cuda tensors, n_points an int32 cuda tensor [1] or None.  One launch, no synchronisation.  Returns dict
        mask uint8 [P, C] (rows past n_points untouched), stats int32 [4] = views in, kept, dropped, rows emptied."""
        torch = _torch()
        if out is None:
            out = {"mask": torch.empty_like(mask), "stats": torch.empty((4,), dtype=torch.int32, device=mask.device)}
        self.use_current_stream()
        self._check(self.lib.mocap_screen_observations_dev(self.h, _ptr(obs), _ptr(mask), obs.shape[0], _ptr(n_points), _ptr(R), _ptr(t),
                                                           float(threshold_px), _ptr(out["mask"]), _ptr(out["stats"])))
        return out

    def screen_observations(self, obs, mask, poses, threshold_px):
        """The same on host arrays: obs float64 [P, C, 2], mask uint8 [P, C], poses a list of {"R", "t"}.  Returns dict
        mask uint8 [P, C], stats int32 [4]."""
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        R = np.ascontiguousarray(np.stack([np.asarray(p["R"], dtype=np.float64).reshape(3, 3) for p in poses]))
        t = np.ascontiguousarray(np.stack([np.asarray(p["t"], dtype=np.float64).reshape(3) for p in poses]))
        out = np.zeros_like(mask)
        stats = np.zeros((4,), dtype=np.int32)
        self._check(self.lib.mocap_screen_observations_host(self.h, _np_ptr(obs), _np_ptr(mask), obs.shape[0], None, _np_ptr(R), _np_ptr(t),
                                                            float(threshold_px), _np_ptr(out), _np_ptr(stats)))
        return {"mask": out, "stats": stats}

    def bundle_adjust_screened(self, obs, mask, poses, threshold_px, rounds=2, first_mask=None, **ba_kw):
        """Bundle adjustment that screens mismatched views out between rounds, all on the device with no synchronisation
        until the final copy-out: ``bundle_adjust_dev(first_mask)``, then ``rounds`` times [screen the ORIGINAL mask at
        the current poses -> ``bundle_adjust_dev(screened mask)``].  A view dropped under early poses can come back once
        they improve.  ``first_mask`` (None: ``mask``) is what the first solve sees: the mismatched views a solve keeps
        pull the poses so far that the first screen would lose most good views with them (INTEGRATION.md section 2), so
        a cleaner first guess -- e.g. the views that are RANSAC inliers with a neighbouring camera -- helps.  obs / mask
        host arrays, poses a list of {"R", "t"}; ``ba_kw`` go to every solve.  Returns (poses, report of the last solve,
        kept mask uint8 [P, C] -- the first solve's mask when rounds == 0)."""
        torch = _torch()
        if int(rounds) != rounds or rounds < 0:
            raise ValueError(f"bundle_adjust_screened: rounds must be a non-negative integer (got {rounds!r})")
        if not (threshold_px > 0 and np.isfinite(threshold_px)):
            raise MocapError(-1, f"bundle_adjust_screened: threshold_px must be positive and finite (got {threshold_px})")
        dev = self.torch_device
        d_obs = torch.from_numpy(np.ascontiguousarray(obs, dtype=np.float64)).to(dev)
        d_mask = torch.from_numpy(np.ascontiguousarray(mask, dtype=np.uint8)).to(dev)
        R = torch.from_numpy(np.stack([np.asarray(p["R"], dtype=np.float64).reshape(3, 3) for p in poses])).to(dev)
        t = torch.from_numpy(np.stack([np.asarray(p["t"], dtype=np.float64).reshape(3) for p in poses])).to(dev)
        d_first = d_mask if first_mask is None else torch.from_numpy(np.ascontiguousarray(first_mask, dtype=np.uint8)).to(dev)
        if d_first.shape != d_mask.shape:
            raise ValueError("bundle_adjust_screened: first_mask must have the shape of mask")
        screened = {"mask": torch.empty_like(d_mask), "stats": torch.empty((4,), dtype=torch.int32, device=dev)}
        report = self.bundle_adjust_dev(d_obs, d_first, R, t, **ba_kw)
        for _ in range(int(rounds)):
            self.screen_observations_dev(d_obs, d_mask, R, t, threshold_px, out=screened)
            report = self.bundle_adjust_dev(d_obs, screened["mask"], R, t, report=report, **ba_kw)
        rep = self.decode_ba_report(report)
        if rep["status"] == -3:
            raise MocapError(-1, "bundle_adjust_screened: no point is seen by two cameras")
        kept = (screened["mask"] if rounds else d_first).cpu().numpy()
        R, t = R.cpu().numpy(), t.cpu().numpy()
        return [{"R": R[i].copy(), "t": t[i].copy()} for i in range(self.n_cam)], rep, kept

    @staticmethod
    def decode_ba_report(report):
        rep = BAReport.from_buffer_copy(report.cpu().numpy().tobytes())
        return _report_dict(rep)

    def pipeline_host(self, frames, threshold=THRESHOLD, out=None):
        """Same through HOST memory: frames is a (preferably pinned) uint8 cpu tensor / ndarray;
        returns cpu tensors.  Blocks until the results are in host memory."""
        torch = _torch()
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        ch = 3 if (frames.shape[-1] == 3 and frames.shape[-2] == self.width) else 1
        B = frames.numel() // (self.n_cam * self.width * self.height * ch)
        R = self.cfg.max_roots
        if out is None:
            out = {"obj": torch.empty((B, R, 3), dtype=torch.float64).pin_memory(),
                   "err": torch.empty((B, R), dtype=torch.float64).pin_memory(),
                   "n": torch.empty((B,), dtype=torch.int32).pin_memory(),
                   "flags": torch.empty((B,), dtype=torch.int32).pin_memory()}
        self.use_current_stream()
        self._check(self.lib.mocap_pipeline_host(self.h, _ptr(frames), B, ch, int(threshold),
                                                 _ptr(out["obj"]), _ptr(out["err"]), _ptr(out["n"]), _ptr(out["flags"])))
        return out

    def locate_objects(self, obj, err, n, max_objects=8):
        """obj f64 [B, max_roots, 3], err f64 [B, max_roots], n int32 [B] (matcher output, cuda tensors) ->
        dict: objects f64 [B, max_objects, 5] = x y z heading error, drone_index int32 [B, max_objects], n int32 [B]."""
        torch = _torch()
        B = n.numel()
        dev = obj.device
        out = torch.empty((B, max_objects, 5), dtype=torch.float64, device=dev)
        di = torch.empty((B, max_objects), dtype=torch.int32, device=dev)
        cnt = torch.empty((B,), dtype=torch.int32, device=dev)
        self.use_current_stream()
        self._check(self.lib.mocap_locate_objects_dev(self.h, _ptr(obj), _ptr(err), _ptr(n), B, max_objects, _ptr(out), _ptr(di), _ptr(cnt)))
        return {"objects": out, "drone_index": di, "n": cnt}

    def tracker(self, num_objects=2):
        """A batched drone tracker on this context (:class:`Tracker`): the reference's KalmanFilter.predict_location
        for whole batches of located frame-sets, state kept on the device between batches."""
        return Tracker(self, num_objects)

    # -- explicit correspondences (host arrays) -------------------------------------------
    def triangulate(self, obs, mask, want_err=True):
        """obs float64 [F, C, 2], mask uint8 [F, C] -> (X [F,3], err [F] or None, valid [F])."""
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        F = obs.shape[0]
        X = np.empty((F, 3))
        err = np.empty((F,)) if want_err else None
        valid = np.empty((F,), dtype=np.uint8)
        self._check(self.lib.mocap_triangulate_host(self.h, _np_ptr(obs), _np_ptr(mask), F, _np_ptr(X), _np_ptr(err), _np_ptr(valid)))
        return X, err, valid

    def reprojection_errors(self, obs, mask, X):
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        X = np.ascontiguousarray(X, dtype=np.float64)
        F = obs.shape[0]
        err = np.empty((F,))
        valid = np.empty((F,), dtype=np.uint8)
        self._check(self.lib.mocap_reprojection_errors_host(self.h, _np_ptr(obs), _np_ptr(mask), _np_ptr(X), F, _np_ptr(err), _np_ptr(valid)))
        return err, valid

    def _ransac_options(self, threshold, hypotheses, seed):
        opt = RansacOptions()
        self.lib.mocap_ransac_default_options(C.byref(opt))
        opt.threshold_px, opt.hypotheses, opt.seed = float(threshold), int(hypotheses), int(seed)
        return opt

    def calibrate_init(self, obs, mask, F_given=None, method="8point", threshold=1.0, hypotheses=2048, seed=0, **graph_options):
        """Chain of relative poses from 2D tracks (index.py:229-270).  Returns (poses, F_used [C-1,3,3], votes [C-1,4]).

        ``method="8point"``: each pair's F is a normalised 8-point fit to all common observations, re-fitted on its
        1 px Sampson inliers (or ``F_given``).  ``method="ransac"``: the fit starts from the inliers of a RANSAC model
        (``hypotheses`` 7-point samples per pair from ``seed``, inliers within ``threshold`` px), which mismatched
        points do not pull; the return then also holds the per-pair inlier masks, uint8 [F, C-1].

        ``method="graph"``: every camera placed from every overlapping pair (mocap_calibrate_graph_host, DESIGN section
        1 (f) #4): RANSAC F for all pairs with at least ``min_common`` common observations, the motion chosen in each
        pair's own frame, rotation averaging and the translations of all tracks at once.  ``graph_options`` are the
        fields of ``mocap_graph_options`` (min_common, min_inliers, min_angle_deg, rot_outlier_deg, irls_rounds).
        Returns (poses, pairs, support): pairs a list of dicts (a, b, common, inliers, candidate, in_front,
        median_angle_deg, rot_residual_deg, used), support uint8 [F, C] -- a first bundle-adjustment mask."""
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        Cn = self.n_cam
        if method == "graph":
            if F_given is not None:
                raise ValueError("calibrate_init: F_given and method='graph' exclude each other")
            return self._calibrate_graph(obs, mask, threshold, hypotheses, seed, graph_options)
        if graph_options:
            raise ValueError(f"calibrate_init: {sorted(graph_options)} apply to method='graph' only")
        R = np.empty((Cn, 3, 3)); t = np.empty((Cn, 3))
        Fu = np.empty((Cn - 1, 3, 3)); votes = np.empty((Cn - 1, 4), dtype=np.int32)
        if method == "ransac":
            if F_given is not None:
                raise ValueError("calibrate_init: F_given and method='ransac' exclude each other")
            inl = np.empty((obs.shape[0], Cn - 1), dtype=np.uint8)
            opt = self._ransac_options(threshold, hypotheses, seed)
            self._check(self.lib.mocap_calibrate_init_ransac_host(self.h, _np_ptr(obs), _np_ptr(mask), obs.shape[0], C.byref(opt),
                                                                  _np_ptr(R), _np_ptr(t), _np_ptr(Fu), _np_ptr(votes), _np_ptr(inl)))
            return [{"R": R[i].copy(), "t": t[i].copy()} for i in range(Cn)], Fu, votes, inl
        if method != "8point":
            raise ValueError(f"calibrate_init: unknown method {method!r} (expected '8point', 'ransac' or 'graph')")
        Fg = None if F_given is None else np.ascontiguousarray(np.asarray(F_given, dtype=np.float64).reshape(Cn - 1, 3, 3))
        self._check(self.lib.mocap_calibrate_init_host(self.h, _np_ptr(obs), _np_ptr(mask), obs.shape[0], _np_ptr(Fg),
                                                       _np_ptr(R), _np_ptr(t), _np_ptr(Fu), _np_ptr(votes)))
        return [{"R": R[i].copy(), "t": t[i].copy()} for i in range(Cn)], Fu, votes

    def _calibrate_graph(self, obs, mask, threshold, hypotheses, seed, graph_options):
        Cn = self.n_cam
        gopt = GraphOptions()
        self.lib.mocap_graph_default_options(C.byref(gopt))
        for k, v in graph_options.items():
            if k not in dict(GraphOptions._fields_):
                raise ValueError(f"calibrate_init: unknown graph option {k!r} (expected one of "
                                 f"{', '.join(f for f, _ in GraphOptions._fields_)})")
            setattr(gopt, k, v)
        opt = self._ransac_options(threshold, hypotheses, seed)
        R = np.empty((Cn, 3, 3)); t = np.empty((Cn, 3))
        pairs = (GraphPair * max(1, Cn * (Cn - 1) // 2))()
        n_pairs = C.c_int(0)
        support = np.zeros(mask.shape, dtype=np.uint8)
        self._check(self.lib.mocap_calibrate_graph_host(self.h, _np_ptr(obs), _np_ptr(mask), obs.shape[0], C.byref(opt), C.byref(gopt),
                                                        _np_ptr(R), _np_ptr(t), pairs, C.byref(n_pairs), _np_ptr(support)))
        rep = [{f: getattr(pairs[i], f) for f, _ in GraphPair._fields_} for i in range(n_pairs.value)]
        return [{"R": R[i].copy(), "t": t[i].copy()} for i in range(Cn)], rep, support

    def fundamental_ransac(self, obs, mask, threshold=1.0, hypotheses=2048, seed=0):
        """The RANSAC stage of ``calibrate_init(method="ransac")`` alone: per adjacent pair the winning 7-point model
        and its inliers within ``threshold`` px, before any refinement.  Returns (F [C-1,3,3], inliers uint8 [F, C-1])."""
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        Cn = self.n_cam
        F = np.empty((Cn - 1, 3, 3)); inl = np.empty((obs.shape[0], Cn - 1), dtype=np.uint8)
        opt = self._ransac_options(threshold, hypotheses, seed)
        self._check(self.lib.mocap_fundamental_ransac_host(self.h, _np_ptr(obs), _np_ptr(mask), obs.shape[0], C.byref(opt),
                                                           _np_ptr(F), _np_ptr(inl)))
        return F, inl

    def ba_residuals(self, obs, mask, poses):
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        R = np.ascontiguousarray(np.stack([np.asarray(p["R"], dtype=np.float64).reshape(3, 3) for p in poses]))
        t = np.ascontiguousarray(np.stack([np.asarray(p["t"], dtype=np.float64).reshape(3) for p in poses]))
        F = obs.shape[0]
        r = np.empty((F,), dtype=np.float32)
        valid = np.empty((F,), dtype=np.uint8)
        nv = C.c_int(0)
        self._check(self.lib.mocap_ba_residuals_host(self.h, _np_ptr(obs), _np_ptr(mask), F, _np_ptr(R), _np_ptr(t), _np_ptr(r), _np_ptr(valid), C.byref(nv)))
        return r[valid.astype(bool)]

    def bundle_adjust(self, obs, mask, poses, ftol=1e-2, max_nfev=0, engine=0, prefit=True, jacobian=1, prefit_max_iter=50):
        obs = np.ascontiguousarray(obs, dtype=np.float64)
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        R = np.ascontiguousarray(np.stack([np.asarray(p["R"], dtype=np.float64).reshape(3, 3) for p in poses]))
        t = np.ascontiguousarray(np.stack([np.asarray(p["t"], dtype=np.float64).reshape(3) for p in poses]))
        opt = BAOptions()
        self.lib.mocap_ba_default_options(C.byref(opt))
        opt.ftol = ftol
        opt.max_nfev = max_nfev
        opt.engine, opt.prefit, opt.jacobian, opt.prefit_max_iter = engine, 1 if prefit else 0, jacobian, prefit_max_iter
        rep = BAReport()
        self._check(self.lib.mocap_bundle_adjust_host(self.h, _np_ptr(obs), _np_ptr(mask), obs.shape[0], _np_ptr(R), _np_ptr(t), C.byref(opt), C.byref(rep)))
        out = [{"R": R[i].copy(), "t": t[i].copy()} for i in range(R.shape[0])]
        return out, _report_dict(rep)

    # -- accounting -----------------------------------------------------------------------
    def launch_count(self):
        return int(self.lib.mocap_launch_count(self.h))

    def enable_kernel_timing(self, on=True):
        self._check(self.lib.mocap_enable_kernel_timing(self.h, 1 if on else 0))

    def detect_kernel_ms(self, reset=True):
        ms, n = C.c_double(0), C.c_int(0)
        self._check(self.lib.mocap_detect_kernel_ms(self.h, 1 if reset else 0, C.byref(ms), C.byref(n)))
        return ms.value, n.value


class Tracker:
    """Device-resident state of the reference's ``KalmanFilter(num_objects)`` (mocap_tracker_*): one Kalman filter and
    three low-pass filters per drone.  Every frame-set of a batch counts as one ``predict_location`` call at its
    timestamp; frame-sets without objects only advance time.  Enqueues on torch's current stream, never synchronises.
    Close it (or drop it) before its context."""

    def __init__(self, ctx, num_objects=2):
        self.ctx, self.num_objects = ctx, int(num_objects)
        h = C.c_void_p()
        ctx._check(ctx.lib.mocap_tracker_create(ctx.h, self.num_objects, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.ctx.lib.mocap_tracker_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, prev_time):
        """The reference's ``reset()`` with its clock reading: ``prev_time`` = that reading - 20 s.  Takes effect at the
        next batch: every drone re-initialises at its next present step; covariances and low-pass histories stay."""
        self.ctx._check(self.ctx.lib.mocap_tracker_reset(self.h, float(prev_time)))

    def track_dev(self, located, timestamps, out=None, calls=None):
        """located: the dict ``MocapContext.locate_objects`` returns (objects f64 [B, M, 5], drone_index int32 [B, M],
        n int32 [B]); timestamps: f64 cuda tensor [B] (seconds, one per frame-set).  Returns dict of cuda tensors, per
        frame-set and drone: pos f32 [B, D, 3], vel f32 [B, D, 3] and heading f64 [B, D] (low-pass filtered), present
        uint8 [B, D] and chosen int32 [B, D] (the object row, -1 if absent); pos / vel / heading are 0 where present
        is 0.  Two launches.  ``calls`` (uint8 cuda [B], optional): frame-sets where it is 0 are not predict_location
        calls -- the filters' clock and histories do not move there and the drones are absent
        (mocap_track_objects_gated_dev)."""
        torch = _torch()
        obj, di, n = located["objects"], located["drone_index"], located["n"]
        B, M = obj.shape[0], obj.shape[1]
        D = self.num_objects
        dev = obj.device
        if tuple(timestamps.shape) != (B,) or timestamps.dtype != torch.float64:
            raise ValueError("timestamps must be a float64 tensor with one entry per frame-set")
        if out is None:
            out = {"pos": torch.empty((B, D, 3), dtype=torch.float32, device=dev),
                   "vel": torch.empty((B, D, 3), dtype=torch.float32, device=dev),
                   "heading": torch.empty((B, D), dtype=torch.float64, device=dev),
                   "present": torch.empty((B, D), dtype=torch.uint8, device=dev),
                   "chosen": torch.empty((B, D), dtype=torch.int32, device=dev)}
        self.ctx.use_current_stream()
        if calls is None:
            self.ctx._check(self.ctx.lib.mocap_track_objects_dev(self.h, _ptr(obj.contiguous()), _ptr(di.contiguous()), _ptr(n.contiguous()),
                                                                 M, _ptr(timestamps.contiguous()), B, _ptr(out["pos"]), _ptr(out["vel"]),
                                                                 _ptr(out["heading"]), _ptr(out["present"]), _ptr(out["chosen"])))
            return out
        if tuple(calls.shape) != (B,) or calls.dtype != torch.uint8:
            raise ValueError("calls must be a uint8 tensor with one entry per frame-set")
        self.ctx._check(self.ctx.lib.mocap_track_objects_gated_dev(self.h, _ptr(obj.contiguous()), _ptr(di.contiguous()), _ptr(n.contiguous()),
                                                                   M, _ptr(timestamps.contiguous()), _ptr(calls.contiguous()), B,
                                                                   _ptr(out["pos"]), _ptr(out["vel"]), _ptr(out["heading"]),
                                                                   _ptr(out["present"]), _ptr(out["chosen"])))
        return out


# =================================================================================================
# Reference-signature mirror
# =================================================================================================
def _split_observations(image_points):
    """(F, C, 2) list/object array with None for missing views -> float64 obs + uint8 mask."""
    arr = np.array(image_points, dtype=object)
    if arr.ndim != 3:
        raise ValueError("image_points must be (F, C, 2)")
    F, Cn, _ = arr.shape
    mask = np.empty((F, Cn), dtype=np.uint8)
    obs = np.zeros((F, Cn, 2), dtype=np.float64)
    for f in range(F):
        for c in range(Cn):
            a, b = arr[f, c]
            if a is None and b is None:
                mask[f, c] = 0
            else:
                mask[f, c] = 1
                obs[f, c, 0], obs[f, c, 1] = a, b
    return obs, mask


class MocapSession:
    """What the reference keeps in its ``Cameras`` singleton for this path: the intrinsics
    (helpers.py:19-22) -- plus lazily created CUDA contexts per camera count.  Thread safe
    (one lock per session; the reference's singleton is unsynchronised, Singleton.py:3)."""

    _default = None

    def __init__(self, intrinsics, width=640, height=480, device=0, large_holes=False):
        """``large_holes``: the contexts the session creates reproduce holed blobs wider or taller than 62 pixels as
        cv2 does (MocapContext.set_large_holes); off, find_dot raises on a frame with one."""
        self.intrinsics = [np.asarray(k, dtype=np.float64).reshape(3, 3) for k in intrinsics]
        self.width, self.height, self.device = width, height, device
        self.large_holes = bool(large_holes)
        self._ctxs = {}
        self._live = {}
        self._lock = threading.RLock()

    @classmethod
    def default(cls):
        if cls._default is None:
            raise MocapError(-5, "no MocapSession installed: call MocapSession.install(intrinsics) or install_into(helpers)")
        return cls._default

    @classmethod
    def install(cls, intrinsics, **kw):
        cls._default = cls(intrinsics, **kw)
        return cls._default

    def ctx(self, n_cam, **kw):
        with self._lock:
            key = (n_cam, tuple(sorted(kw.items())))
            if key not in self._ctxs:
                ctx = MocapContext(n_cam, self.width, self.height, self.device, **kw)
                if self.large_holes:
                    ctx.set_large_holes(True)
                self._ctxs[key] = ctx
            return self._ctxs[key]

    def ctx_with_poses(self, camera_poses):
        n = len(camera_poses)
        if n > len(self.intrinsics):
            raise ValueError("more camera poses than intrinsics")
        c = self.ctx(n, **MIRROR_LIMITS)
        c.set_cameras(self.intrinsics[:n], camera_poses)
        return c


def find_dot(img, session=None):
    """Mirror of ``Cameras._find_dot(self, img)`` (helpers.py:143-163): returns
    ``(img, image_points)`` with image_points a list of ``[x, y]`` or ``[[None, None]]``.
    The contour / text overlay the reference draws into ``img`` (helpers.py:148,156-157) is
    cosmetic and is not reproduced; a 1-px centre dot is drawn instead."""
    torch = _torch()
    s = session or MocapSession.default()
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    with s._lock:
        ctx = s._ctxs.get(("detect", w, h))
        if ctx is None:
            ctx = MocapContext(1, w, h, s.device, max_blobs=MIRROR_LIMITS["max_blobs"],
                               max_segments=MIRROR_LIMITS["max_segments"])
            if s.large_holes:
                ctx.set_large_holes(True)
            s._ctxs[("detect", w, h)] = ctx
        d = ctx.detect(torch.from_numpy(img).to(ctx.torch_device))
        raise_on_overflow(d["flags"][0].item(), "find_dot")
        n = int(d["n"][0].item())
        pts = d["xy"][0, :n].cpu().numpy().tolist()
    for x, y in pts:
        if 0 <= y < h and 0 <= x < w:
            img[y, x] = (100, 255, 100) if img.ndim == 3 else 255
    return img, (pts if pts else [[None, None]])


def triangulate_points(image_points, camera_poses, session=None):
    """Mirror of helpers.py:330-336: ndarray (F, 3); rows of ``[None]*3`` (object dtype) where a
    point has fewer than two views."""
    s = session or MocapSession.default()
    if len(image_points) == 0:
        return np.array([])
    obs, mask = _split_observations(image_points)
    with s._lock:
        X, _, valid = s.ctx_with_poses(camera_poses).triangulate(obs, mask, want_err=False)
    if valid.all():
        return X
    out = np.empty((len(X), 3), dtype=object)
    for f in range(len(X)):
        out[f] = list(X[f]) if valid[f] else [None, None, None]
    return out


def triangulate_point(image_points, camera_poses, session=None):
    """Mirror of helpers.py:293-327 (one point)."""
    r = triangulate_points([image_points], camera_poses, session)[0]
    return list(r) if r[0] is None else np.asarray(r, dtype=np.float64)


def calculate_reprojection_errors(image_points, object_points, camera_poses, session=None):
    """Mirror of helpers.py:203-211: float64 vector; points with <= 1 view are skipped."""
    s = session or MocapSession.default()
    if len(image_points) == 0:
        return np.array([])
    obs, mask = _split_observations(image_points)
    X = np.array([[np.nan] * 3 if p[0] is None else [float(v) for v in p] for p in object_points], dtype=np.float64)
    with s._lock:
        err, valid = s.ctx_with_poses(camera_poses).reprojection_errors(obs, mask, X)
    return err[valid.astype(bool)]


def calculate_reprojection_error(image_points, object_point, camera_poses, session=None):
    """Mirror of helpers.py:214-241 (one point): float or None."""
    e = calculate_reprojection_errors([image_points], [object_point], camera_poses, session)
    return float(e[0]) if len(e) else None


def find_point_correspondance_and_object_points(image_points, camera_poses, frames, session=None):
    """Mirror of helpers.py:339-421: returns ``(errors (K,), object_points (K,3), frames)``.
    Like the reference it removes the ``[None, None]`` sentinels from ``image_points`` in
    place (helpers.py:342-346); the epipolar lines the reference draws into ``frames``
    (helpers.py:365) are cosmetic and are not drawn."""
    torch = _torch()
    s = session or MocapSession.default()
    for pts in image_points:
        try:
            pts.remove([None, None])
        except ValueError:
            pass
    n_cam = len(camera_poses)
    with s._lock:
        ctx = s.ctx_with_poses(camera_poses)
        MB = ctx.cfg.max_blobs
        xy = np.zeros((n_cam, MB, 2), dtype=np.int32)
        n = np.zeros((n_cam,), dtype=np.int32)
        for c in range(n_cam):
            k = len(image_points[c])
            if k > MB:
                raise MocapError(-1, f"camera {c} has {k} points; context keeps {MB}")
            n[c] = k
            if k:
                xy[c, :k] = np.asarray(image_points[c], dtype=np.int32)
        d = ctx.match_triangulate(torch.from_numpy(xy).to(ctx.torch_device), torch.from_numpy(n).to(ctx.torch_device))
        raise_on_overflow(d["flags"][0].item(), "find_point_correspondance_and_object_points")
        k = int(d["n"][0].item())
        errors = d["err"][0, :k].cpu().numpy()
        object_points = d["obj"][0, :k].cpu().numpy()
    return errors, object_points, frames


def locate_objects(object_points, errors, session=None):
    """Mirror of helpers.py:424-480: list of {"pos": ndarray(3), "heading", "error", "droneIndex"}."""
    torch = _torch()
    s = session or MocapSession.default()
    pts = np.asarray(object_points, dtype=np.float64).reshape(-1, 3)
    errs = np.asarray(errors, dtype=np.float64).reshape(-1)
    K = pts.shape[0]
    if K == 0:
        return []
    with s._lock:
        ctx = s.ctx(len(s.intrinsics), **MIRROR_LIMITS)
        R = ctx.cfg.max_roots
        if K > R:
            raise MocapError(-1, f"{K} points; context keeps {R}")
        obj = np.zeros((1, R, 3)); err = np.zeros((1, R))
        obj[0, :K] = pts; err[0, :K] = errs
        d = ctx.locate_objects(torch.from_numpy(obj).to(ctx.torch_device), torch.from_numpy(err).to(ctx.torch_device),
                               torch.tensor([K], dtype=torch.int32, device=ctx.torch_device), max_objects=K)      # only i is screened: up to one object per point (helpers.py:433-436)
        k = int(d["n"][0].item())
        rec = d["objects"][0, :k].cpu().numpy()
        di = d["drone_index"][0, :k].cpu().numpy()
    return [{"pos": rec[i, :3].copy(), "heading": float(rec[i, 3]), "error": float(rec[i, 4]), "droneIndex": int(di[i])}
            for i in range(k)]


class KalmanFilter:
    """Mirror of the reference's ``KalmanFilter`` (KalmanFilter.py): ``predict_location(objects)`` takes the list
    ``locate_objects`` returns and gives the list of ``{"pos": f32[3], "vel": f32[3], "heading": float64,
    "droneIndex": d}`` for the drones among the objects; ``reset()`` as the reference's.  Each call is a batch of one
    on a device tracker (``MocapContext.tracker``) and reads ``clock`` once (the reference reads ``time.time()`` twice
    per call)."""

    def __init__(self, num_objects, session=None, clock=time.time):
        self.num_objects = int(num_objects)
        self.session = session or MocapSession.default()
        self.clock = clock
        s = self.session
        with s._lock:
            self._ctx = s.ctx(len(s.intrinsics), **MIRROR_LIMITS)
            self._tracker = self._ctx.tracker(self.num_objects)

    def predict_location(self, objects):
        torch = _torch()
        now = float(self.clock())
        M = max(1, len(objects))
        obj = np.zeros((1, M, 5), dtype=np.float64)
        di = np.full((1, M), -1, dtype=np.int32)
        for i, o in enumerate(objects):
            obj[0, i, :3] = np.asarray(o["pos"], dtype=np.float64).reshape(3)
            obj[0, i, 3] = o["heading"]
            d = o["droneIndex"]
            di[0, i] = d if 0 <= d < self.num_objects else -1
        dev = self._ctx.torch_device
        with self.session._lock:
            located = {"objects": torch.from_numpy(obj).to(dev), "drone_index": torch.from_numpy(di).to(dev),
                       "n": torch.tensor([len(objects)], dtype=torch.int32, device=dev)}
            r = self._tracker.track_dev(located, torch.tensor([now], dtype=torch.float64, device=dev))
            r = {k: v[0].cpu().numpy() for k, v in r.items()}
        return [{"pos": r["pos"][d].copy(), "vel": r["vel"][d].copy(), "heading": np.float64(r["heading"][d]), "droneIndex": d}
                for d in range(self.num_objects) if r["present"][d]]

    def reset(self):
        self._tracker.reset(float(self.clock()) - 20)


def bundle_adjustment(image_points, camera_poses, socketio, session=None):
    """Mirror of helpers.py:244-290: returns the list of ``{"R": ndarray 3x3, "t": ndarray (3,)}``.
    ``socketio.emit("camera-pose", ...)`` fires once with the result (the reference emits on
    every residual evaluation, helpers.py:274; the UI only renders the latest, App.tsx:254-263)."""
    s = session or MocapSession.default()
    obs, mask = _split_observations(image_points)
    with s._lock:
        out, _ = s.ctx_with_poses(camera_poses).bundle_adjust(obs, mask, camera_poses)
    if socketio is not None:
        socketio.emit("camera-pose", {"camera_poses": [{"R": p["R"].tolist(), "t": p["t"].tolist()} for p in out]})
    return out


def calculate_camera_poses(image_points, socketio=None, session=None, robust=False, reject_px=None, rounds=2, init="chain"):
    """The computation of the reference's ``calculate-camera-pose`` handler (index.py:229-277): cold-start
    chain of relative poses, then bundle adjustment.  ``image_points`` is the (F, C, 2) list the UI sends
    (``data["cameraPoints"]``) with ``None`` for missing views.  ``robust=True`` starts the chain from RANSAC
    fundamental matrices (``MocapContext.calibrate_init(method="ransac")``), which mismatched points -- a stray
    reflection recorded as a camera's first point -- do not pull.  ``reject_px`` (None: every view enters the
    adjustment, as in the reference) screens views that disagree with their track by more than that many pixels out
    of the adjustment, ``rounds`` times (``MocapContext.bundle_adjust_screened``; INTEGRATION.md recommends a value).
    ``init="graph"`` starts from the pose graph of every overlapping camera pair instead of the chain
    (``MocapContext.calibrate_init(method="graph")``; RANSAC is implied, ``robust`` is ignored); with ``reject_px`` the
    first solve then sees the views the graph's translation step supports.  Returns the list of {"R", "t"}."""
    if init not in ("chain", "graph"):
        raise ValueError(f"calculate_camera_poses: unknown init {init!r} (expected 'chain' or 'graph')")
    s = session or MocapSession.default()
    obs, mask = _split_observations(image_points)
    n_cam = obs.shape[1]
    with s._lock:
        ctx = s.ctx(n_cam)
        ident = [{"R": np.eye(3), "t": np.zeros(3)} for _ in range(n_cam)]
        ctx.set_cameras(s.intrinsics[:n_cam], ident)
        graph = init == "graph"
        init = ctx.calibrate_init(obs, mask, method="graph" if graph else ("ransac" if robust else "8point"))
        start = init[0]
        ctx.set_cameras(s.intrinsics[:n_cam], start)
        if reject_px is None:
            out, _ = ctx.bundle_adjust(obs, mask, start)
        else:
            first = None
            if graph:
                first = init[2]
            elif robust:
                # the first solve sees the views that are RANSAC inliers with a neighbouring camera; the screens that
                # follow start from every view again
                inl = init[3].astype(bool)
                near = np.zeros(mask.shape, dtype=bool)
                near[:, :-1] |= inl
                near[:, 1:] |= inl
                first = (mask.astype(bool) & near).astype(np.uint8)
            out, _, _ = ctx.bundle_adjust_screened(obs, mask, start, reject_px, rounds=rounds, first_mask=first)
    if socketio is not None:
        socketio.emit("camera-pose", {"camera_poses": [{"R": p["R"].tolist(), "t": p["t"].tolist()} for p in out]})
    return out


def live_read_events(res, r, mode, drone_armed):
    """What ``Cameras._camera_read`` emits for read ``r`` of a live result (``MocapContext.live_host``; numpy views):
    returns (events, serial), events a list of (name, payload) for ``socketio.emit`` and serial the list of byte strings
    the reference writes to the drone link (helpers.py:88-133).  Nothing when the gate is closed; ``image-points`` in
    capture-only mode; ``object-points`` when triangulating, with the locator's objects and the filtered drones when
    locating.  An armed drone's heading is rounded to 4 decimals in its serial record and in the emitted payload, an
    unarmed one's is not (helpers.py:114).  A capacity flag of the read raises MocapError, as find_dot does."""
    if mode & LIVE_CAPTURE:
        raise_on_overflow(res["flags"][r], "camera_read")
    if not (mode & LIVE_CAPTURE) or not res["gate"][r]:
        return [], []
    if not (mode & LIVE_TRIANGULATE):
        first = res["first"][r]
        return [("image-points", [[int(x), int(y)] if res["blob_n"][r, c] > 0 else [None, None] for c, (x, y) in enumerate(first)])], []
    k = int(res["n"][r])
    payload = {"object_points": res["obj"][r, :k].tolist(), "errors": res["err"][r, :k].tolist(), "objects": [], "filtered_objects": []}
    serial = []
    if mode & LIVE_LOCATE:
        m = int(res["n_objects"][r])
        rec = res["objects"][r]
        payload["objects"] = [{"pos": rec[i, :3].tolist(), "heading": np.float64(rec[i, 3]), "error": np.float64(rec[i, 4]),
                               "droneIndex": int(res["drone_index"][r, i])} for i in range(m)]
        filtered = []
        for d in np.flatnonzero(res["present"][r]):
            d = int(d)
            pos, vel, heading = res["pos"][r, d], res["vel"][r, d], np.float64(res["heading"][r, d])
            if drone_armed[d]:
                heading = round(heading, 4)
                data = {"pos": [round(x, 4) for x in pos.tolist()] + [heading], "vel": [round(x, 4) for x in vel.tolist()]}
                serial.append(f"{d}{json.dumps(data)}".encode("utf-8"))
            filtered.append({"pos": pos.tolist(), "vel": vel.tolist(), "heading": heading, "droneIndex": d})
        payload["filtered_objects"] = filtered
    return [("object-points", payload)], serial


class _LiveCameras:
    """Device state of one ``Cameras`` object under :func:`camera_read`: the context, built from the first read, and
    what was last sent to it."""

    def __init__(self, ctx, raw_shape):
        self.ctx, self.raw_shape = ctx, raw_shape
        self.poses = self.world = None
        self.tracker, self.filter_obj = None, None


def _live_cameras(cams, s, frames):
    st = s._live.get(id(cams))
    C_ = int(cams.num_cameras)
    shape = tuple(np.shape(frames[0]))
    if st is not None and st.raw_shape == (C_,) + shape:
        return st
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"camera_read: the driver's frames must be H x W x 3 (got {shape})")
    in_h, in_w = shape[0], shape[1]
    params = [cams.camera_params[c] for c in range(C_)]
    rot = [int(p["rotation"]) % 4 for p in params]
    if any(r not in (0, 2) for r in rot):
        raise ValueError(f"camera_read: rotations {rot} -- only 0 and 2 are supported: a quarter turn makes the frame portrait, "
                         f"which the reference's make_square cannot feather (mocap_set_preprocess)")
    S = max(in_w, in_h)
    ctx = MocapContext(C_, S, S, s.device, **MIRROR_LIMITS)
    if s.large_holes:
        ctx.set_large_holes(True)
    ctx.set_preprocess(in_w, in_h, rot, [np.asarray(p["intrinsic_matrix"], dtype=np.float64) for p in params],
                       [np.asarray(p["distortion_coef"], dtype=np.float64).reshape(-1)[:5] for p in params])
    if st is not None:
        st.ctx.close()
    st = s._live[id(cams)] = _LiveCameras(ctx, (C_,) + shape)
    return st


def camera_read(cams, session=None, clock=time.time, jpeg=None):
    """Replacement of ``Cameras._camera_read(self)`` (helpers.py:68-135) on the device: ``cams.cameras.read()``, then
    one ``live_host`` call whose mode follows ``is_capturing_points`` / ``is_triangulating_points`` /
    ``is_locating_objects`` as the reference nests them, then the reference's emits and serial writes
    (:func:`live_read_events`).  Returns the processed frames -- with the centre dots while capturing -- in the container
    type the driver gave.  The context is built from ``camera_params`` and the first read's size; poses and the world
    matrix are re-sent only when their values change; a new ``kalman_filter`` object (start_trangulating_points) starts
    a fresh device tracker, which reads ``clock`` once per read.  The filter object itself is never called.
    ``jpeg`` (a quality, 1..100): the same call also encodes the frames side by side on the device as
    cv.imencode('.jpg', np.hstack(frames)) does at that quality (mocap_live_jpeg_host); returns (frames, the JPEG as
    uint8 (N,))."""
    s = session or MocapSession.default()
    frames, _ = cams.cameras.read()
    capture = bool(cams.is_capturing_points)
    tri = capture and bool(cams.is_triangulating_points)
    loc = tri and bool(cams.is_locating_objects)
    mode = (LIVE_CAPTURE if capture else 0) | (LIVE_TRIANGULATE if tri else 0) | (LIVE_LOCATE if loc else 0)
    with s._lock:
        st = _live_cameras(cams, s, frames)
        ctx = st.ctx
        if tri:
            poses = np.concatenate([np.concatenate([np.asarray(p["R"], dtype=np.float64).reshape(9), np.asarray(p["t"], dtype=np.float64).reshape(3)])
                                    for p in cams.camera_poses])
            if st.poses is None or not np.array_equal(st.poses, poses):
                ctx.set_cameras([np.asarray(cams.camera_params[c]["intrinsic_matrix"], dtype=np.float64) for c in range(ctx.n_cam)],
                                cams.camera_poses)
                st.poses = poses
            if cams.to_world_coords_matrix is None:
                raise TypeError("camera_read: to_world_coords_matrix is None; the reference's world transform needs it (helpers.py:99)")
            world = np.asarray(cams.to_world_coords_matrix, dtype=np.float64).reshape(4, 4)
            if st.world is None or not np.array_equal(st.world, world):
                ctx.set_world_transform(world)
                st.world = world.copy()
        tracker = None
        if loc:
            if st.tracker is None or cams.kalman_filter is not st.filter_obj:
                if st.tracker is not None:
                    st.tracker.close()
                st.tracker, st.filter_obj = Tracker(ctx, int(cams.num_objects)), cams.kalman_filter
            tracker = st.tracker
        raw = np.stack([np.asarray(f, dtype=np.uint8) for f in frames])[None]
        res = ctx.live_host(raw, mode, [float(clock())] if loc else None, tracker, want_frames=True,
                            **(dict(jpeg=True, quality=int(jpeg)) if jpeg is not None else {}))
    events, serial = live_read_events(res, 0, mode, cams.drone_armed if loc else ())
    for name, payload in events:
        cams.socketio.emit(name, payload)
    for line in serial:
        with cams.serialLock:
            cams.ser.write(line)
            time.sleep(0.001)
    out = res["frames"][0]
    if isinstance(frames, np.ndarray):
        pass
    elif isinstance(frames, tuple):
        out = type(frames)(out[c] for c in range(len(out)))
    else:
        out = [out[c] for c in range(len(out))]
    if jpeg is None:
        return out
    return out, res["jpeg"][0, :int(res["jpeg_len"][0])].copy()


class StreamFrames(np.ndarray):
    """What ``Cameras.get_frames`` returns under ``install_into(..., stream=True)``: np.hstack of the read's frames
    (helpers.py:137-141), carrying the JPEG the device made of exactly these pixels -- ``jpeg`` uint8 (N,), made at
    ``jpeg_quality`` -- for :class:`StreamCv`'s imencode.  It is read-only, so the bytes always describe its pixels; a
    caller that draws on the frames draws on a copy (``np.array(frames)``), which carries nothing.  Views and results of
    operations carry nothing either."""

    def __array_finalize__(self, obj):
        self.jpeg, self.jpeg_quality = None, None


def stream_frames(frames, jpeg, quality):
    out = np.hstack(list(frames)).view(StreamFrames)
    out.jpeg, out.jpeg_quality = jpeg, int(quality)
    out.flags.writeable = False
    return out


class StreamCv:
    """A thin proxy of the cv2 module for the reference's index.py: ``imencode('.jpg' / '.jpeg', img, params)`` of a
    :class:`StreamFrames` whose params ask for nothing but the quality its bytes were made at returns those bytes, as
    ``(True, uint8 ndarray (N,))`` -- what cv2 returns for it, byte for byte.  Every other call and attribute is cv2's."""

    def __init__(self, cv):
        self.__dict__["_cv"] = cv

    def __getattr__(self, name):
        return getattr(self._cv, name)

    def __setattr__(self, name, value):
        setattr(self._cv, name, value)

    def imencode(self, ext, img, params=None):
        if isinstance(img, StreamFrames) and img.jpeg is not None and isinstance(ext, str) and ext.lower() in (".jpg", ".jpeg"):
            p = [] if params is None else [int(v) for v in np.asarray(params).reshape(-1)]
            pairs = list(zip(p[0::2], p[1::2]))
            if len(p) % 2 == 0 and all(k == self._cv.IMWRITE_JPEG_QUALITY and v == img.jpeg_quality for k, v in pairs) \
                    and (pairs or img.jpeg_quality == JPEG_QUALITY):
                return True, img.jpeg.copy()
        return self._cv.imencode(ext, img) if params is None else self._cv.imencode(ext, img, params)


PATCHED_NAMES = ("triangulate_point", "triangulate_points", "calculate_reprojection_error",
                 "calculate_reprojection_errors", "find_point_correspondance_and_object_points",
                 "bundle_adjustment", "locate_objects")


def install_into(helpers_module, *also, session=None, tracker=False, large_holes=False, live=False, stream=False):
    """Point a loaded reference ``helpers`` module at the CUDA path (INTEGRATION.md).

    ``also``: modules that imported the hot-path names BY VALUE -- the reference's ``index.py`` does
    (``from helpers import ... bundle_adjustment, triangulate_points, calculate_reprojection_errors``,
    index.py:1), so ``calculate_camera_pose`` (index.py:254,272,274,275) would keep the CPU functions.
    Every name of PATCHED_NAMES such a module holds is re-bound as well:
    ``install_into(helpers, sys.modules[__name__])`` from inside index.py.

    ``tracker=True`` also re-binds ``KalmanFilter`` (in helpers and in every module of ``also`` that holds it) to
    :class:`KalmanFilter` on this session, which ``start_trangulating_points`` (helpers.py:175) looks up at call
    time; the default leaves the reference's CPU filter in place.

    ``large_holes=True``: the session made here reproduces holed blobs wider or taller than 62 pixels (a marker close to
    a camera, which preprocessing turns into a ring; a lit fixture with dark spots) as cv2 does, at about 166 KB of
    device memory per SM; by default ``_find_dot`` raises on such a frame.  A ``session`` passed in keeps its own
    setting.

    ``live=True`` also replaces ``_camera_read`` on the decorated class with :func:`camera_read`: the whole read --
    preprocessing, S1-S3, the world transform, locate_objects and the tracker -- in one device call per read, the
    driver call, emits and serial writes staying in Python.

    ``stream=True`` (with ``live=True``) also moves the camera stream's JPEG encoding (index.py:55-56) into that call:
    ``get_frames`` returns np.hstack of the read's frames as a :class:`StreamFrames` carrying the JPEG the device made of
    them at cv2's default quality, and ``cv`` in every module of ``also`` that holds it is re-bound to a
    :class:`StreamCv` proxy, whose ``imencode('.jpg', frames)`` returns those bytes -- cv2's, byte for byte -- and hands
    every other call to cv2."""
    if stream and not live:
        raise ValueError("install_into: stream=True needs live=True (the JPEG is made in the live read's device call)")
    cams = helpers_module.Cameras.instance()
    s = session or MocapSession.install([np.asarray(p["intrinsic_matrix"], dtype=np.float64) for p in cams.camera_params],
                                        large_holes=large_holes)
    # helpers.Cameras is a Singleton WRAPPER object (Singleton.py:17-37); _camera_read looks _find_dot up on the
    # decorated class of the instance, so that is where the replacement goes
    type(cams)._find_dot = lambda self, img: find_dot(img, s)
    if live:
        def _camera_read(self):
            return camera_read(self, s)
        _camera_read.__mocap_b200__ = True
        type(cams)._camera_read = _camera_read
    if stream:
        def get_frames(self):
            frames, jpeg = camera_read(self, s, jpeg=JPEG_QUALITY)
            return stream_frames(frames, jpeg, JPEG_QUALITY)
        get_frames.__mocap_b200__ = True
        type(cams).get_frames = get_frames
        for mod in also:
            cv = getattr(mod, "cv", None)
            if cv is not None and not isinstance(cv, StreamCv):
                mod.cv = StreamCv(cv)
    repl = {
        "triangulate_point": lambda ip, cp: triangulate_point(ip, cp, s),
        "triangulate_points": lambda ip, cp: triangulate_points(ip, cp, s),
        "calculate_reprojection_error": lambda ip, op, cp: calculate_reprojection_error(ip, op, cp, s),
        "calculate_reprojection_errors": lambda ip, op, cp: calculate_reprojection_errors(ip, op, cp, s),
        "find_point_correspondance_and_object_points":
            lambda ip, cp, fr: find_point_correspondance_and_object_points(ip, cp, fr, s),
        "bundle_adjustment": lambda ip, cp, sio: bundle_adjustment(ip, cp, sio, s),
        "locate_objects": lambda op, er: locate_objects(op, er, s),
    }
    for name, fn in repl.items():
        fn.__name__ = name
        fn.__mocap_b200__ = True
        setattr(helpers_module, name, fn)
        for mod in also:
            if hasattr(mod, name):
                setattr(mod, name, fn)
    if tracker:
        class _KalmanFilter(KalmanFilter):
            __mocap_b200__ = True

            def __init__(self, num_objects, session=None, clock=time.time):
                super().__init__(num_objects, session or s, clock)
        _KalmanFilter.__name__ = _KalmanFilter.__qualname__ = "KalmanFilter"
        setattr(helpers_module, "KalmanFilter", _KalmanFilter)
        for mod in also:
            if hasattr(mod, "KalmanFilter"):
                setattr(mod, "KalmanFilter", _KalmanFilter)
    return s

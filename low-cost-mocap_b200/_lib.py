"""ctypes binding of libmocap_b200.so (include/mocap_b200.h).  No fallback: if the
library or an H100 is missing, every entry point raises."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmocap_b200.so")

MOCAP_OK = 0
F_SEGMENTS, F_BLOBS, F_ROOTS, F_CANDS, F_GROUPS = 1, 2, 4, 8, 16


class MocapError(RuntimeError):
    def __init__(self, status, text):
        super().__init__(f"libmocap_b200 status {status}: {text}")
        self.status = status


class Config(C.Structure):
    _fields_ = [("device", C.c_int), ("n_cam", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("max_blobs", C.c_int), ("max_segments", C.c_int), ("max_roots", C.c_int),
                ("max_cands", C.c_int), ("max_groups", C.c_int)]


class BAOptions(C.Structure):
    _fields_ = [("ftol", C.c_double), ("xtol", C.c_double), ("gtol", C.c_double),
                ("max_nfev", C.c_int), ("jacobian", C.c_int), ("prefit", C.c_int), ("prefit_max_iter", C.c_int), ("engine", C.c_int)]


class BAReport(C.Structure):
    _fields_ = [("cost_initial", C.c_double), ("cost_final", C.c_double), ("optimality", C.c_double),
                ("n_iterations", C.c_int), ("n_fev", C.c_int), ("status", C.c_int), ("n_residuals", C.c_int),
                ("prefit_cost_initial", C.c_double), ("prefit_cost_final", C.c_double),
                ("prefit_iterations", C.c_int), ("n_launches", C.c_int), ("n_tr_solves", C.c_int),
                ("n_tr_newton", C.c_int), ("phase_ms", C.c_float * 8)]


class RansacOptions(C.Structure):
    _fields_ = [("threshold_px", C.c_double), ("hypotheses", C.c_int), ("seed", C.c_uint64)]


class GraphOptions(C.Structure):
    _fields_ = [("min_common", C.c_int), ("min_inliers", C.c_int), ("min_angle_deg", C.c_double), ("rot_outlier_deg", C.c_double),
                ("irls_rounds", C.c_int)]


class GraphPair(C.Structure):
    _fields_ = [("a", C.c_int), ("b", C.c_int), ("common", C.c_int), ("inliers", C.c_int), ("candidate", C.c_int),
                ("in_front", C.c_int), ("median_angle_deg", C.c_double), ("rot_residual_deg", C.c_double), ("used", C.c_int)]


class BAProblem(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("mask", C.c_void_p), ("n_points_max", C.c_int), ("n_points", C.c_void_p),
                ("R", C.c_void_p), ("t", C.c_void_p), ("report", C.c_void_p)]


LIVE_SLICES = ("flags", "gate", "blob_n", "first", "n", "obj", "err", "n_objects", "objects", "drone_index", "called", "pos",
               "vel", "heading", "present", "chosen")


class LiveLayout(C.Structure):
    _fields_ = [(name, C.c_uint64) for name in LIVE_SLICES] + [("total", C.c_uint64)]


MOCAP_BA_MAX_BATCH = 16

# every symbol include/mocap_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "mocap_default_config": (None, [C.POINTER(Config), C.c_int, C.c_int, C.c_int]),
    "mocap_create": (C.c_int, [C.POINTER(_P), C.POINTER(Config)]),
    "mocap_destroy": (None, [_P]),
    "mocap_last_error": (C.c_char_p, [_P]),
    "mocap_status_string": (C.c_char_p, [C.c_int]),
    "mocap_set_stream": (C.c_int, [_P, _P]),
    "mocap_set_cameras": (C.c_int, [_P, _P, _P, _P]),
    "mocap_set_world_transform": (C.c_int, [_P, _P]),
    "mocap_set_large_holes": (C.c_int, [_P, C.c_int]),
    "mocap_detect_dev": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
    "mocap_match_triangulate_dev": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, _P]),
    "mocap_pipeline_dev": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
    "mocap_pipeline_host": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
    "mocap_set_preprocess": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P]),
    "mocap_preprocess_dev": (C.c_int, [_P, _P, C.c_int, _P]),
    "mocap_pipeline_raw_dev": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "mocap_get_undistort_map": (C.c_int, [_P, C.c_int, _P, _P]),
    "mocap_locate_objects_dev": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "mocap_triangulate_dev": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P]),
    "mocap_triangulate_host": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P]),
    "mocap_reprojection_errors_host": (C.c_int, [_P, _P, _P, _P, C.c_int, _P, _P]),
    "mocap_calibrate_init_host": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, _P]),
    "mocap_ransac_default_options": (None, [C.POINTER(RansacOptions)]),
    "mocap_calibrate_init_ransac_host": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(RansacOptions), _P, _P, _P, _P, _P]),
    "mocap_fundamental_ransac_host": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(RansacOptions), _P, _P]),
    "mocap_graph_default_options": (None, [C.POINTER(GraphOptions)]),
    "mocap_calibrate_graph_host": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(RansacOptions), C.POINTER(GraphOptions), _P, _P,
                                             _P, C.POINTER(C.c_int), _P]),
    "mocap_ba_default_options": (None, [C.POINTER(BAOptions)]),
    "mocap_bundle_adjust_host": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, C.POINTER(BAOptions), C.POINTER(BAReport)]),
    "mocap_bundle_adjust_dev": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, C.POINTER(BAOptions), _P]),
    "mocap_set_ba_grid": (C.c_int, [_P, C.c_int]),
    "mocap_bundle_adjust_batch_dev": (C.c_int, [_P, C.POINTER(BAProblem), C.c_int, C.POINTER(BAOptions)]),
    "mocap_tracks_to_observations_dev": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_double, _P, _P, _P, C.c_int]),
    "mocap_pipeline_tracks_dev": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "mocap_screen_observations_dev": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, C.c_double, _P, _P]),
    "mocap_screen_observations_host": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, C.c_double, _P, _P]),
    "mocap_tracker_create": (C.c_int, [_P, C.c_int, C.POINTER(_P)]),
    "mocap_tracker_destroy": (None, [_P]),
    "mocap_tracker_reset": (C.c_int, [_P, C.c_double]),
    "mocap_track_objects_dev": (C.c_int, [_P, _P, _P, _P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P]),
    "mocap_track_objects_gated_dev": (C.c_int, [_P, _P, _P, _P, C.c_int, _P, _P, C.c_int, _P, _P, _P, _P, _P]),
    "mocap_live_layout": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(LiveLayout)]),
    "mocap_live_dev": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "mocap_live_host": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "mocap_jpeg_bound": (C.c_uint64, [C.c_int, C.c_int]),
    "mocap_encode_jpeg_dev": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_uint64, _P]),
    "mocap_live_jpeg_host": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, _P, C.c_uint64, _P]),
    "mocap_ba_residuals_host": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, C.POINTER(C.c_int)]),
    "mocap_host_alloc": (C.c_int, [C.POINTER(_P), C.c_uint64]),
    "mocap_host_free": (None, [_P]),
    "mocap_launch_count": (C.c_uint64, [_P]),
    "mocap_enable_kernel_timing": (C.c_int, [_P, C.c_int]),
    "mocap_detect_kernel_ms": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
}

_lib = None


def load():
    """dlopen the in-tree library and type every symbol.  Raises if it is not built."""
    global _lib
    if _lib is None:
        path = os.environ.get("MOCAP_B200_LIB", LIB_PATH)        # a differently-built libmocap_b200.so (tuning runs)
        if not os.path.exists(path):
            raise MocapError(-2, f"{path} is not built (run python __graft_entry__.py build); there is no CPU fallback")
        lib = C.CDLL(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(status, ctx=None):
    if status != MOCAP_OK:
        lib = load()
        text = lib.mocap_last_error(ctx).decode() if ctx else lib.mocap_status_string(status).decode()
        if not text:
            text = lib.mocap_status_string(status).decode()
        raise MocapError(status, text)

"""mocap_b200 -- H100 (sm_90a) multi-view marker-tracking core behind the Python call
surface of jyjblrd/Low-Cost-Mocap's computer_code/api/helpers.py.

  api.MocapContext   batched device API over libmocap_b200.so (C ABI, include/mocap_b200.h)
  api.*              drop-in mirrors of the reference functions (same names, arguments, results)
  synth              seeded synthetic camera streams (tests, bench)
"""
from . import synth  # noqa: F401
from ._lib import MocapError, LIB_PATH  # noqa: F401
from .api import (  # noqa: F401
    MocapContext,
    MocapSession,
    find_dot,
    find_point_correspondance_and_object_points,
    triangulate_point,
    triangulate_points,
    calculate_reprojection_error,
    calculate_reprojection_errors,
    bundle_adjustment,
    locate_objects,
    calculate_camera_poses,
    install_into,
    KalmanFilter,
    Tracker,
    camera_read,
    live_read_events,
    StreamFrames,
    StreamCv,
)

"""Runs the emulated single-pass kernel (libfused_emu built with -fsanitize=thread) on a few golden frame-sets.
Started by tests/test_device_code_on_host.py in a subprocess with libtsan preloaded."""
import ctypes
import sys

import numpy as np

root, lib_path, case = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path.insert(0, root)
from tests.hostbuild import bind, ptr  # noqa: E402
from tests.util import load_golden  # noqa: E402

lib = bind(ctypes.CDLL(lib_path), "fused_emu")
z = load_golden(case, n=4)
C, B = int(z["C"]), 4
frames = np.ascontiguousarray(z["frames"][:B])
if "crowded" in sys.argv[4:]:                            # a crowded image: the deferral path
    for k in range(70):
        y, x = 10 + 6 * (k // 35), 20 + 16 * (k % 35)
        frames[1, 1, y:y + 3, x:x + 3] = 255
K = np.ascontiguousarray(np.stack([z["K"]] * C)); R = np.ascontiguousarray(z["R"]); t = np.ascontiguousarray(z["t"].reshape(C, 3))
RM, MB, E = 128, 64, 1024
obj = np.zeros((B, RM, 3)); err = np.zeros((B, RM)); k = np.zeros(B, np.int32); fl = np.zeros(B, np.int32)
bxy = np.zeros((B * C, MB, 2), np.int32); bn = np.zeros(B * C, np.int32)
iw = np.zeros(B * C, np.uint32); sw = np.zeros(B, np.uint32); cnt = np.zeros(4, np.int64)
rc = lib.hc_pipeline_fused(ptr(frames), B, C, 640, 480, 51, ptr(K), ptr(R), ptr(t), MB, E, RM, 8, ctypes.c_uint(4096), 8, 2,
                           ptr(obj), ptr(err), ptr(k), ptr(fl), ptr(bxy), ptr(bn), ptr(iw), ptr(sw), ptr(cnt), 1)
print("RESULT", rc, cnt.tolist(), k.tolist())

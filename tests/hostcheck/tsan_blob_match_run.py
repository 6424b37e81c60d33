"""Runs the emulated blob code (warp and 128-thread variants, light and crowded image) and the emulated matcher
(libblob_emu / libmatch_emu built with -fsanitize=thread).  Started by tests/test_device_code_on_host.py in a
subprocess with libtsan preloaded."""
import ctypes
import sys

import numpy as np

root, blob_lib, match_lib = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path.insert(0, root)
from tests.hostbuild import bind, ptr  # noqa: E402
from tests.util import load_golden  # noqa: E402

bl, ml = bind(ctypes.CDLL(blob_lib), "blob_emu"), bind(ctypes.CDLL(match_lib), "match_emu")
z = load_golden("pipe_c8_m16", n=2)
img = np.ascontiguousarray(z["frames"][0, 0])
crowd = img.copy()
for k in range(70):
    y, x = 10 + 6 * (k // 35), 20 + 16 * (k % 35)
    crowd[y:y + 3, x:x + 3] = 255
for im in (img, crowd):
    for force in (0, 1):
        xy = np.zeros((64, 2), np.int32); n = np.zeros(1, np.int32); mom = np.zeros((64, 4), np.int64); fl = np.zeros(1, np.int32)
        rc = bl.hc_blob_detect(ptr(im), 640, 480, 51, 64, 4096, force, 1, ptr(xy), ptr(n), ptr(mom), ptr(fl))
        print("BLOB", rc, n[0], fl[0])
C, B = 8, 2
K = np.ascontiguousarray(np.stack([z["K"]] * C)); R = np.ascontiguousarray(z["R"]); t = np.ascontiguousarray(z["t"].reshape(C, 3))
xy = np.ascontiguousarray(z["blob_xy"][:B].astype(np.int32)); nn = np.ascontiguousarray(z["blob_n"][:B].astype(np.int32))
obj = np.zeros((B, 128, 3)); err = np.zeros((B, 128)); k = np.zeros(B, np.int32); fl = np.zeros(B, np.int32)
ml.hc_match_triangulate(ptr(K), ptr(R), ptr(t), C, ptr(xy), ptr(nn), B, 64, 128, 8, ctypes.c_uint(4096), ptr(obj), ptr(err), ptr(k), ptr(fl))
print("MATCH", k.tolist() == z["nroot"][:B].tolist())
# the chunked matcher on a grid of 2 CTAs: items of 64 groups, partial results through "global" memory, arrival counters
obj2 = np.zeros((B, 128, 3)); err2 = np.zeros((B, 128)); k2 = np.zeros(B, np.int32); fl2 = np.zeros(B, np.int32)
txy = np.zeros((B, 128, C, 2), np.int32); stats = np.zeros(3, np.int64)
ml.hc_match_triangulate_chunked(ptr(K), ptr(R), ptr(t), C, ptr(xy), ptr(nn), B, 64, 128, 8, ctypes.c_uint(4096), ctypes.c_uint(64), ctypes.c_uint(1024), 2,
                                ptr(obj2), ptr(err2), ptr(k2), ptr(fl2), ptr(txy), ptr(stats))
print("CHUNKED", bool(k2.tolist() == k.tolist() and stats[0] > 0 and stats[2] == 0 and all(np.array_equal(obj2[b, :k[b]], obj[b, :k[b]]) for b in range(B))))

"""Run under ThreadSanitizer by tests/test_large_holes_on_host.py: the full-size S1 reduction with the whole-image window
(blob_large_holes_host.cpp) on the images of an .npz (img<k>, and want<k> / flags<k>, the expected items and flags,
computed outside the sanitizer); prints LARGE <equal> per image."""
import ctypes
import sys

import numpy as np

root, lib_path, cases = sys.argv[1], sys.argv[2], np.load(sys.argv[3])
sys.path.insert(0, root)
from tests.hostbuild import bind, ptr  # noqa: E402

lib = bind(ctypes.CDLL(lib_path), "blob_large_holes")
k = 0
while f"img{k}" in cases:
    img = np.ascontiguousarray(cases[f"img{k}"], np.uint8)
    H, W = img.shape
    xy = np.zeros((64, 2), np.int32); n = np.zeros(1, np.int32); mom = np.zeros((64, 4), np.int64); fl = np.zeros(1, np.int32)
    lib.hc_blob_detect_large(ptr(img), W, H, 51, 64, 4096, 1, 3, ptr(xy), ptr(n), ptr(mom), ptr(fl))
    got = np.concatenate([mom[:n[0]], xy[:n[0]].astype(np.int64)], axis=1)
    print("LARGE", np.array_equal(got, cases[f"want{k}"].reshape(-1, 6)) and int(fl[0]) == int(cases[f"flags{k}"]), flush=True)
    k += 1

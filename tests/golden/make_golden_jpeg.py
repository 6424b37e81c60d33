"""Writes tests/golden/jpeg_cv2.npz: the bytes cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) gave for a handful
of images, with the cv2 and libjpeg-turbo versions that made them (cv2 4.13.0, libjpeg-turbo 3.1.2).  The images are
not stored: tests/jpeg_util.make_image makes them again from their seeds, and a SHA-256 of each pins that it did.  The
numpy model and the device are held to these bytes, so a cv2 elsewhere that encodes differently shows up as a failure
instead of a moved target.

    python tests/golden/make_golden_jpeg.py
"""
import hashlib
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.jpeg_util import cv2_encode, make_image  # noqa: E402

# (content, h, w, quality): every edge case of the MCU grid, every quality class, the stream's own frames
CASES = [("noise", 1, 1, 10), ("constant", 8, 8, 75), ("gradient", 16, 16, 50), ("noise", 17, 23, 1), ("dots", 33, 47, 100),
         ("frames", 240, 320, 95), ("noise", 33, 47, 100), ("frames", 320, 1280, 95)]


def main():
    digests, data, lens = [], [], []
    for content, h, w, q in CASES:
        img = make_image(content, h, w, seed=5)
        b = cv2_encode(img, q)
        digests.append(hashlib.sha256(img.tobytes()).hexdigest())
        data.append(b)
        lens.append(len(b))
    jpeg = [l for l in cv2.getBuildInformation().splitlines() if l.strip().startswith("JPEG:")]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "jpeg_cv2.npz"),
                        shapes=np.array([[h, w] for _, h, w, _ in CASES], np.int32), quality=np.array([q for *_, q in CASES], np.int32),
                        content=np.array([c for c, *_ in CASES]), sha256=np.array(digests), jpeg=np.concatenate(data),
                        jpeg_len=np.array(lens, np.int64), cv2_version=np.array(cv2.__version__), jpeg_library=np.array(jpeg[0].strip() if jpeg else ""))


if __name__ == "__main__":
    main()

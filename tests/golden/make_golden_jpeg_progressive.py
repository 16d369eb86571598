"""Generates tests/golden/jpeg_progressive_golden.npz: progressive JPEGs written by libjpeg-turbo (through cv2's
IMWRITE_JPEG_PROGRESSIVE, which is what the reference's JpegProgressive option runs), with the pixels they were
written from.  Small images over gray / BGR / BGRA, odd sizes and the quality range, so that a cv2 whose
libjpeg-turbo writes different bytes shows up as a fixture mismatch in tests/test_jpeg_progressive_core.py.

Run:  python tests/golden/make_golden_jpeg_progressive.py
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests.jpeg_progressive_cases import image  # noqa: E402

CASES = [("noise", 7, 5, 1, 100), ("gradient", 33, 47, 3, 75), ("edges", 40, 24, 4, 10), ("noise", 16, 16, 3, 1),
         ("gradient", 15, 17, 1, 50), ("edges", 64, 48, 3, 95), ("noise", 31, 9, 3, 85)]


def main():
    out = {}
    for content, w, h, ch, q in CASES:
        img = image(content, w, h, ch, seed=1)
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
        assert ok
        name = f"{content}_{w}x{h}c{ch}q{q}"
        out[name + "_img"] = img
        out[name + "_jpg"] = np.frombuffer(enc.tobytes(), dtype=np.uint8)
        out[name + "_q"] = np.int32(q)
    path = os.path.join(ROOT, "tests", "golden", "jpeg_progressive_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

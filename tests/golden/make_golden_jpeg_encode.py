"""Writes tests/golden/jpeg_encode/jpeg_encode.npz: a few frames of the encoder corpus and the files cv2.imencode('.jpg') wrote for them, so that the
GPU encoder's test has OpenCV's bytes where cv2 is not installed.  Run from the repository root: python tests/golden/make_golden_jpeg_encode.py"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import jpeg_encode_spec as E  # noqa: E402

CASES = [("noise", 17, 23, 95), ("blurred", 64, 48, 50), ("checker", 9, 9, 100), ("ffbytes", 40, 24, 95), ("gradient", 333, 217, 10)]


def main():
    out = {}
    for i, (kind, w, h, q) in enumerate(CASES):
        img = E.frame(kind, w, h)
        out[f"img{i}"] = img
        out[f"jpg{i}"] = np.frombuffer(cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes(), np.uint8)
        out[f"q{i}"] = np.int32(q)
    np.savez_compressed(os.path.join(HERE, "jpeg_encode", "jpeg_encode.npz"), n=np.int32(len(CASES)), **out)


if __name__ == "__main__":
    main()

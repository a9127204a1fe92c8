"""Writes tests/golden/reference_jpeg_encode.npz: cv2.imencode's bytes (OpenCV 4.13, libjpeg-turbo 3.1.2) for a subset
of tests/jpeg_encode_cases.py's frames, so the encoder is checked against the files that defined its contract as well
as against whatever cv2 the test machine has.  Keys: 'jpg:<h>x<w>:<kind>:<q>' uint8 bytes; the frames are regenerated
from tests/jpeg_encode_cases.py."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import jpeg_encode_cases as C  # noqa: E402

CASES = [(1, 1, "noise", 95), (1, 17, "smooth", 75), (7, 9, "noise", 100), (17, 33, "overlay", 95),
         (17, 33, "saturated", 1), (97, 131, "noise", 50), (97, 131, "overlay", 5), (240, 427, "smooth", 95),
         (480, 854, "overlay", 95), (480, 854, "smooth", 75)]


def key(h, w, kind, q):
    return f"jpg:{h}x{w}:{kind}:{q}"


def main():
    import cv2
    out = {"cv2_version": np.array(cv2.__version__)}
    for h, w, kind, q in CASES:
        ok, buf = cv2.imencode(".jpg", C.frame(h, w, kind), [cv2.IMWRITE_JPEG_QUALITY, q])
        assert ok
        out[key(h, w, kind, q)] = buf.reshape(-1)
    np.savez_compressed(os.path.join(HERE, "reference_jpeg_encode.npz"), **out)


if __name__ == "__main__":
    main()

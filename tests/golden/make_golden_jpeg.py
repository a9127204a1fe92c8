"""Writes tests/golden/reference_jpeg.npz: a subset of tests/jpeg_cases.py's files with cv2.imdecode's decodes
(OpenCV 4.13, libjpeg-turbo 3.1.2), so the device decoder is checked against the decodes that defined the contract
as well as against whatever cv2 the test machine has.  Keys: 'file:<name>' (uint8 bytes), 'bgr:<name>'."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import jpeg_cases  # noqa: E402

NAMES = ["cv2_444_q75_97x131", "cv2_422_q95_97x131", "cv2_440_q50_33x45", "cv2_420_q100_97x131", "cv2_420_q5_48x70",
         "cv2_420_q100_sat", "cv2_420_opt", "cv2_420_rst7", "cv2_422_rstrow", "cv2_gray_33x45", "cv2_420_q75_1x17"]


def main():
    import cv2
    files = dict(jpeg_cases.cv2_matrix())
    files.update(jpeg_cases.pillow_files())
    out = {}
    for name in NAMES + ["pil_420_q90", "pil_422_q30"]:
        out["file:" + name] = np.frombuffer(files[name], np.uint8)
    out["file:cut_short"] = np.frombuffer(jpeg_cases.cut_short(files["cv2_420_q75_97x131"]), np.uint8)
    for k in list(out):
        name = k[len("file:"):]
        out["bgr:" + name] = cv2.imdecode(out[k], cv2.IMREAD_COLOR)
    np.savez_compressed(os.path.join(HERE, "reference_jpeg.npz"), **out)


if __name__ == "__main__":
    main()

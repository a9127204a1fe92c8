"""Writes tests/golden/reference_overlay.npz: the reference's own overlay_mask (dataloaders/helpers.py:15-36,
unmodified, OpenCV 4.13) on seeded frames and masks, so tests/test_overlay.py holds ops.overlay_mask's rule to the
picture the reference drew.

Run in the build container only (needs /root/reference and cv2; neither is needed to USE the fixture):

    python tests/golden/make_golden_overlay.py

helpers.py does not import on numpy 2 as it stands (``np.bool``); the script sets ``np.bool = bool`` before loading it
and changes nothing else.  The helper is called as the reference's test loop would call it with a frame scaled to
[0, 1] (frame / 255, not im_normalize's min-max stretch) and the colour BGR red (0, 0, 1).  Keys: 'frame:<k>' uint8
[H,W,3], 'mask:<k>' uint8 [H,W], 'out:<k>' float32 [H,W,3] on the 0..1 scale."""
import importlib.util
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/dataloaders/helpers.py"
CASES = [(48, 70), (33, 45), (97, 131), (120, 214), (5, 7)]


def main():
    import cv2
    import scipy.ndimage  # noqa: F401  (imported before the shim: numpy.ma does not load with np.bool set)
    np.bool = bool                                             # the helper's ma.astype(np.bool) on numpy 2
    spec = importlib.util.spec_from_file_location("ref_helpers", REF)
    helpers = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(helpers)
    rng = np.random.default_rng(23)
    out = {"cv2_version": np.array(cv2.__version__)}
    for k, (h, w) in enumerate(CASES):
        frame = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        yy, xx = np.mgrid[0:h, 0:w]
        blob = ((yy - h * 0.5) ** 2 / (h * 0.3) ** 2 + (xx - w * 0.4) ** 2 / (w * 0.3) ** 2) < 1.0
        hole = ((yy - h * 0.5) ** 2 + (xx - w * 0.4) ** 2) < (min(h, w) * 0.08) ** 2
        mask = (blob & ~hole) | (rng.random((h, w)) > 0.985)
        if k == 4:
            mask[:, :] = True                                  # touches every border
        mask = mask.astype(np.uint8)
        res = helpers.overlay_mask(frame / 255.0, mask, color=np.array([0.0, 0.0, 1.0]))
        out[f"frame:{k}"] = frame
        out[f"mask:{k}"] = mask
        out[f"out:{k}"] = res.astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "reference_overlay.npz"), **out)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Draws a folder of result PNGs over their DAVIS frames on the GPU and writes the pictures as JPEG files and / or one
MJPEG video per sequence: any run's ``Results/`` folder, this project's or the reference's, or another method's masks,
the same folders evaluate_results.py scores.

    python visualize_results.py                                  # <save root>/Results over <db root>, val_seqs.txt
    python visualize_results.py --results DIR --seq blackswan --video --fps 24 --out overlays
    python visualize_results.py --davis 2017 --results DIR --db-root DAVIS-2017 --video   # label maps, per object

Each result ``<seq>/<stem>.png`` is drawn over ``JPEGImages/480p/<seq>/<stem>.jpg`` (osvos_pytorch_b200/visualize.py,
DESIGN.md §25) and written as ``<out>/<seq>_overlay/<stem>.jpg`` (``--frames``, the default when ``--video`` is not
given) and / or ``<out>/<seq>_overlay.avi`` (``--video``; its frames are those JPEG files byte for byte).
``--threshold``: with DAVIS-2016 a pixel is the object when its byte is >= T, drawn in red with a black outline (128
is probability 0.5 for masks and probability maps; the reference's bytescaled files are min-max stretched per frame, so
there 128 is half way between the frame's extremes).  ``--davis 2017``: the results are PNGs of object ids, each object
drawn in its palette colour (the file's own palette, else the DAVIS palette) with its own outline."""
import argparse
import os

import torch

from mypath import Path
from osvos_pytorch_b200 import visualize


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--results", default=None, help="folder with one sub-folder of PNGs per sequence "
                                                    "(default: <save root>/Results)")
    ap.add_argument("--db-root", default=None, help="DAVIS root with JPEGImages/480p (default: mypath.Path.db_root_dir())")
    ap.add_argument("--seq", action="append", default=None, metavar="NAME",
                    help="draw this sequence (repeatable; default: the sequences of the split's list that have results)")
    ap.add_argument("--davis", default="2016", choices=["2016", "2017"],
                    help="2017: palette result files of object ids, each object in its own colour")
    ap.add_argument("--threshold", type=int, default=None, help="the object is byte >= T (default 128; DAVIS-2016 only)")
    ap.add_argument("--quality", type=int, default=95, help="JPEG quality (1..100; 95 is cv2.imwrite's default)")
    ap.add_argument("--frames", action="store_true", help="write <out>/<seq>_overlay/<stem>.jpg (default unless --video)")
    ap.add_argument("--video", action="store_true", help="write <out>/<seq>_overlay.avi (MJPEG)")
    ap.add_argument("--fps", type=float, default=24.0, help="frame rate of --video (DAVIS is 24 frames/s)")
    ap.add_argument("--out", default=None, help="output folder (default: the results folder)")
    ap.add_argument("--decode", default="device", choices=["host", "device"],
                    help="decode the JPEGs and PNGs on the GPU (device) or with cv2 / Pillow (host); the files written "
                         "are the same")
    ap.add_argument("--gpu-id", type=int, default=0)
    a = ap.parse_args(argv)
    if a.davis == "2017" and a.threshold is not None:
        ap.error("--threshold has no meaning with --davis 2017: the results are object ids, not probabilities")
    if not 1 <= a.quality <= 100:
        ap.error("--quality must lie in 1..100")
    if not a.fps > 0:
        ap.error("--fps must be positive")
    threshold = 128 if a.threshold is None else a.threshold
    results = a.results if a.results is not None else os.path.join(Path.save_root_dir(), "Results")
    db_root = a.db_root if a.db_root is not None else Path.db_root_dir()
    device = torch.device("cuda", a.gpu_id)
    with torch.cuda.device(device):
        res = visualize.render_results(results, db_root, sequences=a.seq, davis=a.davis, threshold=threshold,
                                       quality=a.quality, frames=a.frames or not a.video, video=a.video, fps=a.fps,
                                       out_dir=a.out, device=device, decode=a.decode)
    out = a.out if a.out is not None else results
    for seq, n in res["sequences"].items():
        print(f"{seq}: {n} frames -> " + ", ".join(
            ([os.path.join(out, seq + "_overlay", "")] if a.frames or not a.video else [])
            + ([os.path.join(out, seq + "_overlay.avi")] if a.video else [])))
    print(f"[{res['frames']} frames; {res['fallback_files']} files decoded on the host, {res['redecoded_files']} "
          "re-decoded after a decoder status]")
    return res


if __name__ == "__main__":
    main()

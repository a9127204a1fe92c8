#!/usr/bin/env python
"""Scores a folder of result PNGs against the DAVIS-2016 annotations (J and F: mean, recall, decay), the way the
benchmark is used: any run's ``Results/`` folder, this project's or the reference's, or another method's masks.

    python evaluate_results.py                                  # <save root>/Results against <db root>, val_seqs.txt
    python evaluate_results.py --results DIR --seq blackswan --seq cows --threshold 128 --json scores.json
    python evaluate_results.py --davis 2017 --results DIR --db-root DAVIS-2017   # per object, ImageSets/2017/val.txt

The files are decoded on the GPU (osvos_pytorch_b200/png.py, DESIGN.md §22).  ``--threshold``: a pixel is foreground
when its byte is >= T.  128 is probability 0.5 for masks and probability maps; the reference's files are min-max
stretched per frame (bytescale), so there 128 is half way between the frame's extremes, not probability 0.5.

``--davis 2017``: the results and annotations are PNGs of object ids (palette files, DESIGN.md §24); every object of
every sequence is scored on its own and the dataset line is the mean over all objects, with J&F = (J_M + F_M) / 2."""
import argparse
import json
import os

import torch

from mypath import Path
from osvos_pytorch_b200 import evaluation


def line(name, st):
    return name + " (frames 1 .. n-2): " + "  ".join(
        f"{m} M/O/D: {st[m]['M']:.4f} / {st[m]['O']:.4f} / {st[m]['D']:.4f}" for m in ("J", "F"))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--results", default=None, help="folder with one sub-folder of PNGs per sequence "
                                                    "(default: <save root>/Results)")
    ap.add_argument("--db-root", default=None, help="DAVIS-2016 root (default: mypath.Path.db_root_dir())")
    ap.add_argument("--seq", action="append", default=None, metavar="NAME",
                    help="score this sequence (repeatable; default: the sequences of val_seqs.txt that have results)")
    ap.add_argument("--threshold", type=int, default=None, help="foreground is byte >= T (default 128; DAVIS-2016 only)")
    ap.add_argument("--davis", default="2016", choices=["2016", "2017"],
                    help="2017: palette result and annotation files of object ids, scored per object")
    ap.add_argument("--decode", default="device", choices=["host", "device"],
                    help="decode the PNGs on the GPU (device) or with cv2 (host); the scores are the same")
    ap.add_argument("--json", default=None, metavar="OUT", help="write the full result here")
    ap.add_argument("--gpu-id", type=int, default=0)
    a = ap.parse_args(argv)
    if a.davis == "2017" and a.threshold is not None:
        ap.error("--threshold has no meaning with --davis 2017: the results are object ids, not probabilities")
    threshold = 128 if a.threshold is None else a.threshold
    results = a.results if a.results is not None else os.path.join(Path.save_root_dir(), "Results")
    db_root = a.db_root if a.db_root is not None else Path.db_root_dir()
    device = torch.device("cuda", a.gpu_id)
    with torch.cuda.device(device):
        res = evaluation.score_results(results, db_root, sequences=a.seq, threshold=threshold, device=device,
                                       decode=a.decode, davis=a.davis)
    host = "Pillow" if a.davis == "2017" else "cv2"
    tail = (f"  [{res['frames']} frames; {res['fallback_files']} files decoded by {host}, {res['redecoded_files']} "
            "re-decoded after a decoder status]")
    if a.davis == "2017":
        for seq, r in res["sequences"].items():
            for k, ob in r["objects"].items():
                print(line(f"Scores of {seq} object {k}", ob["statistics"]))
        d = res["dataset"]
        print(line(f"Scores of the dataset, mean over {d['objects']} objects", d) + f"  J&F: {d['J&F']:.4f}" + tail)
    else:
        for seq, r in res["sequences"].items():
            print(line("Scores of " + seq, r["statistics"]))
        print(line(f"Scores of the dataset, mean over {len(res['sequences'])} sequences", res["dataset"]) + tail)
    if a.json:
        with open(a.json, "w") as f:
            extra = dict(davis="2017") if a.davis == "2017" else dict(threshold=threshold)
            json.dump(dict(results=os.path.abspath(results), **extra, **res), f, indent=1)
    return res


if __name__ == "__main__":
    main()

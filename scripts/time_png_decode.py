#!/usr/bin/env python
"""Times the device PNG decoder (ops.decode_png, DESIGN.md §22) at 480x854 against single-thread cv2.imdecode, and the
results scorer with decode="device" against decode="host".

    python scripts/time_png_decode.py [--rounds 5] [--frames 240] [--json OUT]

Device times are CUDA events around `reps` back-to-back calls on blobs already on the device (upload excluded), the
variants alternated over `rounds` rounds, median reported.  Host figures are wall clock on one thread.  The card's
name, power limit and maximum SM clock are printed with the table: an absolute time is worth nothing without them."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import png_cases as C          # noqa: E402
import png_decode_cases as D   # noqa: E402
from osvos_pytorch_b200 import evaluation, ops, png   # noqa: E402

H, W = 480, 854


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the table is still worth printing
        return f"unknown ({e})"


def own(maps):
    out, lengths = ops.encode_png(torch.from_numpy(np.stack(maps)).cuda())
    out, lengths = out.cpu().numpy(), lengths.cpu().tolist()
    return [out[i, :ln].tobytes() for i, ln in enumerate(lengths)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=240, help="frames of the synthetic tree the scorer is timed on")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_png_decode.py measures the GPU decoder; no CUDA device found")
    import cv2
    cv2.setNumThreads(1)
    maps = {k: [C.content(k, H, W, seed=i) for i in range(64)] for k in ("bytescale", "mask")}
    sets = {}
    for kind, ms in maps.items():
        sets[f"own {kind}"] = own(ms)
        sets[f"pillow {kind}"] = [D.pillow(m) for m in ms]
        sets[f"cv2 {kind}"] = [D.opencv(m) for m in ms]
    rows = []
    variants = []
    for name, files in sets.items():
        t0 = time.perf_counter()
        for f in files:
            cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_GRAYSCALE)
        host_us = (time.perf_counter() - t0) / len(files) * 1e6
        t0 = time.perf_counter()
        parsed = [png.parse(f) for f in files]
        blob = png.pack(parsed)
        pack_us = (time.perf_counter() - t0) / len(files) * 1e6
        for batch in (1, 12, 64):
            b = png.pack(parsed[:batch])
            variants.append(dict(name=name, batch=batch, blob=torch.from_numpy(b).cuda(), nseg=png.segment_count(b),
                                 out=torch.empty((batch, H, W), dtype=torch.uint8, device="cuda"), times=[],
                                 host_us=host_us, pack_us=pack_us, bytes=sum(len(f) for f in files) / len(files)))
    for v in variants:   # warm up every shape, and check the pixels once
        out, status = ops.decode_png(v["blob"], v["batch"], H, W, v["nseg"], out=v["out"])
        kind = v["name"].split()[1]
        assert int(status.abs().sum()) == 0 and np.array_equal(out.cpu().numpy(), np.stack(maps[kind][:v["batch"]]))
    for _ in range(a.rounds):
        for v in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.reps):
                ops.decode_png(v["blob"], v["batch"], H, W, v["nseg"], out=v["out"])
            e1.record()
            e1.synchronize()
            v["times"].append(e0.elapsed_time(e1) * 1e3 / a.reps / v["batch"])
    print(f"card: {card()}")
    print(f"{'files':18s} {'batch':>5s} {'segments/file':>13s} {'device us/frame':>16s} {'min..max':>15s} "
          f"{'cv2 1 thread us':>16s} {'parse+pack us':>14s} {'file bytes':>10s}")
    for v in variants:
        med = statistics.median(v["times"])
        rows.append(dict(files=v["name"], batch=v["batch"], segments=v["nseg"] / v["batch"], device_us=med,
                         device_us_min=min(v["times"]), device_us_max=max(v["times"]), cv2_us=v["host_us"],
                         parse_pack_us=v["pack_us"], file_bytes=v["bytes"]))
        print(f"{v['name']:18s} {v['batch']:5d} {v['nseg'] / v['batch']:13.0f} {med:16.1f} "
              f"{min(v['times']):7.1f}..{max(v['times']):<7.1f} {v['host_us']:16.1f} {v['pack_us']:14.1f} {v['bytes']:10.0f}")

    # the scorer on a synthetic tree: results in the project's own format, annotations by Pillow as DAVIS ships them
    scorer = {}
    with tempfile.TemporaryDirectory() as tmp:
        nseq, per = 4, a.frames // 4
        os.makedirs(os.path.join(tmp, "db"))
        with open(os.path.join(tmp, "db", "val_seqs.txt"), "w") as f:
            f.write("\n".join(f"s{k}" for k in range(nseq)) + "\n")
        for k in range(nseq):
            rd, ad = os.path.join(tmp, "Results", f"s{k}"), os.path.join(tmp, "db", "Annotations", "480p", f"s{k}")
            os.makedirs(rd)
            os.makedirs(ad)
            for i in range(per):
                j = (k * per + i) % 64
                with open(os.path.join(rd, f"{i:05d}.png"), "wb") as f:
                    f.write(sets["own mask"][j])
                with open(os.path.join(ad, f"{i:05d}.png"), "wb") as f:
                    f.write(sets["pillow mask"][(j + 1) % 64])
        ref = None
        for mode, readers in (("device", 1), ("host", 1), ("device", 4), ("host", 4)):
            times = []
            for _ in range(3):
                t0 = time.perf_counter()
                res = evaluation.score_results(os.path.join(tmp, "Results"), os.path.join(tmp, "db"), decode=mode,
                                               readers=readers)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            counts = {s: r["counts"] for s, r in res["sequences"].items()}
            assert ref is None or counts == ref
            ref = counts
            scorer[f"{mode}, {readers} reader(s)"] = min(times[1:])
            print(f"score_results on {nseq * per} frames, decode={mode}, {readers} reader thread(s): "
                  f"{min(times[1:]):.3f} s ({min(times[1:]) / (nseq * per) * 1e3:.2f} ms per frame)")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card(), decode=rows, score_results_s=scorer), f, indent=1)


if __name__ == "__main__":
    main()

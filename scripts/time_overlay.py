"""Timing of the segmentation overlays (DESIGN.md §23): ops.overlay_mask + ops.encode_jpeg (csrc/jpeg_encode.cu)
against cv2.imencode on this host, and what writing overlays costs SequenceSegmenter.

    python scripts/time_overlay.py [--out results] [--iters 200] [--frames 200] [--rounds 3]

Measures:
  1. overlay + encode device time per 480x854 frame from CUDA events, at batch 1 and 12, quality 75 and 95, and the
     encode alone; file sizes against cv2.imencode's (they are equal byte for byte);
  2. cv2.imencode('.jpg') of the same frames on this host, one thread;
  3. SequenceSegmenter (bgr8 frames, output bytescale) frames/s at 480x854: no writing, encode="png" files written,
     encode="png" + overlay="jpeg" files written, alternated over the rounds.
Writes <out>/time_overlay.json; the GPU's name, power limit and SM clocks and the CPU count go with the numbers.  Files
are written to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from time_output_res import event_ms, gpu_info  # noqa: E402


def frames_and_logits(n, h=480, w=854):
    import jpeg_encode_cases
    frames = np.stack([jpeg_encode_cases.frame(h, w, "smooth", seed=i) for i in range(n)])
    yy, xx = np.mgrid[0:h, 0:w]
    logits = np.stack([(1.0 - (yy - h * 0.5) ** 2 / (h * 0.3) ** 2 - (xx - w * (0.4 + 0.01 * i)) ** 2 / (w * 0.25) ** 2)
                       for i in range(n)]).astype(np.float32)[:, None]
    return frames, logits


def time_kernels(iters):
    import cv2
    from osvos_pytorch_b200 import ops
    host_f, host_l = frames_and_logits(12)
    rows = []
    for q in (75, 95):
        for n in (1, 12):
            x = torch.from_numpy(host_f[:n]).cuda()
            lg = torch.from_numpy(host_l[:n]).cuda()
            img = ops.overlay_mask(x, lg)
            out, lengths = ops.encode_jpeg(img, q)

            def both():
                ops.overlay_mask(x, lg, out=img)
                ops.encode_jpeg(img, q, out=out, lengths=lengths)
            ms = event_ms(both, iters)
            ms_enc = event_ms(lambda: ops.encode_jpeg(img, q, out=out, lengths=lengths), iters)
            sizes = lengths.cpu().tolist()
            files = out.cpu().numpy()
            ref = [cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes() for f in img.cpu().numpy()]
            same = all(files[i, :ln].tobytes() == r for i, (ln, r) in enumerate(zip(sizes, ref)))
            rows.append(dict(quality=q, batch=n, us_per_frame=1e3 * ms / n, encode_us_per_frame=1e3 * ms_enc / n,
                             bytes=sizes, cv2_bytes=[len(r) for r in ref], identical_to_cv2=same))
            print(f"overlay + encode_jpeg 480x854 q{q} batch {n:2d}: {1e3 * ms / n:7.1f} us/frame (encode alone "
                  f"{1e3 * ms_enc / n:7.1f})  {sum(sizes) / n:8.0f} B/frame, identical to cv2: {same}", flush=True)
    return rows


def time_cv2(k=48):
    import cv2
    cv2.setNumThreads(1)
    host_f, _ = frames_and_logits(12)
    rows = []
    for q in (75, 95):
        fr = list(host_f) * (k // 12)
        t0 = time.perf_counter()
        for f in fr:
            cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, q])
        us = 1e6 * (time.perf_counter() - t0) / len(fr)
        rows.append(dict(quality=q, us_per_frame_1_thread=us))
        print(f"cv2.imencode 480x854 q{q}: {us:7.1f} us/frame on 1 thread", flush=True)
    return rows


def time_segmenter(frames_n, rounds):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    net.cuda().eval()
    host_f, _ = frames_and_logits(8)
    frames = [torch.from_numpy(host_f[i % 8][None].copy()).pin_memory() for i in range(frames_n)]
    opts = dict(output="bytescale", frames="bgr8")
    segs = {"no writing": SequenceSegmenter(net, **opts),
            "png + write": SequenceSegmenter(net, encode="png", **opts),
            "png + overlay jpeg + write": SequenceSegmenter(net, encode="png", overlay="jpeg", **opts)}
    out_dir = tempfile.mkdtemp(prefix="time_overlay_")

    def run(name, n=frames_n):
        for i, r in enumerate(segs[name](iter(frames[:n]))):
            if name == "no writing":
                continue
            pngs, jpgs = r if name.startswith("png + overlay") else (r, [])
            for j, f in enumerate(pngs):
                with open(os.path.join(out_dir, f"{i:05d}_{j}.png"), "wb") as fh:
                    fh.write(f)
            for j, f in enumerate(jpgs):
                with open(os.path.join(out_dir, f"{i:05d}_{j}.jpg"), "wb") as fh:
                    fh.write(f)
    for name in segs:                                    # warm-up: allocation and graph capture of every slot
        run(name, 8)
    res = {name: [] for name in segs}
    for _ in range(rounds):
        for name in segs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(name)
            torch.cuda.synchronize()
            res[name].append(frames_n / (time.perf_counter() - t0))
    for k, v in res.items():
        print(f"SequenceSegmenter 480x854 bytescale, {k}: " + " / ".join(f"{f:.1f}" for f in v) + " frames/s",
              flush=True)
    return {"d2h_bytes_per_frame": {k: s.d2h_bytes_per_frame for k, s in segs.items()}, "frames_per_s": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_overlay.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock):", gpu, "| os.cpu_count():", os.cpu_count(), flush=True)
    res = {"gpu": gpu, "cpu_count": os.cpu_count(), "overlay_encode": time_kernels(a.iters), "cv2": time_cv2(),
           "segmenter": time_segmenter(a.frames, a.rounds)}
    res["gpu_after"] = gpu_info()
    print("GPU after:", res["gpu_after"], flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_overlay.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

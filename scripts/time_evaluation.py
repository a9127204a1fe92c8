"""Timing of DAVIS-2016 J and F scoring on the device (csrc/measures.cu, ops.davis_measures).

    python scripts/time_evaluation.py [--out results] [--launches 500] [--frames 200]

Measures:
  1. the scoring kernels (memset + three launches): us per frame over many launches (CUDA events) at batch 1 and 12
     at 480x854 and batch 1 at 1080x1920, on masks that look like segmentations (smooth blobs, a few speckles), and
     GB/s of the 5 bytes per pixel it must read (fp32 logit + uint8 mask).  Device time comes from replaying a CUDA
     graph of 50 calls; the rate of calls issued one by one from Python is reported beside it;
  2. SequenceSegmenter frames/s at 480x854, batch 1, bytescale output, with and without score=True, alternated three
     times each;
  3. the host numpy / scipy restatement (tests/davis_measures_ref.py) per 480x854 and 1080x1920 frame, on this host.
Writes <out>/time_evaluation.json; the GPU's name, power limit and SM clock limit go with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def masks(n, h, w, seed):
    """n segmentation-like masks [n,h,w] bool: two ellipses each, plus sparse speckle."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    out = np.zeros((n, h, w), dtype=bool)
    for k in range(n):
        for _ in range(2):
            cy, cx = rng.uniform(0.2, 0.8) * h, rng.uniform(0.2, 0.8) * w
            out[k] |= ((y - cy) / (0.2 * h)) ** 2 + ((x - cx) / (0.15 * w)) ** 2 <= 1
        out[k] ^= rng.random((h, w)) < 0.001
    return out


def time_kernel(n, h, w, launches):
    from osvos_pytorch_b200 import evaluation, ops
    p = masks(n, h, w, 1)
    g = masks(n, h, w, 2)
    logits = torch.from_numpy(np.where(p, 2.0, -2.0).astype(np.float32)).cuda()
    gt = torch.from_numpy(g.astype(np.uint8) * 255).cuda()
    out = torch.empty((n, 6), dtype=torch.int32, device="cuda")
    for _ in range(20):
        ops.davis_measures(logits, gt, out=out)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        ops.davis_measures(logits, gt, out=out)
    b.record()
    b.synchronize()
    us_python = a.elapsed_time(b) * 1e3 / launches
    # device time without the Python wrapper's host cost: 50 calls captured in one CUDA graph, replayed
    per_graph = 50
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        for _ in range(per_graph):
            ops.davis_measures(logits, gt, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    replays = max(1, launches // per_graph)
    a.record()
    for _ in range(replays):
        graph.replay()
    b.record()
    b.synchronize()
    us_call = a.elapsed_time(b) * 1e3 / (replays * per_graph)
    return {"n": n, "h": h, "w": w, "r": evaluation.bound_pix(h, w), "us_per_call_from_python": us_python,
            "us_per_call": us_call, "us_per_frame": us_call / n,
            "GB_per_s": 5.0 * n * h * w / (us_call * 1e-6) / 1e9,
            "share_of_hbm_datasheet": 5.0 * n * h * w / (us_call * 1e-6) / HBM_BYTES_PER_S}


def time_segmenter(frames, pairs=3):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200.inference import SequenceSegmenter
    h, w = 480, 854
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    net = net.cuda().eval()
    g = torch.Generator().manual_seed(0)
    imgs = [torch.randint(0, 256, (1, h, w, 3), generator=g, dtype=torch.uint8).pin_memory() for _ in range(8)]
    gts = [torch.from_numpy(masks(1, h, w, 10 + k).astype(np.uint8) * 255).pin_memory() for k in range(8)]

    def run(score):
        seg = SequenceSegmenter(net, output="bytescale", frames="bgr8", score=score)
        src = ((imgs[i % 8], gts[i % 8]) if score else imgs[i % 8] for i in range(frames))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in seg(src):
            pass
        if score:
            seg.frame_counts()
        torch.cuda.synchronize()
        return frames / (time.perf_counter() - t0)

    run(False)
    run(True)                                          # warm-up: graph captures, allocations
    res = {"plain": [], "score": []}
    for _ in range(pairs):
        res["plain"].append(run(False))
        res["score"].append(run(True))
    return res


def time_host(h, w, reps=5):
    import davis_measures_ref as ref
    p = masks(1, h, w, 1)[0]
    g = masks(1, h, w, 2)[0].astype(np.uint8) * 255
    logit = np.where(p, 2.0, -2.0).astype(np.float32)
    ref.counts(logit, g)
    t0 = time.perf_counter()
    for _ in range(reps):
        ref.counts(logit, g)
    return (time.perf_counter() - t0) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--frames", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_evaluation.py measures the GPU path and needs a CUDA device")
    from osvos_pytorch_b200 import build
    build.build()
    res = {"gpu": gpu_info(), "host_cpus": os.cpu_count()}
    print("GPU:", res["gpu"])
    res["kernel"] = [time_kernel(n, h, w, a.launches) for n, h, w in [(1, 480, 854), (12, 480, 854), (1, 1080, 1920)]]
    for k in res["kernel"]:
        print(f"kernel n={k['n']} {k['h']}x{k['w']} r={k['r']}: {k['us_per_call']:.2f} us/call on the device "
              f"({k['us_per_call_from_python']:.2f} us/call issued from Python), "
              f"{k['us_per_frame']:.2f} us/frame, {k['GB_per_s']:.0f} GB/s of the 5 B/pixel read")
    res["segmenter_fps"] = time_segmenter(a.frames)
    print("SequenceSegmenter 480x854 frames/s, alternated: plain " +
          " / ".join(f"{v:.1f}" for v in res["segmenter_fps"]["plain"]) + ", score=True " +
          " / ".join(f"{v:.1f}" for v in res["segmenter_fps"]["score"]))
    res["host_ms_per_frame"] = {"480x854": time_host(480, 854), "1080x1920": time_host(1080, 1920, reps=2)}
    print("host numpy/scipy restatement, ms per frame: " +
          ", ".join(f"{k} {v:.1f}" for k, v in res["host_ms_per_frame"].items()))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_evaluation.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Cost of online adaptation (DESIGN.md §28): the device time of ops.adaptation_labels at 480x854 and 1080x1920 (a CUDA
graph of repeated calls, replayed), and frames/s of the 480x854 test loop (SequenceSegmenter, bytescale PNGs encoded on
the device) with and without the default adaptation on a seeded synthetic sequence.  Prints one JSON line with the
card's name, power limit and maximum SM clock.

    python scripts/time_adaptation.py [--frames 40] [--calls 50]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from osvos_pytorch_b200 import augment, ops, training  # noqa: E402
from osvos_pytorch_b200.inference import SequenceSegmenter  # noqa: E402
from osvos_pytorch_b200.networks import vgg_osvos as vo  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _blob_mask(h, w, dev):
    """An ellipse covering about a fifth of the frame: the default erosion and distance both bite."""
    y, x = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    inside = ((y - h / 2) / (h / 4)) ** 2 + ((x - w / 2) / (w / 4)) ** 2 <= 1
    return (inside.to(torch.uint8) * 255)[None].to(dev)


def time_labels(h, w, calls, dev):
    g = torch.Generator().manual_seed(h)
    logits = (torch.randn(1, 1, h, w, generator=g) * 4).to(dev)
    mask = _blob_mask(h, w, dev)
    out = torch.empty(1, 1, h, w, device=dev)
    for _ in range(3):
        ops.adaptation_labels(logits, mask, 0.97, 15, 220, out=out)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(calls):
            ops.adaptation_labels(logits, mask, 0.97, 15, 220, out=out)
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls


def time_loop(net, frames, first, sample_fn, adapt):
    # erosion 0: the He-initialised network's masks are noise that the default erosion empties, and a frame whose
    # eroded mask is empty takes no step; the cost of an adapted frame does not depend on the radius
    ad = training.OnlineAdaptation(net, sample_fn, first, 1e-10, 0.0002, erosion=0) if adapt else None
    seg = SequenceSegmenter(net, output="bytescale", frames="bgr8", encode="png", adapt=ad)
    for _ in seg(iter(frames[:8])):                     # warm-up: allocation, graph captures of every ring slot
        pass
    skipped = ad.skipped if ad is not None else 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = sum(1 for _ in seg(iter(frames)))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return n / dt, (ad.skipped - skipped if ad is not None else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--calls", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {"card": _card(), "labels_ms": {}}
    for h, w in ((480, 854), (1080, 1920)):
        res["labels_ms"][f"{h}x{w}"] = round(time_labels(h, w, a.calls, dev), 4)
    h, w = 480, 854
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    net.to(dev)
    g = torch.Generator().manual_seed(1)
    base = torch.randint(0, 256, (1, h, w, 3), dtype=torch.uint8, generator=g)
    frames = [torch.roll(base, shifts=2 * i, dims=2).pin_memory() for i in range(a.frames)]   # a slowly panning frame
    first = _blob_mask(h, w, dev)
    img_u8 = frames[0].to(dev)
    stats = ops.label_stats_u8(first)
    rng = random.Random(0)

    def sample_fn(it):
        return augment.affine_warp_u8(img_u8, first, augment.draw_params(1, rng=rng), stats)
    plain, _ = time_loop(net, frames, first, sample_fn, False)
    adapted, skipped = time_loop(net, frames, first, sample_fn, True)
    res.update(frames=a.frames, loop_fps={"plain": round(plain, 1), "adapt": round(adapted, 2)},
               adapt_ms_per_frame=round(1000.0 / adapted, 1), adapt_skipped=skipped)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Cost of the dense CRF (DESIGN.md §29): the device time per frame of ops.dense_crf at 480x854 and 240x427 for K = 1, 2
and 4 objects (a CUDA graph of repeated calls, replayed), the lattice's vertex count, the share of a call spent building
the lattice (from the times at T = 1 and T = 5), the per-kernel device time of one 480x854 K = 1 call (torch.profiler),
and frames/s of the 480x854 test loop (SequenceSegmenter, bytescale PNGs encoded on the device) with and without the
default CRF, on a seeded synthetic sequence.  Prints one JSON line with the card's name, power limit and maximum SM
clock.

    python scripts/time_crf.py [--frames 40] [--calls 20]"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from osvos_pytorch_b200 import ops  # noqa: E402
from osvos_pytorch_b200.inference import SequenceSegmenter  # noqa: E402
from osvos_pytorch_b200.networks import vgg_osvos as vo  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _scene(h, w, dev, seed=0):
    """A colour ramp with an ellipse of one colour and some noise: a frame with edges and flat regions."""
    g = torch.Generator().manual_seed(seed)
    y, x = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    img = torch.stack([x * 255 // (w - 1), y * 255 // (h - 1), (x + y) % 256], -1)
    img = img + torch.randint(-12, 13, (h, w, 3), generator=g)
    inside = ((y - h / 2) / (h / 4)) ** 2 + ((x - w / 2) / (w / 4)) ** 2 <= 1
    img[inside] = torch.tensor([40, 180, 220])
    logits = (inside.float() * 6 - 3 + torch.randn(h, w, generator=g) * 2)[None, None]
    return img.clamp(0, 255).to(torch.uint8)[None].to(dev), logits.to(dev)


def time_crf(h, w, k, iterations, calls, dev):
    frame, logit = _scene(h, w, dev)
    maps = [torch.roll(logit, shifts=7 * i, dims=3).contiguous() for i in range(k)]
    crf = ops.CRF(iterations=iterations)
    out = torch.empty(k, 1, 1, h, w, device=dev)
    verts = torch.empty(1, dtype=torch.int32, device=dev)
    for _ in range(3):
        ops.dense_crf(frame, maps, crf, out=out, vertices=verts)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(calls):
            ops.dense_crf(frame, maps, crf, out=out)
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / calls, int(verts.item())


def profile_crf(h, w, dev):
    """Device time by kernel of one default call (the summed CUB sort and scan kernels under one name each)."""
    frame, logit = _scene(h, w, dev)
    for _ in range(3):
        ops.dense_crf(frame, [logit])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ops.dense_crf(frame, [logit])
        torch.cuda.synchronize()
    by = collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            name = ev.name
            for short in ("crf_elevate", "crf_mark", "crf_compact", "crf_neighbours", "crf_splat", "crf_blur",
                          "crf_slice", "crf_gauss_rows", "crf_update", "crf_taps", "RadixSort", "Onesweep", "Scan"):
                if short in name:
                    name = short
                    break
            by[name] += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
    return {k: round(v, 1) for k, v in by.most_common()}


def time_loop(net, frames, crf):
    seg = SequenceSegmenter(net, output="bytescale", frames="bgr8", encode="png", crf=crf)
    for _ in seg(iter(frames[:8])):                     # warm-up: allocation, graph captures of every ring slot
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = sum(1 for _ in seg(iter(frames)))
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {"card": _card(), "crf_ms": {}, "vertices": {}, "build_share": {}}
    for h, w in ((480, 854), (240, 427)):
        for k in (1, 2, 4):
            t5, verts = time_crf(h, w, k, 5, a.calls, dev)
            t1, _ = time_crf(h, w, k, 1, a.calls, dev)
            key = f"{h}x{w}_K{k}"
            res["crf_ms"][key] = round(t5, 4)
            res["build_share"][key] = round(max(0.0, t1 - (t5 - t1) / 4) / t5, 3)
            res["vertices"][f"{h}x{w}"] = verts
    res["profile_480x854_K1_us"] = profile_crf(480, 854, dev)
    h, w = 480, 854
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    net.to(dev)
    frame, _ = _scene(h, w, "cpu")
    frames = [torch.roll(frame, shifts=2 * i, dims=2).pin_memory() for i in range(a.frames)]   # a slowly panning frame
    res.update(frames=a.frames, loop_fps={"plain": round(time_loop(net, frames, None), 1),
                                          "crf": round(time_loop(net, frames, ops.CRF()), 1)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()

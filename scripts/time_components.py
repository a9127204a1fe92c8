"""Cost of the connected components and the component filter (DESIGN.md §30): the device time per call of
ops.connected_components and ops.filter_components ("largest" and "near") at 480x854 and 1080x1920, N = 1 and 12 frames,
K = 1, 2 and 4 objects, on blob masks and on the two worst cases of the labelling (a serpentine through every tile, a
checkerboard at connectivity 4); each time from a CUDA graph of `--calls` calls, replayed.  Then frames/s of the 480x854
test loop (SequenceSegmenter, bytescale PNGs encoded on the device) without the filter, with "largest" and with "near",
alternated over `--rounds` rounds.  Prints one JSON line with the card's name, power limit and maximum SM clock.

    python scripts/time_components.py [--calls 50] [--frames 60] [--rounds 3]"""
import argparse
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


def _pattern(kind, n, h, w, dev, seed=0):
    """uint8 [n,h,w]: blobs (a large ellipse and small discs, shifted per frame), the serpentine or the checkerboard."""
    y, x = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    if kind == "checkerboard":
        return ((y + x) % 2).to(torch.uint8).expand(n, h, w).contiguous().to(dev)
    if kind == "serpentine":
        m = (y % 2 == 0)
        m |= (y % 4 == 1) & (x == w - 1)
        m |= (y % 4 == 3) & (x == 0)
        return m.to(torch.uint8).expand(n, h, w).contiguous().to(dev)
    g = torch.Generator().manual_seed(seed)
    out = torch.empty(n, h, w, dtype=torch.uint8)
    for j in range(n):
        m = ((y - h / 2) / (h / 4)) ** 2 + ((x - w / 2 - 3 * j) / (w / 5)) ** 2 <= 1
        for _ in range(20):
            cy, cx = (torch.rand(2, generator=g) * torch.tensor([h, w])).tolist()
            r = 2 + 10 * float(torch.rand(1, generator=g))
            m |= (y - cy) ** 2 + (x - cx) ** 2 <= r * r
        out[j] = m
    return out.to(dev)


def _graph_ms(fn, calls):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(calls):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    graph.replay()
    b.record()
    torch.cuda.synchronize()
    del graph
    return round(a.elapsed_time(b) / calls, 4)


def time_ops(calls, dev):
    res = {}
    for h, w in ((480, 854), (1080, 1920)):
        for n in (1, 12):
            for kind, conn in (("blobs", 8), ("serpentine", 8), ("checkerboard", 4)):
                masks = _pattern(kind, n, h, w, dev)
                res[f"cc_{h}x{w}_N{n}_{kind}_c{conn}"] = _graph_ms(lambda: ops.connected_components(masks, conn), calls)
                for k in (1, 2, 4):
                    maps = [(masks.float() * 2 - 1).roll(5 * i, dims=2).unsqueeze(1).contiguous() for i in range(k)]
                    prior = _pattern("blobs", k, h, w, dev, seed=9)
                    out = torch.empty(k, n, 1, h, w, device=dev)
                    for mode in ("largest", "near"):
                        p = ops.Components(mode, connectivity=conn)
                        key = f"filter_{mode}_{h}x{w}_N{n}_K{k}_{kind}_c{conn}"
                        res[key] = _graph_ms(lambda: ops.filter_components(maps, p, prior=prior if mode == "near" else None,
                                                                           out=out), calls)
                    del maps, out
                del masks
                torch.cuda.empty_cache()
    return res


def time_loop(net, frames, components, prior):
    seg = SequenceSegmenter(net, output="bytescale", frames="bgr8", encode="png", components=components,
                            components_prior=prior if components is not None and components.mode == "near" else None)
    for _ in seg(iter(frames[:8])):                     # warm-up: allocation, graph captures of every ring slot
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = sum(1 for _ in seg(iter(frames)))
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {"card": _card(), "ms": time_ops(a.calls, dev)}
    h, w = 480, 854
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    net.to(dev)
    g = torch.Generator().manual_seed(0)
    base = (torch.rand(h, w, 3, generator=g) * 255).to(torch.uint8)
    frames = [torch.roll(base, shifts=2 * i, dims=1)[None].contiguous().pin_memory() for i in range(a.frames)]
    prior = _pattern("blobs", 1, h, w, dev)
    variants = {"plain": None, "largest": ops.Components("largest"), "near": ops.Components("near")}
    fps = {k: [] for k in variants}
    for _ in range(a.rounds):                           # alternated, so drift affects every variant alike
        for name, comp in variants.items():
            fps[name].append(round(time_loop(net, frames, comp, prior), 1))
    res.update(frames=a.frames, loop_fps=fps,
               loop_fps_median={k: sorted(v)[len(v) // 2] for k, v in fps.items()})
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Timing of segmentation at the stored size (DESIGN.md §18): the fp32 resize of fused logits (csrc/resize.cu,
ops.resize_f32) and what ``SequenceSegmenter(output_res="stored")`` costs against ``"network"``.

    python scripts/time_output_res.py [--out results] [--iters 400]

Measures, with CUDA events:
  1. resize_f32 device time per frame at batch 1 and 12, for 240x427 -> 480x854 and 360x640 -> 480x854, and GB/s of
     the bytes it moves (source read, the fp32 intermediate written and read, result written);
  2. inference.SequenceSegmenter frames/s on 480x854 bgr8 frames at input_res (240, 427), output bytescale:
     output_res "network" against "stored", without and with score=True, alternated over the rounds.
Writes <out>/time_output_res.json; the GPU's name, power limit and SM clocks (current and maximum) go with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def event_ms(fn, iters, warmup=20):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def resize_bytes(n, src, dst):
    (h, w), (oh, ow) = src, dst
    moved = 4 * n * (h * w + oh * ow)
    if h != oh and w != ow:
        moved += 2 * 4 * n * h * ow                   # intermediate: written, then read (upper bound: every source row)
    return moved


def time_kernels(iters):
    from osvos_pytorch_b200 import ops
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    dst = (480, 854)
    for src in ((240, 427), (360, 640)):
        for n in (1, 12):
            x = 10 * torch.randn((n, 1) + src, generator=g, device="cuda")
            out = torch.empty((n, 1) + dst, dtype=torch.float32, device="cuda")
            ms = event_ms(lambda: ops.resize_f32(x, dst, out=out), iters)
            nb = resize_bytes(n, src, dst)
            rows.append(dict(src=src, dst=dst, batch=n, us_per_call=1e3 * ms, us_per_frame=1e3 * ms / n, bytes=nb,
                             gb_per_s=nb / ms / 1e6))
            print(f"resize_f32 {src}->{dst} batch {n:2d}: {1e3 * ms:8.2f} us/call {1e3 * ms / n:8.2f} us/frame "
                  f"{nb / ms / 1e6:7.1f} GB/s", flush=True)
    return rows


def time_segmenter(frames_n, rounds, input_res=(240, 427)):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    net.cuda().eval()
    g = torch.Generator().manual_seed(0)
    frames = [torch.randint(0, 256, (1, 480, 854, 3), generator=g, dtype=torch.uint8).pin_memory()
              for _ in range(frames_n)]
    gts = [(255 * (torch.rand((1, 480, 854), generator=g) > 0.7)).to(torch.uint8).pin_memory() for _ in range(frames_n)]
    configs = [(o, s) for s in (False, True) for o in ("network", "stored")]
    segs = {c: SequenceSegmenter(net, output="bytescale", frames="bgr8", input_res=input_res, output_res=c[0],
                                 score=c[1]) for c in configs}

    def feed(score, n=frames_n):
        return iter(list(zip(frames[:n], gts[:n])) if score else frames[:n])
    for c in configs:                                    # warm-up: allocation and graph capture of every slot
        for _ in segs[c](feed(c[1], 8)):
            pass
    out = {f"{o} score={s}": [] for o, s in configs}
    for _ in range(rounds):
        for c in configs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in segs[c](feed(c[1])):
                pass
            torch.cuda.synchronize()
            out[f"{c[0]} score={c[1]}"].append(frames_n / (time.perf_counter() - t0))
    for k, v in out.items():
        print(f"SequenceSegmenter 480x854 bgr8 input_res={input_res} output_res={k}: "
              + " / ".join(f"{f:.1f}" for f in v) + " frames/s", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_output_res.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock):", gpu, flush=True)
    res = {"gpu": gpu, "resize_f32": time_kernels(a.iters), "segmenter_frames_per_s": time_segmenter(a.frames, a.rounds)}
    res["gpu_after"] = gpu_info()
    print("GPU after:", res["gpu_after"], flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_output_res.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Timing of the device PNG encoder (DESIGN.md §21): ops.encode_png (csrc/png.cu) against Pillow on this host, and what
writing the result files costs SequenceSegmenter with host encoding (train_online.py --encode host) and with
encode="png" (--encode device).

    python scripts/time_png.py [--out results] [--iters 200] [--frames 200] [--rounds 3]

Measures:
  1. encode_png device time per frame from CUDA events, at batch 1 and 12, for 480x854 bytescale and mask maps, with
     GB/s of raw map bytes;
  2. Pillow's Image.fromarray(map, "L").save(PNG) on this host, one thread and a pool of os.cpu_count() threads;
  3. file sizes against Pillow's;
  4. SequenceSegmenter (bgr8 frames, output bytescale) frames/s at 480x854 and at input_res (240, 427) with
     output_res "stored": without writing, writing Pillow files, writing encode="png" files, alternated over the rounds.
Writes <out>/time_png.json; the GPU's name, power limit and SM clocks and the CPU count go with the numbers.  Files are
written to a temporary directory.
"""
import argparse
import io
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from time_output_res import event_ms, gpu_info  # noqa: E402


def maps(kind, n, h=480, w=854):
    import png_cases
    return np.stack([png_cases.content(kind, h, w, seed=i) for i in range(n)])


def pillow_bytes(a):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(a, "L").save(b, "PNG")
    return b.getvalue()


def time_kernels(iters):
    from osvos_pytorch_b200 import ops
    rows = []
    for kind in ("bytescale", "mask"):
        host = maps(kind, 12)
        for n in (1, 12):
            x = torch.from_numpy(host[:n]).cuda()
            out, lengths = ops.encode_png(x)
            ms = event_ms(lambda: ops.encode_png(x, out=out, lengths=lengths), iters)
            nb = x.numel()
            sizes = lengths.cpu().tolist()
            pil = [len(pillow_bytes(m)) for m in host[:n]]
            rows.append(dict(kind=kind, batch=n, us_per_call=1e3 * ms, us_per_frame=1e3 * ms / n,
                             gb_per_s=nb / ms / 1e6, bytes=sizes, pillow_bytes=pil,
                             size_ratio=sum(sizes) / sum(pil)))
            print(f"encode_png 480x854 {kind:9s} batch {n:2d}: {1e3 * ms:8.1f} us/call {1e3 * ms / n:7.1f} us/frame "
                  f"{nb / ms / 1e6:6.1f} GB/s  size {sum(sizes) / n:9.0f} B/frame = {sum(sizes) / sum(pil):.3f}x Pillow",
                  flush=True)
    return rows


def time_pillow(k=48):
    rows = []
    threads = os.cpu_count() or 1
    for kind in ("bytescale", "mask"):
        host = list(maps(kind, 12)) * (k // 12)
        t0 = time.perf_counter()
        for m in host:
            pillow_bytes(m)
        one = len(host) / (time.perf_counter() - t0)
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(pillow_bytes, host[:threads]))
            t0 = time.perf_counter()
            list(ex.map(pillow_bytes, host))
            pool = len(host) / (time.perf_counter() - t0)
        rows.append(dict(kind=kind, frames_per_s_1_thread=one, threads=threads, frames_per_s_pool=pool))
        print(f"Pillow save 480x854 {kind:9s}: {one:7.1f} frames/s on 1 thread, {pool:7.1f} on {threads} threads",
              flush=True)
    return rows


def time_segmenter(frames_n, rounds, input_res):
    import networks.vgg_osvos as vo
    from PIL import Image
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    net.cuda().eval()
    g = torch.Generator().manual_seed(0)
    frames = [torch.randint(0, 256, (1, 480, 854, 3), generator=g, dtype=torch.uint8).pin_memory()
              for _ in range(frames_n)]
    opts = dict(output="bytescale", frames="bgr8")
    if input_res is not None:
        opts.update(input_res=input_res, output_res="stored")
    segs = {"no writing": SequenceSegmenter(net, **opts), "host encode + write": SequenceSegmenter(net, **opts),
            "encode=png + write": SequenceSegmenter(net, encode="png", **opts)}
    out_dir = tempfile.mkdtemp(prefix="time_png_")

    def run(name, n=frames_n):
        i = 0
        for r in segs[name](iter(frames[:n])):
            if name == "host encode + write":
                arr = r.numpy()
                for j in range(arr.shape[0]):
                    Image.fromarray(arr[j, 0], mode="L").save(os.path.join(out_dir, f"{i:05d}_{j}.png"))
            elif name == "encode=png + write":
                for j, f in enumerate(r):
                    with open(os.path.join(out_dir, f"{i:05d}_{j}.png"), "wb") as fh:
                        fh.write(f)
            i += 1
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
    tag = "480x854" if input_res is None else f"input_res={input_res} -> stored 480x854"
    for k, v in res.items():
        print(f"SequenceSegmenter {tag} bytescale, {k}: " + " / ".join(f"{f:.1f}" for f in v) + " frames/s", flush=True)
    return {"config": tag, "d2h_bytes_per_frame": {k: s.d2h_bytes_per_frame for k, s in segs.items()},
            "frames_per_s": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_png.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock):", gpu, "| os.cpu_count():", os.cpu_count(), flush=True)
    res = {"gpu": gpu, "cpu_count": os.cpu_count(), "encode_png": time_kernels(a.iters), "pillow": time_pillow(),
           "segmenter": [time_segmenter(a.frames, a.rounds, None), time_segmenter(a.frames, a.rounds, (240, 427))]}
    res["gpu_after"] = gpu_info()
    print("GPU after:", res["gpu_after"], flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_png.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

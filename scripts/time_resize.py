"""Timing of the frame resize (csrc/resize.cu, ops.resize_u8) and of what running at a reduced resolution buys.

    python scripts/time_resize.py [--out results] [--iters 400]

Measures, with CUDA events:
  1. resize device time per frame at batch 1 and 12, for 480x854 -> 240x427 and 1080x1920 -> 480x854, image (bilinear,
     3 channels) and mask (nearest), and GB/s of the bytes the resize must move (source read, result written, and the
     bilinear intermediate written and read once);
  2. graphed online fine-tuning (training.online_finetune, batch 1, nAveGrad 5) fwd+bwd/s at 240x427, 360x640 and
     480x854 (the two smaller sizes are what --input-res gives a 480x854 sequence);
  3. inference.SequenceSegmenter frames/s on 480x854 bgr8 frames (output bytescale) without input_res and with
     input_res (240, 427) and (360, 640), alternated.
Writes <out>/time_resize.json; the GPU's name, power limit and SM clock limit go with the numbers.
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def resize_bytes(n, src, dst, c, mode):
    (h, w), (oh, ow) = src, dst
    moved = n * c * (h * w + oh * ow)
    if mode == "bilinear" and h != oh and w != ow:
        moved += 2 * n * c * h * ow                   # intermediate: written, then read (upper bound: every source row)
    return moved


def time_kernels(iters):
    from osvos_pytorch_b200 import ops
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for src, dst in (((480, 854), (240, 427)), ((1080, 1920), (480, 854))):
        for n in (1, 12):
            for mode, c in (("bilinear", 3), ("nearest", 1)):
                shape = (n,) + src + ((3,) if c == 3 else ())
                x = torch.randint(0, 256, shape, generator=g, device="cuda", dtype=torch.uint8)
                out = torch.empty((n,) + dst + shape[3:], dtype=torch.uint8, device="cuda")
                ms = event_ms(lambda: ops.resize_u8(x, dst, mode, out=out), iters)
                nb = resize_bytes(n, src, dst, c, mode)
                rows.append(dict(src=src, dst=dst, batch=n, mode=mode, channels=c, us_per_call=1e3 * ms,
                                 us_per_frame=1e3 * ms / n, bytes=nb, gb_per_s=nb / ms / 1e6))
                print(f"resize {mode:8s} c={c} {src}->{dst} batch {n:2d}: {1e3 * ms / n:8.2f} us/frame "
                      f"{nb / ms / 1e6:7.1f} GB/s", flush=True)
    return rows


def time_online(sizes, steps, warmup):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200 import training
    rows = []
    for h, w in sizes:
        net = vo.OSVOS(pretrained=0, verbose=False)
        vo.he_init_(net, seed=0)
        net.cuda()
        sample = training.synthetic_batch(1, h, w, 1234, torch.device("cuda"))
        ev = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]

        def sample_fn(it):
            if it == warmup:
                ev[0].record()
            return sample
        training.online_finetune(net, sample_fn, warmup + steps, 5, 1e-10, 0.0002, log_every=0)
        ev[1].record()
        ev[1].synchronize()
        ms = ev[0].elapsed_time(ev[1]) / steps
        rows.append(dict(h=h, w=w, ms_per_fwd_bwd=ms, fwd_bwd_per_s=1e3 / ms))
        print(f"online fine-tune {h}x{w}: {1e3 / ms:7.1f} fwd+bwd/s ({ms:.3f} ms)", flush=True)
        del net
        torch.cuda.empty_cache()
    return rows


def time_segmenter(frames_n, rounds):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    net.cuda().eval()
    g = torch.Generator().manual_seed(0)
    frames = [torch.randint(0, 256, (1, 480, 854, 3), generator=g, dtype=torch.uint8).pin_memory()
              for _ in range(frames_n)]
    res_list = [None, (240, 427), (360, 640)]
    segs = {r: SequenceSegmenter(net, output="bytescale", frames="bgr8", input_res=r) for r in res_list}
    for r in res_list:                                   # warm-up: allocation and graph capture of every slot
        for _ in segs[r](iter(frames[:8])):
            pass
    out = {str(r): [] for r in res_list}
    for _ in range(rounds):
        for r in res_list:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in segs[r](iter(frames)):
                pass
            torch.cuda.synchronize()
            out[str(r)].append(frames_n / (time.perf_counter() - t0))
    for r in res_list:
        print(f"SequenceSegmenter 480x854 bgr8 input_res={r}: " + " / ".join(f"{v:.1f}" for v in out[str(r)])
              + " frames/s", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--online-steps", type=int, default=500)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_resize.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU:", gpu, flush=True)
    res = {"gpu": gpu, "resize": time_kernels(a.iters),
           "online": time_online([(240, 427), (360, 640), (480, 854)], a.online_steps, 50),
           "segmenter_frames_per_s": time_segmenter(a.frames, a.rounds)}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_resize.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Timing of the per-object upsample fused with the merge (ops.upsample_merge_objects, DESIGN.md §27).

    python scripts/time_upsample_merge.py [--out results] [--frames 160] [--rounds 3]

Measures:
  1. Device time of ops.upsample_merge_objects against the composition it replaces (K x ops.resize_f32 into
     preallocated stored-size buffers, then ops.merge_objects): 50 calls captured in one CUDA graph and replayed (CUDA
     events), as DESIGN.md §24 times the merge.  N = 1 and 12, K = 1 .. 4, 240x427 and 360x640 -> 480x854.  GB/s are
     over the algorithmic bytes, K*N*h*w*4 read and N*480*854 written; at N = 12 that working set (up to 64 MB at
     360x640, K = 4) is about the size of the 50 MB L2, so repeated calls partly hit in L2.
  2. SequenceSegmenter frames/s, nets = K He-initialised networks, output "labels", 480x854 bgr8 frames,
     input_res=(240, 427), output_res="stored", with and without score=True: the fused op against the composition
     (monkeypatched in for ops.upsample_merge_objects), and the full-resolution K-net segmenter for the ratio; the
     variants alternate over the rounds.
Writes <out>/time_upsample_merge.json; the GPU's name, power limit and SM clocks go with the numbers.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from time_objects import graph_ms  # noqa: E402
from time_output_res import gpu_info  # noqa: E402

H0, W0 = 480, 854
HBM_BYTES_PER_S = 3.35e12


def composition(bufs):
    """ops.upsample_merge_objects restated as K resize_f32 calls into stored-size buffers and one merge_objects."""
    from osvos_pytorch_b200 import ops

    def fn(maps, size, out=None):
        ups = []
        for j, m in enumerate(maps):
            key = (j, tuple(m.shape[:-2]) + tuple(size))
            if key not in bufs:
                bufs[key] = torch.empty(key[1], dtype=torch.float32, device=m.device)
            ups.append(ops.resize_f32(m, size, out=bufs[key]))
        return ops.merge_objects(ups, out=out)
    return fn


def time_kernels():
    from osvos_pytorch_b200 import ops
    rows = []
    for src in ((240, 427), (360, 640)):
        for n in (1, 12):
            for k in (1, 2, 3, 4):
                rng = np.random.default_rng(n * 10 + k)
                maps = [torch.from_numpy(rng.normal(0, 4, (n, 1) + src).astype(np.float32)).cuda() for _ in range(k)]
                out = torch.empty((n, H0, W0), dtype=torch.uint8, device="cuda")
                ref = torch.empty_like(out)
                composed = composition({})
                ops.upsample_merge_objects(maps, (H0, W0), out=out)
                composed(maps, (H0, W0), out=ref)
                same = torch.equal(out, ref)
                ms_fused = graph_ms(lambda: ops.upsample_merge_objects(maps, (H0, W0), out=out))
                ms_comp = graph_ms(lambda: composed(maps, (H0, W0), out=ref))
                moved = 4 * k * n * src[0] * src[1] + n * H0 * W0
                row = dict(src=list(src), batch=n, objects=k, fused_us=1e3 * ms_fused, composition_us=1e3 * ms_comp,
                           speedup=ms_comp / ms_fused, bytes=moved, fused_gb_per_s=moved / (ms_fused * 1e-3) / 1e9,
                           fused_share_of_hbm=moved / (ms_fused * 1e-3) / HBM_BYTES_PER_S, bit_identical=same)
                rows.append(row)
                print(f"{src[0]}x{src[1]} -> {H0}x{W0} N {n:2d} K {k}: fused {row['fused_us']:7.1f} us "
                      f"({row['fused_gb_per_s']:6.0f} GB/s, {100 * row['fused_share_of_hbm']:4.1f} % of 3.35 TB/s) | "
                      f"composition {row['composition_us']:7.1f} us | {row['speedup']:4.2f}x | identical {same}",
                      flush=True)
    return rows


def time_segmenter(frames_n, rounds):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter

    def he(seed):
        net = vo.OSVOS(pretrained=0, verbose=False)
        vo.he_init_(net, seed=seed)
        return net.cuda().eval()
    nets = [he(s) for s in range(4)]
    rng = np.random.default_rng(1)
    frames = [torch.from_numpy(rng.integers(0, 256, (1, H0, W0, 3), dtype=np.uint8)).pin_memory() for _ in range(8)]
    gts = [torch.from_numpy(rng.integers(0, 5, (1, H0, W0)).astype(np.uint8)).pin_memory() for _ in range(8)]
    fused_op, composed = ops.upsample_merge_objects, composition({})
    variants = {}
    for k in (2, 4):
        for score in (False, True):
            tag = f"K={k}{' score' if score else ''}"
            variants[f"{tag} 240x427 fused"] = (k, score, (240, 427), fused_op)
            variants[f"{tag} 240x427 composition"] = (k, score, (240, 427), composed)
            variants[f"{tag} 480x854"] = (k, score, None, fused_op)

    def run(name, n):
        k, score, res, op = variants[name]
        ops.upsample_merge_objects = op
        try:
            seg = SequenceSegmenter(nets=nets[:k], output="labels", frames="bgr8", score=score, input_res=res,
                                    output_res="stored")
            items = [(frames[i % 8], gts[i % 8]) if score else frames[i % 8] for i in range(n)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in seg(iter(items)):
                pass
            if score:
                seg.frame_counts()
            torch.cuda.synchronize()
            return n / (time.perf_counter() - t0)
        finally:
            ops.upsample_merge_objects = fused_op
    for name in variants:
        run(name, 16)
    res = {name: [] for name in variants}
    for _ in range(rounds):
        for name in variants:
            res[name].append(run(name, frames_n))
    summary = {}
    for name, v in res.items():
        k, score, r, _ = variants[name]
        full = float(np.mean(res[f"K={k}{' score' if score else ''} 480x854"]))
        summary[name] = dict(frames_per_s=v, over_full_resolution=float(np.mean(v)) / full)
        print(f"SequenceSegmenter 480x854 frames, {name}: " + " / ".join(f"{f:.1f}" for f in v)
              + f" frames/s ({summary[name]['over_full_resolution']:.2f}x the full-resolution K-net segmenter)",
              flush=True)
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--frames", type=int, default=160)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_upsample_merge.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock):", gpu, flush=True)
    res = {"gpu": gpu, "kernels": time_kernels(), "segmenter": time_segmenter(a.frames, a.rounds)}
    res["gpu_after"] = gpu_info()
    print("GPU after:", res["gpu_after"], flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_upsample_merge.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Timing of the DAVIS-2017 device stages (DESIGN.md §24) at 480x854.

    python scripts/time_objects.py [--out results] [--iters 200] [--frames 120] [--rounds 2]

Kernel times are device times: 50 calls captured in one CUDA graph and replayed (CUDA events), as DESIGN.md §14
times ops.davis_measures; merge + measures is also given as issued one by one from Python.  Measures:
  1. ops.merge_objects of K = 1, 2, 4 fused maps at batch N = 1 and 12, with the bytes it moves (K fp32 reads and one
     uint8 write per pixel) over its time, against the H100 SXM's 3.35 TB/s of HBM3;
  2. ops.davis_measures_objects at K = 1, 2, 3, 4, N = 1 and 12, beside ops.davis_measures (one object) of the same
     frames, and merge + per-object measures at K = 3, N = 1;
  3. palette encode (ops.encode_png with a palette) and palette decode (png.pack + ops.decode_png of those files;
     the device time only) of K-object label maps;
  4. SequenceSegmenter frames/s (bgr8 frames, no writing): the single-object path (output "mask") against
     nets = K He-initialised networks with output "labels", K = 1, 2, 4, alternated over the rounds.
Writes <out>/time_objects.json; the GPU's name, power limit and SM clocks go with the numbers.
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

from time_output_res import event_ms, gpu_info  # noqa: E402

H, W = 480, 854
HBM_BYTES_PER_S = 3.35e12


def graph_ms(fn, replays=20, per_graph=50):
    """Device time of one fn() call: per_graph calls captured in one CUDA graph, replayed `replays` times."""
    fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        for _ in range(per_graph):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(replays):
        graph.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / (replays * per_graph)


def scenes(n, k, seed=0):
    """Fused-logit-like maps [K,N,1,H,W] of K elliptic objects, and annotations [N,H,W] with a void band."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    maps = np.empty((k, n, 1, H, W), np.float32)
    gt = np.zeros((n, H, W), np.uint8)
    for i in range(n):
        for j in range(k):
            cy, cx = rng.uniform(0.2, 0.8) * H, rng.uniform(0.2, 0.8) * W
            e = 1.0 - ((yy - cy) / (0.2 * H)) ** 2 - ((xx - cx) / (0.15 * W)) ** 2
            maps[j, i, 0] = 4 * e
            gt[i][e + rng.normal(0, 0.05) > 0.05] = j + 1
        gt[i, :, W // 2:W // 2 + 4] = 255
    return maps, gt


def time_kernels(iters):
    from osvos_pytorch_b200 import ops, png
    rows = []
    for n in (1, 12):
        for k in (1, 2, 3, 4):
            maps_h, gt_h = scenes(n, k, seed=n * 10 + k)
            maps = torch.from_numpy(maps_h).cuda()
            parts = list(maps.unbind(0))
            gt = torch.from_numpy(gt_h).cuda()
            labels = ops.merge_objects(parts)
            counts = ops.davis_measures_objects(labels, gt, k)
            ms_merge = graph_ms(lambda: ops.merge_objects(parts, out=labels))
            ms_meas = graph_ms(lambda: ops.davis_measures_objects(labels, gt, k, out=counts))

            def both():
                ops.merge_objects(parts, out=labels)
                ops.davis_measures_objects(labels, gt, k, out=counts)
            ms_both = graph_ms(both)
            ms_both_py = event_ms(both, iters)
            one = torch.where(labels == 1, 1.0, -1.0).to(torch.float32)
            c1 = ops.davis_measures(one, gt)
            ms_2016 = graph_ms(lambda: ops.davis_measures(one, gt, out=c1))
            pal = bytes(range(3 * max(2, k + 1)))
            files, lengths = ops.encode_png(labels, palette=pal)
            ms_enc = graph_ms(lambda: ops.encode_png(labels, out=files, lengths=lengths, palette=pal), 5, 10)
            datas = [files[i, :int(lengths[i])].cpu().numpy().tobytes() for i in range(n)]
            blob = png.pack([png.parse(d, palette="index") for d in datas])
            dev_blob = torch.from_numpy(blob).cuda()
            nseg = png.segment_count(blob)
            dec, status = ops.decode_png(dev_blob, n, H, W, nseg)
            ok = int(status.abs().sum()) == 0 and torch.equal(dec, labels)
            ms_dec = graph_ms(lambda: ops.decode_png(dev_blob, n, H, W, nseg, out=dec, status=status), 5, 10)
            moved = n * H * W * (4 * k + 1)
            row = dict(batch=n, objects=k, merge_us=1e3 * ms_merge, merge_bytes=moved,
                       merge_share_of_hbm=moved / (ms_merge * 1e-3) / HBM_BYTES_PER_S,
                       measures_objects_us=1e3 * ms_meas, merge_plus_measures_us=1e3 * ms_both,
                       merge_plus_measures_us_from_python=1e3 * ms_both_py,
                       davis_measures_one_object_us=1e3 * ms_2016, palette_encode_us_per_frame=1e3 * ms_enc / n,
                       palette_decode_us_per_frame=1e3 * ms_dec / n, palette_bytes_per_frame=sum(map(len, datas)) / n,
                       round_trip_ok=ok)
            rows.append(row)
            print(f"N {n:2d} K {k}: merge {row['merge_us']:7.1f} us ({moved / (ms_merge * 1e-3) / 1e9:6.0f} GB/s, "
                  f"{100 * row['merge_share_of_hbm']:4.1f} % of HBM) | measures_objects {row['measures_objects_us']:7.1f}"
                  f" us (davis_measures {row['davis_measures_one_object_us']:6.1f}) | merge + measures "
                  f"{row['merge_plus_measures_us']:7.1f} us ({row['merge_plus_measures_us_from_python']:6.1f} issued "
                  f"from Python) | palette encode {row['palette_encode_us_per_frame']:6.1f}"
                  f" decode {row['palette_decode_us_per_frame']:7.1f} us/frame | round trip {ok}", flush=True)
    return rows


def time_segmenter(frames_n, rounds):
    import networks.vgg_osvos as vo
    from osvos_pytorch_b200.inference import SequenceSegmenter

    def he(seed):
        net = vo.OSVOS(pretrained=0, verbose=False)
        vo.he_init_(net, seed=seed)
        return net.cuda().eval()
    nets = [he(s) for s in range(4)]
    rng = np.random.default_rng(1)
    frames = [torch.from_numpy(rng.integers(0, 256, (1, H, W, 3), dtype=np.uint8)).pin_memory() for _ in range(8)]
    frames = [frames[i % 8] for i in range(frames_n)]
    segs = {"single (mask)": SequenceSegmenter(nets[0], output="mask", frames="bgr8")}
    for k in (1, 2, 4):
        segs[f"labels K={k}"] = SequenceSegmenter(nets=nets[:k], output="labels", frames="bgr8")

    def run(name, n=frames_n):
        for _ in segs[name](iter(frames[:n])):
            pass
    for name in segs:
        run(name, 8)
    res = {name: [] for name in segs}
    for _ in range(rounds):
        for name in segs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(name)
            torch.cuda.synchronize()
            res[name].append(frames_n / (time.perf_counter() - t0))
    single = float(np.mean(res["single (mask)"]))
    summary = {}
    for name, v in res.items():
        k = 1 if name.startswith("single") else int(name.split("=")[1])
        summary[name] = dict(frames_per_s=v, share_of_single_over_k=float(np.mean(v)) / (single / k))
        print(f"SequenceSegmenter 480x854, {name}: " + " / ".join(f"{f:.1f}" for f in v)
              + f" frames/s ({100 * summary[name]['share_of_single_over_k']:.1f} % of single / K)", flush=True)
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_objects.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock):", gpu, flush=True)
    res = {"gpu": gpu, "kernels": time_kernels(a.iters), "segmenter": time_segmenter(a.frames, a.rounds)}
    res["gpu_after"] = gpu_info()
    print("GPU after:", res["gpu_after"], flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_objects.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Timing of the results overlays (DESIGN.md §25): ops.overlay_labels and visualize.render_results at 480x854.

    python scripts/time_visualize.py [--out results] [--frames 80] [--rounds 3]

Measures:
  1. ops.overlay_labels device time at N = 1 and 12, K = 1 .. 4 objects: 50 calls captured in one CUDA graph and
     replayed (CUDA events), as scripts/time_objects.py times the merge, with GB/s over its algorithmic bytes (3 frame
     bytes and 1 label byte read, 3 bytes written per pixel) against the H100 SXM's 3.35 TB/s of HBM3; ops.overlay_mask
     at N = 12 beside it (4 logit bytes instead of the label byte).
  2. visualize.render_results frames/s on a synthetic 480p DAVIS-2016 tree (one sequence of --frames frames, mask
     results) and a DAVIS-2017 tree (3 objects, palette results), with --decode device and host, writing the JPEG
     files and with the MJPEG video too, against a host pipeline on the same host and one thread: cv2.imread of frame
     and result, the overlay in numpy, cv2.imencode and the file write.  Alternated over --rounds.
Writes <out>/time_visualize.json; the GPU's name, power limit and SM clocks and the CPU count go with the numbers.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from time_objects import graph_ms  # noqa: E402
from time_output_res import gpu_info  # noqa: E402

H, W = 480, 854
HBM_BYTES_PER_S = 3.35e12


def scene(n, k, seed):
    """Frames [N,H,W,3] (smooth content with texture) and label maps [N,H,W] of k elliptic objects."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    frames = np.empty((n, H, W, 3), np.uint8)
    labels = np.zeros((n, H, W), np.uint8)
    for i in range(n):
        base = np.stack([(xx // 3 + 7 * i) % 256, (yy // 2) % 256, ((xx + yy) // 4) % 256], -1)
        frames[i] = np.clip(base + rng.integers(-12, 13, (H, W, 3)), 0, 255)
        for j in range(1, k + 1):
            cy, cx = rng.uniform(0.2, 0.8) * H, rng.uniform(0.2, 0.8) * W
            labels[i][((yy - cy) / (0.2 * H)) ** 2 + ((xx - cx) / (0.15 * W)) ** 2 <= 1] = j
    return frames, labels


def time_kernel():
    from osvos_pytorch_b200 import ops
    rows = []
    for n in (1, 12):
        for k in (1, 2, 3, 4):
            f, lab = scene(n, k, seed=10 * n + k)
            x, y = torch.from_numpy(f).cuda(), torch.from_numpy(lab).cuda()
            out = ops.overlay_labels(x, y)
            ms = graph_ms(lambda: ops.overlay_labels(x, y, out=out))
            moved = n * H * W * 7
            row = dict(batch=n, objects=k, us=1e3 * ms, bytes=moved, gb_per_s=moved / (ms * 1e-3) / 1e9,
                       share_of_hbm=moved / (ms * 1e-3) / HBM_BYTES_PER_S)
            if n == 12 and k == 1:
                logits = torch.where(y > 0, 1.0, -1.0).to(torch.float32)
                ms_mask = graph_ms(lambda: ops.overlay_mask(x, logits, out=out))
                row.update(overlay_mask_us=1e3 * ms_mask,
                           overlay_mask_gb_per_s=n * H * W * 10 / (ms_mask * 1e-3) / 1e9)
            rows.append(row)
            print(f"overlay_labels N {n:2d} K {k}: {row['us']:7.1f} us, {row['gb_per_s']:6.0f} GB/s "
                  f"({100 * row['share_of_hbm']:4.1f} % of HBM)"
                  + (f" | overlay_mask {row['overlay_mask_us']:.1f} us ({row['overlay_mask_gb_per_s']:.0f} GB/s)"
                     if "overlay_mask_us" in row else ""), flush=True)
    return rows


def make_tree(root, davis, frames_n):
    """A synthetic DAVIS tree of one 480x854 sequence 'seq' and its results folder root/res."""
    import cv2
    from PIL import Image

    from osvos_pytorch_b200 import png
    k = 1 if davis == "2016" else 3
    f, lab = scene(frames_n, k, seed=5)
    img_dir = os.path.join(root, "JPEGImages", "480p", "seq")
    res_dir = os.path.join(root, "res", "seq")
    os.makedirs(img_dir)
    os.makedirs(res_dir)
    for i in range(frames_n):
        cv2.imwrite(os.path.join(img_dir, f"{i:05d}.jpg"), f[i])
        if davis == "2016":
            cv2.imwrite(os.path.join(res_dir, f"{i:05d}.png"), lab[i] * 255)
        else:
            im = Image.fromarray(lab[i], "P")
            im.putpalette(png.davis_palette(k + 1))
            im.save(os.path.join(res_dir, f"{i:05d}.png"))
    with open(os.path.join(root, "val_seqs.txt"), "w") as fh:
        fh.write("seq\n")
    os.makedirs(os.path.join(root, "ImageSets", "2017"))
    with open(os.path.join(root, "ImageSets", "2017", "val.txt"), "w") as fh:
        fh.write("seq\n")


def host_pipeline(root, davis, out_dir, quality=95):
    """cv2.imread + numpy overlay + cv2.imencode + write, one frame at a time."""
    import cv2
    from PIL import Image

    from osvos_pytorch_b200 import png
    os.makedirs(out_dir, exist_ok=True)
    res_dir = os.path.join(root, "res", "seq")
    table = np.zeros((256, 3), np.int32)
    if davis == "2016":
        table[1] = (0, 0, 255)
    else:
        table[:] = np.frombuffer(png.davis_palette(), np.uint8).reshape(256, 3)[:, ::-1]
    for name in sorted(os.listdir(res_dir)):
        frame = cv2.imread(os.path.join(root, "JPEGImages", "480p", "seq", name[:-4] + ".jpg")).astype(np.int32)
        if davis == "2016":
            lab = (cv2.imread(os.path.join(res_dir, name), 0) >= 128).astype(np.int32)
        else:
            lab = np.array(Image.open(os.path.join(res_dir, name))).astype(np.int32)
        p = np.pad(lab, 1, constant_values=-1)
        edge = (lab != 0) & ~((p[:-2, 1:-1] == lab) & (p[2:, 1:-1] == lab) & (p[1:-1, :-2] == lab)
                              & (p[1:-1, 2:] == lab))
        img = np.where((lab != 0)[..., None], (frame + table[lab] + 1) >> 1, frame)
        img[edge] = 0
        ok, buf = cv2.imencode(".jpg", img.astype(np.uint8), [cv2.IMWRITE_JPEG_QUALITY, quality])
        with open(os.path.join(out_dir, name[:-4] + ".jpg"), "wb") as fh:
            fh.write(buf.tobytes())


def time_tool(frames_n, rounds):
    from osvos_pytorch_b200 import visualize
    summary = {}
    for davis in ("2016", "2017"):
        root = tempfile.mkdtemp(prefix=f"time_visualize_{davis}_")
        try:
            make_tree(root, davis, frames_n)
            res = os.path.join(root, "res")

            def tool(decode, video):
                def run():
                    visualize.render_results(res, root, davis=davis, decode=decode, video=video,
                                             out_dir=os.path.join(root, "out"))
                return run
            ways = {"render_results device decode": tool("device", False),
                    "render_results host decode": tool("host", False),
                    "render_results device decode + video": tool("device", True),
                    "cv2 host pipeline": lambda: host_pipeline(root, davis, os.path.join(root, "host"))}
            for fn in ways.values():
                fn()                                        # warm-up: module loads, first launches
            rates = {name: [] for name in ways}
            for _ in range(rounds):
                for name, fn in ways.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    rates[name].append(frames_n / (time.perf_counter() - t0))
            host = float(np.mean(rates["cv2 host pipeline"]))
            for name, v in rates.items():
                summary[f"{davis} {name}"] = dict(frames_per_s=v, speedup_over_host=float(np.mean(v)) / host)
                print(f"DAVIS-{davis} 480x854, {frames_n} frames, {name}: " + " / ".join(f"{x:.1f}" for x in v)
                      + f" frames/s ({float(np.mean(v)) / host:.1f}x the host pipeline)", flush=True)
            same = all(open(os.path.join(root, "out", "seq_overlay", f), "rb").read()
                       == open(os.path.join(root, "host", f), "rb").read()
                       for f in os.listdir(os.path.join(root, "host")))
            summary[f"{davis} files equal the host pipeline's"] = same
            print(f"DAVIS-{davis}: render_results files equal the host pipeline's: {same}", flush=True)
        finally:
            shutil.rmtree(root, ignore_errors=True)
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_visualize.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build
    build.build()
    gpu = gpu_info()
    print("GPU (name, power limit, SM clock, max SM clock):", gpu, "| CPUs:", os.cpu_count(), flush=True)
    res = {"gpu": gpu, "cpu_count": os.cpu_count(), "kernel": time_kernel(), "tool": time_tool(a.frames, a.rounds)}
    res["gpu_after"] = gpu_info()
    print("GPU after:", res["gpu_after"], flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "time_visualize.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

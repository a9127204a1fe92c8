"""Data-path timing for real DAVIS-layout data at 480x854 (osvos_pytorch_b200.davis, csrc/frames.cu).

    python scripts/time_data.py [--out results] [--frames 240] [--steps 200]

Builds a synthetic DAVIS tree of 480x854 JPEG frames and PNG masks in a temporary directory and measures:
  1. each ingest kernel: us per frame (CUDA events, batch of 12) and GB/s of the bytes it must move, against the
     H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s;
  2. decoded samples/s of the native loader (DAVIS2016Frames + collate, pinned in the main
     thread as davis.to_device does) at 1, 2 and 4 workers;
  3. the same for a host restatement of the reference's pipeline (cv2 decode, float32 conversion, mean subtraction,
     mask normalisation, flip, warpAffine, ToTensor), at the same worker counts;
  4. train_parent.py frames/s with --loader native on that tree next to --synthetic (second epoch, batch 1);
  5. the device frame store (davis.DeviceFrames): its build time at 1, 2 and 4 workers; the indexed warp of a batch of
     12 against collate + upload + affine_warp_u8 of the same frames; and frames/s of resident parent epochs at batch 12
     (training.parent_epoch fed by DeviceFrames.batches) alternated with training.timed_parent_steps on
     device-resident synthetic batches, with the host time per step that is not spent waiting for the device.
Writes <out>/time_data.json; the GPU's name, power limit and SM clock limit go with the numbers.
"""
import argparse
import json
import os
import random
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
H, W = 480, 854


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_tree(root, frames):
    """Three train sequences and one val sequence of 480x854 frames: smooth colour fields with texture and noise (what
    a JPEG encoder sees in natural video more than white noise), masks 0/255 blobs."""
    import cv2
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    seqs = {"s0": frames // 3, "s1": frames // 3, "s2": frames - 2 * (frames // 3), "v0": 8}
    for seq, n in seqs.items():
        os.makedirs(os.path.join(root, "JPEGImages/480p", seq))
        os.makedirs(os.path.join(root, "Annotations/480p", seq))
        for i in range(n):
            ph = 0.05 * i
            img = np.stack([127 + 100 * np.sin(xx / 37 + ph), 127 + 100 * np.cos(yy / 23 - ph),
                            127 + 100 * np.sin((xx + yy) / 51 + 2 * ph)], -1)
            img = np.clip(img + rng.normal(0, 12, img.shape), 0, 255).astype(np.uint8)
            cv2.imwrite(os.path.join(root, "JPEGImages/480p", seq, "%05d.jpg" % i), img)
            m = (((yy - H / 2) ** 2 / 150 ** 2 + (xx - W / 2 - 3 * i) ** 2 / 220 ** 2) < 1).astype(np.uint8) * 255
            cv2.imwrite(os.path.join(root, "Annotations/480p", seq, "%05d.png" % i), m)
    with open(os.path.join(root, "train_seqs.txt"), "w") as f:
        f.write("s0\ns1\ns2\n")
    with open(os.path.join(root, "val_seqs.txt"), "w") as f:
        f.write("v0\n")


def time_kernels(steps, n=12):
    from osvos_pytorch_b200 import augment, ops
    g = torch.Generator().manual_seed(0)
    img = torch.randint(0, 256, (n, H, W, 3), generator=g, dtype=torch.uint8).cuda()
    gt = ((torch.rand(n, H, W, generator=g) > 0.7).to(torch.uint8) * 255).cuda()
    stats = ops.label_stats_u8(gt)
    f_img = torch.empty(n, 3, H, W, device="cuda")
    f_gt = torch.empty(n, 1, H, W, device="cuda")
    params = augment.draw_params(n, rng=random.Random(0))
    px = H * W
    # bytes each kernel must move per frame (reads + writes; the warp's taps are assumed to hit in cache)
    cases = {
        "image_from_bgr8": (lambda: ops.image_from_bgr8(img, out=f_img), px * (3 + 12)),
        "label_stats_u8": (lambda: ops.label_stats_u8(gt), px * 1),
        "label_from_u8": (lambda: ops.label_from_u8(gt, stats, out=f_gt), px * (1 + 4)),
        "affine_warp_u8": (lambda: augment.affine_warp_u8(img, gt, params, stats), px * (3 + 1 + 12 + 4)),
        "affine_warp_f32_after_ingest": (lambda: (augment.affine_warp(f_img, params, "cubic"),
                                                 augment.affine_warp(f_gt, params, "nearest")), px * (12 + 4) * 2),
    }
    out = {}
    for name, (fn, nbytes) in cases.items():
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / steps / n
        gbs = nbytes / (us * 1e-6) / 1e9
        out[name] = {"us_per_frame": round(us, 2), "bytes_per_frame": nbytes, "GB_per_s": round(gbs, 1),
                     "share_of_hbm_peak": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)}
        print(f"{name:30s} {us:8.2f} us/frame  {gbs:7.1f} GB/s  ({100 * gbs * 1e9 / HBM_BYTES_PER_S:.1f} % of 3.35 TB/s)")
    return out


class ReferenceHostPipeline(torch.utils.data.Dataset):
    """Host restatement of the reference's per-sample work for parent training: make_img_gt_pair (cv2.imread, float32,
    mean subtraction, gt / max), RandomHorizontalFlip, ScaleNRotate (cv2.warpAffine, cubic image, nearest 0/1 mask) and
    ToTensor.  Only for timing; the native path never runs it."""

    def __init__(self, frames):
        self.d = frames

    def __len__(self):
        return len(self.d)

    def __getitem__(self, idx):
        import cv2
        root = self.d.db_root_dir
        img = np.subtract(np.array(cv2.imread(os.path.join(root, self.d.img_list[idx])), dtype=np.float32),
                          np.array(self.d.meanval, dtype=np.float32))
        gt = np.array(cv2.imread(os.path.join(root, self.d.labels[idx]), 0), dtype=np.float32)
        gt = gt / np.max([gt.max(), 1e-8])
        sample = {"image": img, "gt": gt}
        if random.random() < 0.5:
            sample = {k: cv2.flip(v, flipCode=1) for k, v in sample.items()}
        rot, sc = 60 * random.random() - 30, 0.5 * random.random() - 0.25 + 1
        for k, v in sample.items():
            h, w = v.shape[:2]
            m = cv2.getRotationMatrix2D((w / 2, h / 2), rot, sc)
            flag = cv2.INTER_NEAREST if ((v == 0) | (v == 1)).all() else cv2.INTER_CUBIC
            v = cv2.warpAffine(v, m, (w, h), flags=flag)
            sample[k] = torch.from_numpy((v[:, :, None] if v.ndim == 2 else v).transpose((2, 0, 1)))
        return sample


def time_loader(dataset, workers, collate_fn=None, samples=200, post=lambda b: b):
    from torch.utils.data import DataLoader
    loader = DataLoader(dataset, batch_size=1, shuffle=True, num_workers=workers, collate_fn=collate_fn,
                        persistent_workers=True)
    it = iter(loader)
    for _ in range(2 * workers):                     # workers started and their first batches ready
        next(it)
    t0 = time.perf_counter()
    got = 0
    while got < samples:
        try:
            post(next(it))
        except StopIteration:
            it = iter(loader)
            continue
        got += 1
    dt = time.perf_counter() - t0
    del it, loader
    return round(samples / dt, 1)


def parent_fps(extra, env, frames):
    cmd = [sys.executable, os.path.join(ROOT, "train_parent.py"), "--epochs", "2", "--pretrained", "0",
           "--test-interval", "1000", "--snapshot", "1000"] + extra
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"{' '.join(cmd)} failed:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    times = [float(t) for t in re.findall(r"\[Epoch: \d+\].*Execution time: ([\d.]+)", r.stdout)]
    return round(frames / times[-1], 1), times


def time_store(frames, workers, steps, epochs=4, batch=12):
    """Leg 5: build time of the store per worker count, the indexed warp against the streaming path's
    collate + upload + affine_warp_u8, and resident parent epochs against timed_parent_steps on resident batches."""
    from torch.utils.data import DataLoader
    from osvos_pytorch_b200 import augment, davis, parallel, training
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS, he_init_
    dev = torch.device("cuda")
    res = {"build_s": {}}
    for nw in workers:
        store = davis.DeviceFrames(frames, dev, workers=nw)
        res["build_s"][nw] = round(store.build_s, 2)
        print(f"DeviceFrames build, {nw} worker(s): {store.build_s:.2f} s for {len(store)} frames "
              f"({store.nbytes / 1e9:.2f} GB)")
        del store
    torch.cuda.empty_cache()
    store = davis.DeviceFrames(frames, dev, workers=max(workers))
    res["frames"], res["store_GB"] = len(store), round(store.nbytes / 1e9, 3)

    idx = list(range(0, batch * 5, 5))[:batch]
    params = augment.draw_params(batch, rng=random.Random(0))
    items = [frames[i] for i in idx]

    def streamed():
        return davis.to_device(davis.collate(items), dev, augment=params)

    for name, fn in (("indexed_warp", lambda: store.augmented(idx, params)),
                     ("collate_upload_affine_warp_u8", streamed)):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3 / steps
        res[name] = {"device_ms_per_batch": round(e0.elapsed_time(e1) / steps, 3), "wall_ms_per_batch": round(wall, 3)}
        print(f"{name:32s} batch {batch}: {res[name]['device_ms_per_batch']:.3f} ms device, {wall:.3f} ms wall")

    net = he_init_(OSVOS(pretrained=0, verbose=False), seed=0)
    with torch.no_grad():                   # keep the synthetic logits O(10), as bench.py's dp leg does
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    net = net.to(dev)
    opt = training.make_optimizer(net, "parent", lr=1e-10, fused=True)
    bucket = parallel.GradientBucket(parallel.trainable_parameters(net), dev)
    index_loader = DataLoader(range(len(store)), batch_size=batch, shuffle=True, num_workers=0, drop_last=True)
    steps_per_epoch = len(index_loader)
    synth = [training.synthetic_batch(batch, H, W, i, dev) for i in range(2)]
    rng = random.Random(0)
    resident, synthetic, host_ms = [], [], []
    for epoch in range(epochs + 1):         # epoch 0 warms up both paths
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        training.parent_epoch(net, opt, bucket, store.batches(index_loader, rng=rng), epoch, 240, 1)
        host = time.perf_counter() - t0     # enqueue finished; the device may still be working
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        ms = training.timed_parent_steps(net, opt, bucket, lambda i: synth[i % 2], steps_per_epoch, 2 if epoch == 0 else 0)
        if epoch:
            resident.append(round(steps_per_epoch * batch / dt, 1))
            synthetic.append(round(batch * 1e3 / ms, 1))
            host_ms.append(round(host * 1e3 / steps_per_epoch, 2))
    res["parent_batch12"] = {"resident_epoch_frames_per_s": resident, "timed_parent_steps_frames_per_s": synthetic,
                             "resident_host_enqueue_ms_per_step": host_ms, "steps_per_epoch": steps_per_epoch}
    print(f"parent epoch at batch {batch} from the store: {resident} frames/s; timed_parent_steps on resident "
          f"synthetic batches: {synthetic} frames/s; host enqueue per step {host_ms} ms")
    # share of a 240-epoch run over DAVIS-2016's 2,079 train frames, at the measured per-frame rates
    per_frame_build = res["build_s"][max(workers)] / len(store)
    run_s = 240 * 2079 / float(np.median(resident))
    res["build_share_of_240_epochs"] = round(per_frame_build * 2079 / (per_frame_build * 2079 + run_s), 5)
    print(f"store build ({max(workers)} workers) scaled to 2,079 frames: {per_frame_build * 2079:.1f} s, "
          f"{100 * res['build_share_of_240_epochs']:.3f} % of a 240-epoch run")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", os.path.join(ROOT, "results")))
    ap.add_argument("--frames", type=int, default=240, help="training frames in the synthetic tree")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--workers", default="1,2,4")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_data.py measures on the GPU; no CUDA device found")
    from osvos_pytorch_b200 import build, davis
    build.build()
    res = {"gpu": gpu_info(), "cpu_count": os.cpu_count(), "shape": [H, W]}
    print("GPU:", res["gpu"], "| host CPUs:", res["cpu_count"])
    res["kernels"] = time_kernels(a.steps)
    workers = [int(v) for v in a.workers.split(",")]
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        make_tree(root, a.frames)
        print(f"tree of {a.frames} train frames written in {time.perf_counter() - t0:.1f} s")
        frames = davis.DAVIS2016Frames(train=True, db_root_dir=root)
        res["native_loader_samples_per_s"], res["reference_host_pipeline_samples_per_s"] = {}, {}
        for nw in workers:
            res["native_loader_samples_per_s"][nw] = time_loader(frames, nw, davis.collate,
                                                                 post=lambda b: davis.pinned(b["data"]))
            res["reference_host_pipeline_samples_per_s"][nw] = time_loader(ReferenceHostPipeline(frames), nw)
            print(f"{nw} worker(s): native loader {res['native_loader_samples_per_s'][nw]} samples/s, reference host "
                  f"pipeline {res['reference_host_pipeline_samples_per_s'][nw]} samples/s")
        env = dict(os.environ, OSVOS_DB_ROOT=root, OSVOS_SAVE_ROOT=os.path.join(root, "models"))
        res["train_parent"] = {}
        for nw in workers:
            fps, times = parent_fps(["--loader", "native", "--workers", str(nw)], env, len(frames))
            res["train_parent"][f"native_{nw}_workers"] = {"frames_per_s": fps, "epoch_s": times}
            print(f"train_parent.py --loader native --workers {nw}: {fps} frames/s (epoch times {times})")
        fps, times = parent_fps(["--synthetic", "--iters-per-epoch", str(len(frames))], env, len(frames))
        res["train_parent"]["synthetic"] = {"frames_per_s": fps, "epoch_s": times}
        print(f"train_parent.py --synthetic: {fps} frames/s (epoch times {times})")
        res["device_store"] = time_store(frames, workers, a.steps)
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, "time_data.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()

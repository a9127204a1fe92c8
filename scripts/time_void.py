"""Cost of void labels (DESIGN.md §26): the graphed online step (batch 1) and the parent step (batch 12) at 480x854 with
and without void, in alternated pairs, and the id-mode indexed warp against the plain indexed warp at batch 12.
Prints one JSON line with the card's name and power limit.

    python scripts/time_void.py [--pairs 3] [--steps 50]"""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from osvos_pytorch_b200 import augment, ops, parallel, training  # noqa: E402
from osvos_pytorch_b200.networks import vgg_osvos as vo  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _events_ms(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _labels(n, h, w, dev, void):
    g = torch.Generator().manual_seed(5)
    gt = (torch.rand(n, 1, h, w, generator=g) > 0.7).float()
    if void:
        gt[:, :, h // 2:h // 2 + 16, :] = -1            # a void band, as DAVIS-2017 annotations have
    return gt.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    h, w = 480, 854
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=0)
    net.to(dev).train()
    res = {"card": _card(), "online_ms": {"plain": [], "void": []}, "parent_ms": {"plain": [], "void": []}}

    x1 = torch.randn(1, 3, h, w, device=dev)
    online = {}
    for void in (False, True):
        sample = {"image": x1, "gt": _labels(1, h, w, dev, void)}
        online[void] = training.GraphedTrainStep(net, training.ONLINE_WEIGHTS, sample, grad_scale=0.2, void=void)
    x12 = torch.randn(12, 3, h, w, device=dev)
    gts = {void: _labels(12, h, w, dev, void) for void in (False, True)}
    opt = training.make_optimizer(net, "parent", 1e-12, 0.0002, fused=True)
    bucket = parallel.GradientBucket(parallel.trainable_parameters(net), dev)

    def parent(void):
        training.parent_epoch(net, opt, bucket, [{"image": x12, "gt": gts[void]}], 0, 240, 1, void=void)

    for void in (False, True):                            # warm-up of every shape and path
        for _ in range(3):
            online[void]()
            parent(void)
    torch.cuda.synchronize()
    for _ in range(a.pairs):
        for void in (False, True):
            key = "void" if void else "plain"
            res["online_ms"][key].append(_events_ms(online[void], a.steps))
            res["parent_ms"][key].append(_events_ms(lambda: parent(void), max(5, a.steps // 5)))

    # indexed warp of a 12-frame batch from a 60-frame store: 0/255 masks (plain) against object ids (id mode)
    g = torch.Generator().manual_seed(9)
    img = torch.randint(0, 256, (60, h, w, 3), generator=g, dtype=torch.uint8).to(dev)
    ids = torch.randint(0, 4, (60, h, w), generator=g, dtype=torch.uint8).to(dev)
    masks = torch.where(ids != 0, 255, 0).to(torch.uint8)
    stats = ops.label_stats_u8(masks)
    params = augment.draw_params(12, rng=random.Random(1))
    index = list(range(0, 60, 5))
    warp = {"plain": lambda: augment.affine_warp_u8(img, masks, params, stats, index=index),
            "ids": lambda: augment.affine_warp_u8(img, ids, params, index=index, ids="all")}
    for fn in warp.values():
        fn()
    res["warp_ms"] = {k: [] for k in warp}
    for _ in range(a.pairs):
        for k, fn in warp.items():
            res["warp_ms"][k].append(_events_ms(fn, a.steps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()

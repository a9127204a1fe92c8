"""Cost of torch.use_deterministic_algorithms(True) on the training path (DESIGN.md §16).

Times train480 (graphed online fine-tune step, batch 1, 480x854) and parent480 (parent objective step, batch 12,
480x854) with the flag off and on, in alternated pairs, and prints the extra workspace the deterministic forms
allocate per backward.  Device time by CUDA events around `--steps` steps after `--warmup` steps of each mode.

    python scripts/time_deterministic.py [--pairs 3] [--steps 400] [--warmup 20]
    python scripts/time_deterministic.py --profile       # per-kernel device times of train480, off and on
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import osvos_oracle as oc                          # noqa: E402
from osvos_pytorch_b200 import _native as nat, training        # noqa: E402
from osvos_pytorch_b200.networks.vgg_osvos import OSVOS        # noqa: E402
from osvos_pytorch_b200.parallel import GradientBucket, trainable_parameters   # noqa: E402

H, W = 480, 854


def _net():
    m = OSVOS(pretrained=0, verbose=False)
    m.load_state_dict(oc.he_params(seed=0), strict=False)
    with torch.no_grad():
        for mod in list(m.side_prep) + [m.fuse]:
            mod.weight.mul_(0.1)
    return m.cuda().train()


def _timed(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def train480(steps, warmup):
    net = _net()
    x, gt = oc.synthetic_frame(1, H, W, 11)
    sample = {"image": x.cuda(), "gt": gt.cuda()}
    opt = training.make_optimizer(net, "online", 1e-10, fused=True)
    step = training.GraphedTrainStep(net, training.ONLINE_WEIGHTS, sample, grad_scale=0.2, external_pack=True)
    params = [p for g in opt.param_groups for p in g["params"]]

    def one(i):
        step()
        if (i + 1) % 5 == 0:
            opt.step(zero_grad=True)
            step.zero_grads(skip=params)
    return _timed(one, steps, warmup)


def parent480(steps, warmup, batch=12):
    net = _net()
    opt = training.make_optimizer(net, "parent", 1e-10, fused=True)
    bucket = GradientBucket(trainable_parameters(net))
    b = training.synthetic_batch(batch, H, W, 3, "cuda")
    return _timed(lambda i: training.parent_epoch(net, opt, bucket, [b], 0, 240, 1), steps, warmup)


def profile_train480(steps=50, warmup=10):
    """Per-kernel device time of train480 with the flag off and on (torch.profiler, a run of its own): the sites the
    deterministic cost comes from."""
    from torch.profiler import ProfilerActivity, profile
    per = {}
    for mode in (False, True):
        torch.use_deterministic_algorithms(mode)
        net = _net()
        x, gt = oc.synthetic_frame(1, H, W, 11)
        step = training.GraphedTrainStep(net, training.ONLINE_WEIGHTS, {"image": x.cuda(), "gt": gt.cuda()})
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                step()
            torch.cuda.synchronize()
        t = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA":
                name = ev.key.split("(")[0].split("<")[0].replace("void ", "").replace("osvos::", "")
                t[name] = t.get(name, 0.0) + ev.self_device_time_total / steps / 1000.0
        per["on" if mode else "off"] = t
        torch.cuda.empty_cache()
    torch.use_deterministic_algorithms(False)
    names = sorted(set(per["off"]) | set(per["on"]), key=lambda k: per["on"].get(k, 0) - per["off"].get(k, 0),
                   reverse=True)
    rows = [(k, per["off"].get(k, 0.0), per["on"].get(k, 0.0)) for k in names]
    print("train480 per-kernel ms/step (off, on, on - off):")
    for k, a, b in rows:
        if abs(b - a) > 0.005:
            print(f"  {k:40s} {a:7.3f} {b:7.3f} {b - a:+7.3f}")
    print(f"  {'total':40s} {sum(per['off'].values()):7.3f} {sum(per['on'].values()):7.3f}")
    return {k: [a, b] for k, a, b in rows}


def workspace_bytes(n):
    """Extra bytes of one deterministic backward at n x 480 x 854: wgrad slices beyond the default workspaces, and the
    partial rows of the column sums, the side-branch G, conv1_1 and the tail sums."""
    lib = nat.load()
    chans = [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
             (512, 512), (512, 512), (512, 512), (512, 512)]
    stage_of = [0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4]
    wg = colsum = 0
    for (cin, cout), s in zip(chans, stage_of):
        h, w = H, W
        for _ in range(s):
            h, w = (h + 1) // 2, (w + 1) // 2
        if cin > 3:
            wg += (lib.osvos_wgrad_workspace_bytes(n, h, w, cin, cout, nat.FLAG_DETERMINISTIC)
                   - lib.osvos_wgrad_workspace_bytes(n, h, w, cin, cout, 0))
        colsum += lib.osvos_conv3x3_colsum_rows(n, h, w) * cout * 4
    return {"wgrad_slices": int(wg), "colsum_rows_upper_bound": int(colsum),
            "conv1_1_slots": int(lib.osvos_conv_first_bwd_workspace_bytes(n, H, W, nat.FLAG_DETERMINISTIC)),
            "tail_rows": int(lib.osvos_tail_fwd_deterministic_sums(n, H, W) * 8)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile", action="store_true", help="per-kernel times of train480 instead of the timed pairs")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("device:", smi)
    if a.profile:
        print(json.dumps({"device": smi, "train480_kernel_ms_off_on": profile_train480()}))
        return
    res = {"train480": {"off": [], "on": []}, "parent480": {"off": [], "on": []}}
    for p in range(a.pairs):
        for name, fn in (("train480", train480), ("parent480", parent480)):
            for mode in (("off", "on") if p % 2 == 0 else ("on", "off")):
                torch.use_deterministic_algorithms(mode == "on")
                ms = fn(a.steps, a.warmup)
                res[name][mode].append(ms)
                print(f"pair {p} {name} deterministic {mode}: {ms:.3f} ms/step", flush=True)
                torch.cuda.empty_cache()
    torch.use_deterministic_algorithms(False)
    out = {"device": smi, "steps": a.steps, "pairs": a.pairs}
    for name, r in res.items():
        ratios = [on / off for on, off in zip(r["on"], r["off"])]
        out[name] = {"off_ms": r["off"], "on_ms": r["on"], "on_over_off": ratios}
    out["extra_workspace_bytes"] = {"batch1": workspace_bytes(1), "batch12": workspace_bytes(12)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""What the general deconvolution path costs (DESIGN.md §20): the folded bilinear tail against the general tail on the
same bilinear weights (``learn_upsampling`` off against on), 480x854, batch 1, exact precision.

    python scripts/time_upsampling.py [--out results] [--steps 400] [--pairs 3]

Times, with CUDA events over `steps` steps, alternating the two paths `pairs` times:
  1. inference through the replayed CUDA graph (``net(x)`` under no_grad);
  2. forward + backward of the online objective through training.GraphedTrainStep.
Writes <out>/time_upsampling.json; the GPU's name, power limit and SM clocks go with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def event_ms(fn, steps, warmup=20):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.environ.get("OSVOS_RESULTS", "results"))
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    from osvos_pytorch_b200 import training
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS, he_init_
    torch.backends.cudnn.benchmark = False
    sample = training.synthetic_batch(1, 480, 854, 0, "cuda")
    nets, steps = {}, {}
    for learn in (False, True):
        net = he_init_(OSVOS(pretrained=0, verbose=False), seed=0).cuda()
        net.learn_upsampling = learn
        nets[learn] = net
        steps[learn] = training.GraphedTrainStep(net, training.ONLINE_WEIGHTS, sample)
    rows = {"inference_ms": {False: [], True: []}, "train_step_ms": {False: [], True: []}}
    for _ in range(args.pairs):
        for learn in (False, True):
            with torch.no_grad():
                rows["inference_ms"][learn].append(event_ms(lambda: nets[learn](sample["image"]), args.steps))
            rows["train_step_ms"][learn].append(event_ms(steps[learn].graph.replay, args.steps))
    res = {"gpu": gpu_info(), "shape": [1, 3, 480, 854], "precision": "exact", "steps": args.steps}
    for key, by in rows.items():
        res[key] = {"folded": by[False], "general": by[True],
                    "overhead_pct": 100.0 * (min(by[True]) / min(by[False]) - 1.0)}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_upsampling.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

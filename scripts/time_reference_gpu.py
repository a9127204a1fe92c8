"""Times the UNMODIFIED reference modules (oracle/_ref) on the GPU itself - the "real kernel to beat" of SURVEY 8(d):
stock cuDNN with TF32 (torch default for convs), strict fp32 (allow_tf32=False), and channels_last + bf16 autocast.

    python scripts/time_reference_gpu.py [H W] [--train]

Prints one JSON line.  Development aid; bench.py carries the same measurement as `gpu_reference`.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle import osvos_oracle as oc
from oracle import ref_loader


def time_variant(net, x, gt, lay, mode, train, iters=60, warm=10):
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = mode != "fp32"
    torch.backends.cuda.matmul.allow_tf32 = mode != "fp32"
    if mode == "bf16_channels_last":
        net = net.to(memory_format=torch.channels_last)
        x = x.contiguous(memory_format=torch.channels_last)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16_channels_last")):
            if train:
                net.zero_grad(set_to_none=True)
                outs = net(x)
                loss = lay.class_balanced_cross_entropy_loss(outs[-1].float(), gt, size_average=False)
                loss.backward()
            else:
                with torch.no_grad():
                    outs = net(x)
        return outs

    for _ in range(warm):
        outs = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        outs = step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, [o.detach().float() for o in outs]


def main():
    argv = [a for a in sys.argv[1:] if not a.startswith("--")]
    h, w = (int(argv[0]), int(argv[1])) if len(argv) >= 2 else (480, 854)
    train = "--train" in sys.argv
    params = oc.he_params(seed=0)
    ref = ref_loader.load()
    x, gt = oc.synthetic_frame(1, h, w, 1234)
    with torch.no_grad():
        cpu_out = oc.osvos_forward(params, x)
    x, gt = x.cuda(), gt.cuda()
    out = {"h": h, "w": w, "train": train}
    for mode in ("tf32_default", "fp32", "bf16_channels_last"):
        net = ref_loader.build_reference(params, "cuda")
        net.train(train)
        ms, outs = time_variant(net, x, gt, ref.layers, mode, train)
        err = float((outs[-1].cpu() - cpu_out[-1]).abs().max() / cpu_out[-1].abs().max())
        flips = int(((outs[-1].cpu() > 0) != (cpu_out[-1] > 0)).sum())
        out[mode] = {"ms": round(ms, 4), "fps": round(1000 / ms, 1), "fused_maxrel_vs_cpu_fp32": err, "mask_flips_vs_cpu_fp32": flips}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

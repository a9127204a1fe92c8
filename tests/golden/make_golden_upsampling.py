"""Generate tests/golden/reference_upsampling.npz by running the UNMODIFIED reference module with deconvolution weights
that are not interp_surgery's bilinear taps (the general tail, DESIGN.md §20).

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden_upsampling.py

Inputs are regenerated from seeds: the He-init trunk of oracle.he_params(seed=0) and upsampling_ref.deconv_weights
(seed 100, kinds 'noisy' and 'dense').  Stored: the five maps at 48x70 and 33x45 (batch 2), the online and parent
objectives at 48x70, and every one of the 52 parameter gradients (norm, sum and eight sampled values each).
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, "/root/reference")

import networks.vgg_osvos as ref_net          # noqa: E402  (reference, unmodified)
import layers.osvos_layers as ref_layers      # noqa: E402  (reference, unmodified)
from oracle import osvos_oracle as oc         # noqa: E402
from upsampling_ref import KINDS, deconv_weights  # noqa: E402

FWD_CASES = {"48x70": (1, 48, 70, 11), "33x45_n2": (2, 33, 45, 12)}
BWD_CASE = (1, 48, 70, 21)
PARENT_SIDE_WEIGHT = 0.75


def params_for(kind):
    p = oc.he_params(seed=0, include_upscale=True)
    p.update(deconv_weights(100, kind))
    return p


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    fx = {"torch_version": np.array(torch.__version__)}
    for kind in KINDS:
        with contextlib.redirect_stdout(io.StringIO()):
            net = ref_net.OSVOS(pretrained=0)
        net.load_state_dict(params_for(kind))
        for tag, (n, h, w, seed) in FWD_CASES.items():
            x, _ = oc.synthetic_frame(n, h, w, seed)
            with torch.no_grad():
                outs = net(x)
            for i, o in enumerate(outs):
                fx[f"{kind}.fwd_{tag}.out{i}"] = o.numpy().astype(np.float32)
        n, h, w, seed = BWD_CASE
        x, gt = oc.synthetic_frame(n, h, w, seed)
        for obj in ("online", "parent"):
            net.zero_grad()
            outs = net(x)
            if obj == "online":
                loss = ref_layers.class_balanced_cross_entropy_loss(outs[-1], gt, size_average=False)
            else:
                ls = [ref_layers.class_balanced_cross_entropy_loss(o, gt, size_average=False) for o in outs]
                loss = PARENT_SIDE_WEIGHT * sum(ls[:-1]) + ls[-1]
            loss.backward()
            fx[f"{kind}.bwd.{obj}.loss"] = np.array(float(loss))
            for name, p in net.named_parameters():
                if p.grad is None:
                    fx[f"{kind}.bwd.{obj}.none.{name}"] = np.array(0)
                    continue
                g = p.grad.detach().double().flatten()
                idx = torch.linspace(0, g.numel() - 1, steps=min(8, g.numel())).long()
                fx[f"{kind}.bwd.{obj}.norm.{name}"] = np.array(float(g.norm()))
                fx[f"{kind}.bwd.{obj}.sum.{name}"] = np.array(float(g.sum()))
                fx[f"{kind}.bwd.{obj}.idx.{name}"] = idx.numpy()
                fx[f"{kind}.bwd.{obj}.val.{name}"] = g[idx].numpy()
    out = os.path.join(HERE, "reference_upsampling.npz")
    np.savez_compressed(out, **fx)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()

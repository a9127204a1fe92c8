"""fp64 reference of one training step as the package's trainers take it (DESIGN.md §11): the gated forward, the weighted
class-balanced objective and the gradient of every parameter and of the input.

The objective is  sum_k w_k * grad_scale * L_k / n  over the five maps (n = batch), which is how GraphedTrainStep and
OSVOS.forward_objective(size_average=False, batch_average=True) form it.  L_k is the reference's class-balanced BCE
(oc.class_balanced_cross_entropy_loss), or void_loss_ref.void_loss_torch with ``void`` (labels < 0 left out).  The tail
is the oracle's folded one (oc.osvos_forward, bilinear deconvolutions) or, with ``general``, the reference's literal
tail on any deconvolution weights (upsampling_ref.literal_forward).  Parameters that do not reach the objective get no
entry - score_dsn.i when w_i = 0, the deconvolutions unless ``learn_upsampling`` - as the CUDA node returns None for
them.  Runs on whatever device the tensors are on."""
import torch
import torch.nn.functional as F

from oracle import osvos_oracle as oc
from upsampling_ref import literal_forward
from void_loss_ref import void_loss_torch

# loss-weight configurations of the trainers: online fine-tuning (train_online.py:127), parent training at
# epoch / nEpochs = 0.65 (train_parent.py:143-147), and one with zero and non-unit weights mixed
WEIGHTS = {"online": (0.0, 0.0, 0.0, 0.0, 1.0), "parent": (0.35, 0.35, 0.35, 0.35, 1.0),
           "mixed": (1.0, 0.0, 2.0, 0.0, 0.25)}
# per-parameter gradient bound with the CUDA pass's ReLU masks and pool argmax injected into the reference: only fp32
# arithmetic differs (tests/test_gpu_backward.py); a 1 % error in one parameter's gradient exceeds it 20 times
GATED_TOL = 5e-4
# fuse.bias and side_prep.i.bias: sums over every pixel of the maps' loss gradient, with no ReLU or pooling between them
# and the loss.  Their positive and negative terms cancel (the class balance weighs both classes equally), so the fp32
# forward's per-pixel logit error enters them multiplied by sum|g| / |sum g|: measured up to 6.6e-4 at 1x40x56 on an
# H100.  A 1 % error still exceeds this bound 5 times.
SUM_TOL = 2e-3


def tolerance(name):
    """The gated bound of one parameter's gradient."""
    return SUM_TOL if name == "fuse.bias" or (name.startswith("side_prep.") and name.endswith(".bias")) else GATED_TOL


def expected_keys(weights, general=False, learn_upsampling=False):
    """The parameters whose gradient the objective with these loss weights reaches (independent of the reference's
    autograd, which the CPU tests hold to it)."""
    keys = set()
    for k in oc.param_shapes():
        if k.startswith("stages.") or k.startswith("side_prep."):
            keys.add(k)
        elif k.startswith("score_dsn."):
            if weights[int(k.split(".")[1])] != 0.0:
                keys.add(k)
        elif k.startswith("fuse."):
            if weights[4] != 0.0:
                keys.add(k)
        elif general and learn_upsampling:
            i = int(k.split(".")[1])
            if (k.startswith("upscale.") and weights[4] != 0.0) or (k.startswith("upscale_.") and weights[i] != 0.0):
                keys.add(k)
    return keys


def conv_outputs(params, x):
    """The 13 post-ReLU trunk activations of the ungated forward (NCHW, the dtype of x)."""
    names = oc.trunk_conv_names()
    outs, k, a = [], 0, x
    with torch.no_grad():
        for i, chans in enumerate(oc.STAGE_CHANNELS):
            if i > 0:
                a = F.max_pool2d(a, 2, 2, ceil_mode=True)
            for _ in chans:
                a = F.relu(F.conv2d(a, params[names[k] + ".weight"], params[names[k] + ".bias"], padding=1))
                outs.append(a)
                k += 1
    return outs


def gates_of(conv_outs, device=None):
    """oc.gates_from_activations of 13 activations, moved to ``device``."""
    g = oc.gates_from_activations(conv_outs)
    if device is None:
        return g
    return {"relu": [t.to(device) for t in g["relu"]], "pool": [t.to(device) for t in g["pool"]]}


def map_losses(outs, gt, void=False):
    """L_k / n of the five maps."""
    n = int(gt.shape[0])
    if void:
        return [void_loss_torch(o, gt, divisor=float(n)) for o in outs]
    return [oc.class_balanced_cross_entropy_loss(o, gt, size_average=False, batch_average=True) for o in outs]


def reference_step(params, x, gt, weights, grad_scale=1.0, void=False, gates=None, general=False,
                   learn_upsampling=False, want_dx=False):
    """One gated forward + objective + backward in the dtype and on the device of ``x``.  ``params``: state-dict
    tensors (the eight deconvolution weights are read with ``general`` only).
    -> {"loss": weighted objective, "per_map": [5] L_k / n, "grads": {name: gradient}, "dx": input gradient | None}."""
    dt, dev = x.dtype, x.device
    leaves = {}
    for k, v in params.items():
        if k.startswith("upscale") and not general:
            continue
        t = v.detach().to(dev, dt).clone()
        if not k.startswith("upscale") or learn_upsampling:
            t.requires_grad_(True)
        leaves[k] = t
    xin = x.detach().clone().requires_grad_(want_dx)
    gt = gt.to(dev, dt)
    outs = literal_forward(leaves, xin, gates) if general else oc.osvos_forward(leaves, xin, gates=gates)
    per_map = map_losses(outs, gt, void)
    total = None
    for wk, lk in zip(weights, per_map):
        if wk != 0.0:
            term = (float(wk) * float(grad_scale)) * lk
            total = term if total is None else total + term
    total.backward()
    grads = {k: v.grad for k, v in leaves.items() if v.requires_grad and v.grad is not None}
    return {"loss": total.detach(), "per_map": torch.stack([l.detach() for l in per_map]), "grads": grads,
            "dx": xin.grad if want_dx else None}


def relnorm(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def gradient_errors(got, ref):
    """Per-parameter ||got - ref|| / ||ref||.  ``got``: {name: gradient written by the step, or None when it wrote none}
    over every trainable parameter.  The parameters with a gradient must be exactly the reference's: a missing or an
    extra one fails."""
    have = {k for k, v in got.items() if v is not None}
    missing, extra = sorted(set(ref) - have), sorted(have - set(ref))
    assert not missing and not extra, f"gradients missing for {missing}, unexpected for {extra}"
    return {k: relnorm(got[k], ref[k]) for k in ref}


def check_gradients(got, ref):
    """gradient_errors, each under its parameter's ``tolerance`` -> (worst error, its parameter)."""
    errs = gradient_errors(got, ref)
    worst = max(errs, key=errs.get)
    bad = {k: v for k, v in errs.items() if v >= tolerance(k)}
    assert not bad, f"gradient error above its bound: {bad}"
    return errs[worst], worst

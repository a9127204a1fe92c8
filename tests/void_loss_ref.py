"""fp64 restatement of the class-balanced BCE with void labels (DESIGN.md §26) and of the DAVIS-2017 id rule.

Labels hold 1 (object), 0 (background) or -1 (void).  With b = [y >= .5] over the whole tensor:
  P = #{y >= .5}, Nn = #{0 <= y < .5}, N = P + Nn (void pixels are not counted);
  loss = (Nn/N * sum_{y>=.5} (softplus(x) - x) + P/N * sum_{0<=y<.5} softplus(x)) / divisor;
  dL/dx = w * (sigmoid(x) - b) / divisor, w = Nn/N on positives, P/N on negatives, 0 on void;
  N == 0 gives loss 0 and gradient 0.
Id maps: 255 -> -1, an object (1..254, or == object k) -> 1, else 0."""
import numpy as np
import torch

from oracle import osvos_oracle as oc


def void_loss(x, y, divisor=1.0):
    """(loss, dL/dx) in fp64 numpy for logits ``x`` and labels ``y`` (any matching shapes)."""
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    pos, neg = y >= 0.5, (y >= 0) & (y < 0.5)
    p, nn = float(pos.sum()), float(neg.sum())
    n = p + nn
    if n == 0:
        return 0.0, np.zeros_like(x)
    sp = np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))
    loss = (nn / n * (sp - x)[pos].sum() + p / n * sp[neg].sum()) / divisor
    sg = 1.0 / (1.0 + np.exp(-x))
    g = np.where(pos, nn / n * (sg - 1.0), np.where(neg, p / n * sg, 0.0)) / divisor
    return float(loss), g


def void_loss_torch(x, y, divisor=1.0):
    """The same loss as a differentiable torch expression in the dtype of ``x`` (for autograd routes)."""
    pos = (y >= 0.5).to(x.dtype)
    neg = ((y >= 0) & (y < 0.5)).to(x.dtype)
    p, nn = pos.sum(), neg.sum()
    n = p + nn
    if float(n) == 0:
        return (x * 0).sum()
    sp = torch.clamp(x, min=0) + torch.log1p(torch.exp(-x.abs()))
    return (nn / n * (pos * (sp - x)).sum() + p / n * (neg * sp).sum()) / divisor


def labels_of_ids(ids, obj=None):
    """uint8 id maps -> fp32 labels (-1 void, 1 object, 0 else); ``obj`` None: every object 1..254."""
    ids = np.asarray(ids)
    fg = (ids >= 1) & (ids <= 254) if obj is None else ids == obj
    return np.where(ids == 255, -1.0, np.where(fg, 1.0, 0.0)).astype(np.float32)


def warp_ids(ids, rot, sc, flip, obj=None):
    """RandomHorizontalFlip + ScaleNRotate of one id map [H,W] sampled nearest (the oracle's restatement of
    cv2.warpAffine(INTER_NEAREST), out-of-frame ids 0), then the id rule -> fp32 [H,W]."""
    warped = oc.scale_n_rotate(np.asarray(ids, dtype=np.float32)[None], rot, sc, flip, nearest=True)[0]
    return labels_of_ids(warped.astype(np.uint8), obj)

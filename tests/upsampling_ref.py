"""Test aids for the general deconvolution path (DESIGN.md §20): seeded non-bilinear deconvolution weights, the
reference's literal tail (dense ConvTranspose2d, centre crop, cat, 1x1 fuse; networks/vgg_osvos.py:59-74) on a gated
trunk, and the V / H algebra the kernels implement, restated in torch."""
import torch
import torch.nn.functional as F

from oracle import osvos_oracle as oc

KINDS = ("noisy", "dense")


def deconv_weights(seed, kind):
    """{upscale.i.weight, upscale_.i.weight} with the reference's shapes.  'noisy': the bilinear taps plus N(0, 0.05)
    noise (U stays diagonal in its channels only up to the noise); 'dense': a dense U ~ N(0, 0.1) with off-diagonal
    channel mixing and noisy upscale_ taps."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i in range(4):
        s = 2 ** (i + 1)
        k = 2 * s
        bil16, bil1 = oc.interp_weight(16, s), oc.interp_weight(1, s)
        if kind == "noisy":
            out[f"upscale.{i}.weight"] = bil16 + 0.05 * torch.randn(16, 16, k, k, generator=g)
        elif kind == "dense":
            out[f"upscale.{i}.weight"] = 0.1 * torch.randn(16, 16, k, k, generator=g)
        else:
            raise ValueError(kind)
        out[f"upscale_.{i}.weight"] = bil1 + 0.05 * torch.randn(1, 1, k, k, generator=g)
    return out


def literal_forward(params, x, gates=None):
    """The five maps through the reference's literal tail with any upscale* weights, on oc.trunk_forward(gates)."""
    h, w = int(x.shape[-2]), int(x.shape[-1])
    stage_out = oc.trunk_forward(params, x, gates)
    side, side_out = [], []
    for i in range(4):
        s = 2 ** (i + 1)
        feat = F.conv2d(stage_out[i + 1], params[f"side_prep.{i}.weight"], params[f"side_prep.{i}.bias"], padding=1)
        side.append(oc.center_crop(F.conv_transpose2d(feat, params[f"upscale.{i}.weight"], stride=s), h, w))
        score = F.conv2d(feat, params[f"score_dsn.{i}.weight"], params[f"score_dsn.{i}.bias"])
        side_out.append(oc.center_crop(F.conv_transpose2d(score, params[f"upscale_.{i}.weight"], stride=s), h, w))
    out = F.conv2d(torch.cat(side, dim=1), params["fuse.weight"], params["fuse.bias"])
    return side_out + [out]


def literal_forward_backward(params, x, gt, objective="online", side_weight=1.0, gates=None):
    """(loss, outputs, grads of every parameter, the eight deconvolution weights included) of the literal route."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    outs = literal_forward(leaves, x, gates)
    if objective == "online":
        loss = oc.online_objective(outs, gt)
    else:
        loss = oc.parent_objective(outs, gt, side_weight)
    loss.backward()
    return loss.detach(), [o.detach() for o in outs], {k: v.grad for k, v in leaves.items() if v.grad is not None}


def fold_v(u16, fuse_slice):
    """V[t][ci] = sum_co f[co] U[ci][co][t] as [T, 16] (t = ty * 2s + tx)."""
    return torch.einsum("o,iot->ti", fuse_slice, u16.flatten(2))


def tail_by_taps(feat, p, a_taps, v_taps, s, h, w):
    """side / fused contribution of one scale written as the kernels compute it: every output pixel gathers its <= 2 x 2
    sources with per-tap weights.  feat [n,16,hk,wk], p [n,1,hk,wk], a_taps [T], v_taps [T,16] -> ([n,1,h,w] x 2)."""
    n, _, hk, wk = feat.shape
    k = 2 * s
    top, _ = oc.crop_offsets((hk - 1) * s + k, h)
    left, _ = oc.crop_offsets((wk - 1) * s + k, w)
    side = torch.zeros(n, 1, h, w, dtype=feat.dtype)
    fused = torch.zeros(n, 1, h, w, dtype=feat.dtype)
    for y in range(h):
        for x in range(w):
            oy, ox = y + top, x + left
            for iy in (oy // s, oy // s - 1):
                for ix in (ox // s, ox // s - 1):
                    if 0 <= iy < hk and 0 <= ix < wk:
                        t = (oy - iy * s) * k + (ox - ix * s)
                        side[:, 0, y, x] += a_taps[t] * p[:, 0, iy, ix]
                        fused[:, 0, y, x] += (v_taps[t] * feat[:, :, iy, ix]).sum(1)
    return side, fused

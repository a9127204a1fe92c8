"""CPU oracle for the OSVOS per-frame hot path.  TEST INFRASTRUCTURE ONLY.

This file restates, function by function, what the reference computes on the
hot path (reference = kmaninis/OSVOS-PyTorch, files cited as file:line below).
It is the checker for the CUDA path: only ``tests/``, ``__graft_entry__.smoke``
and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it.
The product package (``osvos_pytorch_b200``) never does, and raises if its CUDA
library is missing instead of falling back to anything in here.

Parity pinning: the reference ships no tests / golden vectors (SURVEY.md section 4),
so the oracle is pinned against OUTPUTS OF THE UNMODIFIED REFERENCE run in the
build container: ``tests/golden/make_golden.py`` imports
``/root/reference/networks/vgg_osvos.py`` and ``layers/osvos_layers.py``,
runs them on seeded inputs and commits the results under ``tests/golden/``;
``tests/test_oracle.py`` checks this file against those fixtures and against
the analytic known-answer values of SURVEY.md section 8c.

The arithmetic of the reference lives in PyTorch (torch.nn.Conv2d /
ConvTranspose2d / MaxPool2d, reference pins "PyTorch 0.4", README.md:21; here
torch 2.11).  The dense 3x3 convolutions are restated through
``torch.nn.functional.conv2d`` (the same third-party arithmetic the reference
calls at networks/vgg_osvos.py:142); everything the reference builds on top of
it - the zero-padded bilinear "deconvolution", the crop offsets, the fusion,
the loss and its gradient - is restated in closed form, independently of
ConvTranspose2d / F.pad / autograd, so that the two routes cross-check.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# networks/vgg_osvos.py:19-24 : channel plan of the five trunk stages
STAGE_CHANNELS: Tuple[Tuple[int, ...], ...] = ((64, 64), (128, 128), (256, 256, 256),
                                               (512, 512, 512), (512, 512, 512))
STAGE_IN: Tuple[int, ...] = (3, 64, 128, 256, 512)
SIDE_CHANNELS = 16                       # networks/vgg_osvos.py:41
# dataloaders/davis_2016.py:19 : BGR mean subtracted from 0..255 images
MEANVAL = (104.00699, 116.66877, 122.67892)


# --------------------------------------------------------------------------
# state-dict naming (networks/vgg_osvos.py:27-54, SURVEY.md section 8b)
# --------------------------------------------------------------------------
def trunk_conv_names() -> List[str]:
    """'stages.<i>.<j>' prefixes of the 13 trunk convs in forward order.

    Stage 1 is [conv, relu, conv, relu]; stages 2-5 start with a MaxPool2d
    (networks/vgg_osvos.py:136-145), which shifts the conv indices by one.
    """
    names = []
    for i, chans in enumerate(STAGE_CHANNELS):
        first = 0 if i == 0 else 1
        for j in range(len(chans)):
            names.append(f"stages.{i}.{first + 2 * j}")
    return names


def param_shapes() -> Dict[str, Tuple[int, ...]]:
    """All 52 state-dict tensors (SURVEY.md says 50; the reference has 52) and their shapes (SURVEY.md section 8b)."""
    shapes: Dict[str, Tuple[int, ...]] = {}
    names = trunk_conv_names()
    k = 0
    for i, chans in enumerate(STAGE_CHANNELS):
        cin = STAGE_IN[i]
        for c in chans:
            shapes[names[k] + ".weight"] = (c, cin, 3, 3)
            shapes[names[k] + ".bias"] = (c,)
            cin = c
            k += 1
    for i in range(4):
        c = STAGE_CHANNELS[i + 1][-1]
        ks = 2 ** (i + 2)
        shapes[f"side_prep.{i}.weight"] = (SIDE_CHANNELS, c, 3, 3)
        shapes[f"side_prep.{i}.bias"] = (SIDE_CHANNELS,)
        shapes[f"score_dsn.{i}.weight"] = (1, SIDE_CHANNELS, 1, 1)
        shapes[f"score_dsn.{i}.bias"] = (1,)
        shapes[f"upscale.{i}.weight"] = (SIDE_CHANNELS, SIDE_CHANNELS, ks, ks)
        shapes[f"upscale_.{i}.weight"] = (1, 1, ks, ks)
    shapes["fuse.weight"] = (1, 4 * SIDE_CHANNELS, 1, 1)
    shapes["fuse.bias"] = (1,)
    return shapes


# --------------------------------------------------------------------------
# layers/osvos_layers.py helpers
# --------------------------------------------------------------------------
def upsample_filt(size: int) -> np.ndarray:
    """2-D bilinear tap table, layers/osvos_layers.py:59-67.

    f[t] = 1 - |t - c| / factor with factor = ceil(size/2) and c = factor-1 for
    odd sizes, factor-0.5 for even ones; the 2-D table is the outer product.
    """
    factor = (size + 1) // 2
    center = factor - 1 if size % 2 == 1 else factor - 0.5
    t = np.arange(size, dtype=np.float64)
    f1 = 1.0 - np.abs(t - center) / factor
    return np.outer(f1, f1)


def upsample_taps_1d(stride: int) -> np.ndarray:
    """1-D taps of the kernel-2s/stride-s deconvolution (networks/vgg_osvos.py:45-46)."""
    size = 2 * stride
    t = np.arange(size, dtype=np.float64)
    return 1.0 - np.abs(t - (stride - 0.5)) / stride


def interp_weight(channels: int, stride: int, dtype=torch.float32) -> torch.Tensor:
    """Weight tensor that layers/osvos_layers.py:72-85 (interp_surgery) writes.

    (channels, channels, 2s, 2s), bilinear table on the (i, i) diagonal, exact
    zeros elsewhere (networks/vgg_osvos.py:87-89 zeroes the tensor first).
    """
    k = 2 * stride
    w = torch.zeros(channels, channels, k, k, dtype=dtype)
    filt = torch.from_numpy(upsample_filt(k)).to(dtype)
    for i in range(channels):
        w[i, i] = filt
    return w


def crop_offsets(size: int, target: int) -> Tuple[int, int]:
    """(leading, trailing) rows/cols removed by layers/osvos_layers.py:51-56.

    The reference pads by [ceil(-d/2), floor(-d/2)] with d = size - target, i.e.
    it removes floor(d/2) at the top/left and ceil(d/2) at the bottom/right.
    """
    d = size - target
    return d // 2, d - d // 2


def center_crop(x: torch.Tensor, height: int, width: int) -> torch.Tensor:
    """layers/osvos_layers.py:51-56 restated as slicing."""
    top, bottom = crop_offsets(x.shape[2], height)
    left, right = crop_offsets(x.shape[3], width)
    return x[:, :, top:x.shape[2] - bottom, left:x.shape[3] - right]


def pooled_size(n: int) -> int:
    """MaxPool2d(2, 2, ceil_mode=True) output length, networks/vgg_osvos.py:140."""
    return (n + 1) // 2


def upsample_zero_padded(x: torch.Tensor, stride: int) -> torch.Tensor:
    """Closed form of ConvTranspose2d(C, C, 2s, stride=s, bias=False) with the
    interp_surgery weights (networks/vgg_osvos.py:45-46, layers/osvos_layers.py:72-85).

    out[oy, ox] = sum_{iy, ix} f[oy - iy*s] f[ox - ix*s] in[iy, ix], f = 1-D taps,
    taps outside [0, 2s) are zero; at most two source rows/cols contribute, and
    the border is attenuated (zero padding, not edge replication).
    Output size (h + 1) * s.  Written as two dense matrix products so that it
    shares no code with ConvTranspose2d.
    """
    n, c, h, w = x.shape
    f = upsample_taps_1d(stride)

    def matrix(n_in: int) -> torch.Tensor:
        n_out = (n_in + 1) * stride
        m = np.zeros((n_out, n_in), dtype=np.float64)
        for i in range(n_in):
            m[i * stride:i * stride + 2 * stride, i] = f
        return torch.from_numpy(m).to(x.device, x.dtype)

    my, mx = matrix(h), matrix(w)
    return torch.einsum("oy,ncyx,px->ncop", my, x, mx)


# --------------------------------------------------------------------------
# network forward, networks/vgg_osvos.py:59-74
# --------------------------------------------------------------------------
def trunk_forward(params: Dict[str, torch.Tensor], x: torch.Tensor, gates=None) -> List[torch.Tensor]:
    """Outputs of the five stages (each after its last ReLU), networks/vgg_osvos.py:61,66.

    ``gates`` (test aid, see ``gates_from_activations``): the SELECTIONS of the network's two discontinuous ops taken
    from another implementation's forward pass - ``gates["relu"][k]`` a 0/1 mask replacing ``z > 0`` of conv k,
    ``gates["pool"][i]`` the flat argmax indices of pooling i.  With them the network is the same piecewise-linear
    function evaluated on the other implementation's linear piece, so gradients can be compared without the
    mask / argmax flips that a 1e-5 forward difference causes (tests/test_gpu_backward.py)."""
    names = trunk_conv_names()
    k = 0
    outs = []
    for i, chans in enumerate(STAGE_CHANNELS):
        if i > 0:
            if gates is None:
                x = F.max_pool2d(x, kernel_size=2, stride=2, ceil_mode=True)
            else:
                idx = gates["pool"][i - 1]
                x = x.flatten(2).gather(2, idx.flatten(2)).view(idx.shape)
        for _ in chans:
            z = F.conv2d(x, params[names[k] + ".weight"], params[names[k] + ".bias"], padding=1)
            x = F.relu(z) if gates is None else z * gates["relu"][k].to(z.dtype)
            k += 1
        outs.append(x)
    return outs


def gates_from_activations(conv_outputs: Sequence[torch.Tensor]):
    """ReLU masks and pooling argmax indices implied by the 13 post-ReLU trunk activations (NCHW) of a forward pass."""
    relu = [(a > 0) for a in conv_outputs]
    pool, k = [], 0
    for i, chans in enumerate(STAGE_CHANNELS):
        k += len(chans)
        if i < len(STAGE_CHANNELS) - 1:
            pool.append(F.max_pool2d(conv_outputs[k - 1].float(), kernel_size=2, stride=2, ceil_mode=True,
                                     return_indices=True)[1])
    return {"relu": relu, "pool": pool}


def osvos_forward(params: Dict[str, torch.Tensor], x: torch.Tensor,
                  return_side_feats: bool = False, gates=None):
    """The five logit maps [side_out1..4, fused], networks/vgg_osvos.py:59-74.

    The side branch is computed in the fused form proved equivalent in
    SURVEY.md section 8a (a8): fuse(cat(crop(up(side_i)))) ==
    sum_i crop(up(conv1x1(side_i, Wf[:, 16i:16i+16]))) + b_f, by linearity of
    the (diagonal, bilinear) deconvolution.  ``tests/test_oracle.py`` checks
    this against the reference's literal cat + 1x1-conv route.
    """
    h, w = int(x.shape[-2]), int(x.shape[-1])
    stage_out = trunk_forward(params, x, gates)
    side_out, side_feats = [], []
    fused = None
    wf = params["fuse.weight"]
    for i in range(4):
        s = 2 ** (i + 1)
        feat = F.conv2d(stage_out[i + 1], params[f"side_prep.{i}.weight"],
                        params[f"side_prep.{i}.bias"], padding=1)            # :67 (no ReLU)
        side_feats.append(feat)
        score = F.conv2d(feat, params[f"score_dsn.{i}.weight"], params[f"score_dsn.{i}.bias"])  # :69
        side_out.append(center_crop(upsample_zero_padded(score, s), h, w))
        part = F.conv2d(feat, wf[:, SIDE_CHANNELS * i:SIDE_CHANNELS * (i + 1)])
        part = center_crop(upsample_zero_padded(part, s), h, w)
        fused = part if fused is None else fused + part
    fused = fused + params["fuse.bias"].view(1, 1, 1, 1)                      # :72
    outs = side_out + [fused]
    if return_side_feats:
        return outs, side_feats
    return outs


def osvos_forward_literal(params: Dict[str, torch.Tensor], x: torch.Tensor) -> List[torch.Tensor]:
    """Same maps through the reference's literal op sequence (dense 16x16
    ConvTranspose2d, negative pad, cat, 1x1 fuse; networks/vgg_osvos.py:65-73).
    Uses the ``upscale*.weight`` tensors in ``params`` if present."""
    h, w = int(x.shape[-2]), int(x.shape[-1])
    stage_out = trunk_forward(params, x)
    side, side_out = [], []
    for i in range(4):
        s = 2 ** (i + 1)
        feat = F.conv2d(stage_out[i + 1], params[f"side_prep.{i}.weight"],
                        params[f"side_prep.{i}.bias"], padding=1)
        w16 = params.get(f"upscale.{i}.weight", None)
        if w16 is None:
            w16 = interp_weight(SIDE_CHANNELS, s, x.dtype)
        w1 = params.get(f"upscale_.{i}.weight", None)
        if w1 is None:
            w1 = interp_weight(1, s, x.dtype)
        side.append(center_crop(F.conv_transpose2d(feat, w16, stride=s), h, w))
        score = F.conv2d(feat, params[f"score_dsn.{i}.weight"], params[f"score_dsn.{i}.bias"])
        side_out.append(center_crop(F.conv_transpose2d(score, w1, stride=s), h, w))
    out = F.conv2d(torch.cat(side, dim=1), params["fuse.weight"], params["fuse.bias"])
    return side_out + [out]


# --------------------------------------------------------------------------
# loss, layers/osvos_layers.py:19-48
# --------------------------------------------------------------------------
def class_balanced_cross_entropy_loss(output: torch.Tensor, label: torch.Tensor,
                                      size_average: bool = True, batch_average: bool = True) -> torch.Tensor:
    """Closed form of layers/osvos_layers.py:19-48.

    y = 1[label >= .5]; P = sum y, Nn = sum (1-y) over the WHOLE tensor (:28-32);
    per pixel  -loss_val = softplus(x) - y*x  (:34-36, stable form);
    L = Nn/(P+Nn) * sum_{y=1} (softplus(x) - x) + P/(P+Nn) * sum_{y=0} softplus(x) (:38-41);
    divided by numel if size_average else by batch size if batch_average (:43-46).
    """
    y = (label >= 0.5).to(output.dtype)
    num_pos = y.sum()
    num_neg = (1.0 - y).sum()
    total = num_pos + num_neg
    softplus = torch.clamp(output, min=0) + torch.log1p(torch.exp(-output.abs()))
    per_px = softplus - y * output
    loss = num_neg / total * (y * per_px).sum() + num_pos / total * ((1.0 - y) * per_px).sum()
    if size_average:
        loss = loss / float(np.prod(label.shape))
    elif batch_average:
        loss = loss / label.shape[0]
    return loss


def class_balanced_cross_entropy_grad(output: torch.Tensor, label: torch.Tensor,
                                      size_average: bool = True, batch_average: bool = True) -> torch.Tensor:
    """dL/d(output) of the loss above: w * (sigmoid(x) - y) / divisor with
    w = y*Nn/N + (1-y)*P/N (derivative of layers/osvos_layers.py:34-46)."""
    y = (label >= 0.5).to(output.dtype)
    num_pos = y.sum()
    num_neg = (1.0 - y).sum()
    total = num_pos + num_neg
    wgt = y * (num_neg / total) + (1.0 - y) * (num_pos / total)
    g = wgt * (torch.sigmoid(output) - y)
    if size_average:
        g = g / float(np.prod(label.shape))
    elif batch_average:
        g = g / label.shape[0]
    return g


# --------------------------------------------------------------------------
# objectives of the two entry points
# --------------------------------------------------------------------------
def online_objective(outputs: Sequence[torch.Tensor], gts: torch.Tensor) -> torch.Tensor:
    """train_online.py:127 : fused map only, size_average=False."""
    return class_balanced_cross_entropy_loss(outputs[-1], gts, size_average=False)


def parent_objective(outputs: Sequence[torch.Tensor], gts: torch.Tensor, side_weight: float) -> torch.Tensor:
    """train_parent.py:143-147 : side_weight * sum_{i<4} L_i + L_fuse, side_weight = 1 - epoch/nEpochs."""
    losses = [class_balanced_cross_entropy_loss(o, gts, size_average=False) for o in outputs]
    return side_weight * sum(losses[:-1]) + losses[-1]


def forward_backward(params: Dict[str, torch.Tensor], x: torch.Tensor, gts: torch.Tensor,
                     objective: str = "online", side_weight: float = 1.0,
                     grad_scale: float = 1.0, gates=None):
    """One fwd+bwd of the reference loop body (train_online.py:124-141 /
    train_parent.py:140-164): returns (loss, outputs, grads dict).  ``grad_scale``
    is the 1/nAveGrad factor of train_online.py:140.  Autograd over the oracle
    forward; parameters that do not influence the objective get no entry
    (SURVEY.md section 8c item 9)."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()
              if not k.startswith("upscale")}
    outs = osvos_forward(leaves, x, gates=gates)
    if objective == "online":
        loss = online_objective(outs, gts)
    else:
        loss = parent_objective(outs, gts, side_weight)
    (loss * grad_scale).backward()
    grads = {k: v.grad for k, v in leaves.items() if v.grad is not None}
    return loss.detach(), [o.detach() for o in outs], grads


# --------------------------------------------------------------------------
# deterministic synthetic inputs / weights (SURVEY.md section 8d)
# --------------------------------------------------------------------------
def synthetic_frame(n: int, h: int, w: int, seed: int = 1234) -> Tuple[torch.Tensor, torch.Tensor]:
    """BGR 0..255 mean-subtracted frame + ~30 %-positive mask (dataloaders/davis_2016.py:101-102)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, h, w, generator=g) * 255.0 - torch.tensor(MEANVAL).view(1, 3, 1, 1)
    gt = (torch.rand(n, 1, h, w, generator=g) > 0.7).float()
    return x, gt


def he_params(seed: int = 0, dtype=torch.float32, include_upscale: bool = False) -> Dict[str, torch.Tensor]:
    """Seeded He-normal weights, N(0, 0.01) biases.  The reference's own
    pretrained=0 init (N(0, 0.001), networks/vgg_osvos.py:79) yields logits
    ~1e-12 and is useless for parity (SURVEY.md section 7 hard part 1)."""
    g = torch.Generator().manual_seed(seed)
    out: Dict[str, torch.Tensor] = {}
    for name, shape in param_shapes().items():
        if name.startswith("upscale"):
            if include_upscale:
                out[name] = interp_weight(shape[0], shape[2] // 2, dtype)
            continue
        if name.endswith(".weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            out[name] = (torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_in)).to(dtype)
        else:
            out[name] = (torch.randn(shape, generator=g) * 0.01).to(dtype)
    return out


def conv_flops(h: int, w: int, n: int = 1) -> float:
    """2*M*N*K over the 13 trunk + 4 side_prep 3x3 convs (BASELINE.md section 3)."""
    total = 0.0
    hh, ww = h, w
    for i, chans in enumerate(STAGE_CHANNELS):
        if i > 0:
            hh, ww = pooled_size(hh), pooled_size(ww)
        cin = STAGE_IN[i]
        for c in chans:
            total += 2.0 * n * hh * ww * c * 9 * cin
            cin = c
        if i > 0:
            total += 2.0 * n * hh * ww * SIDE_CHANNELS * 9 * cin
    return total


# --------------------------------------------------------------------------
# 8(f) rows: test-time output and the optimizer step
# --------------------------------------------------------------------------
def png_payload(fused_logits: np.ndarray) -> np.ndarray:
    """The 8-bit image the reference writes for one frame (train_online.py:182-187): ``pred = 1/(1+exp(-pred))``
    in numpy fp32, then ``scipy.misc.imsave`` -> ``toimage`` -> ``bytescale(data, high=255, low=0)`` with
    cmin/cmax = data.min()/data.max().  scipy.misc was removed from SciPy (absent in this image's scipy 1.18; the
    reference pins no version): this restates the published algorithm of scipy 1.0's ``scipy/misc/pilutil.py``
    ``bytescale``: ``cscale = cmax - cmin (1 if 0); scale = 255/cscale; bytedata = (data - cmin)*scale;
    (bytedata.clip(0, 255) + 0.5).astype(uint8)``.  PARITY UNPINNED for this function (the reference's own
    dependency cannot be run here); the anchor is the call site above.  fused_logits: [H, W] fp32."""
    x = np.asarray(fused_logits, dtype=np.float32)
    pred = (1.0 / (1.0 + np.exp(-x))).astype(np.float32)
    cmin, cmax = pred.min(), pred.max()
    cscale = np.float32(cmax - cmin)
    if cscale == 0:
        cscale = np.float32(1.0)
    scale = np.float32(255.0) / cscale
    bytedata = (pred - cmin) * scale
    return (bytedata.clip(0, 255) + 0.5).astype(np.uint8)


def sgd_momentum_step(p: torch.Tensor, g: torch.Tensor, buf, lr: float, wd: float, momentum: float):
    """torch.optim.SGD as the reference configures it (train_online.py:79-88: momentum 0.9, per-group weight_decay,
    dampening 0, no nesterov): g' = g + wd*p; buf = g' on the first step, momentum*buf + g' afterwards;
    p <- p - lr*buf.  Returns (p_new, buf_new).  fp64 inside so it can arbitrate between fp32 implementations."""
    p64, g64 = p.double(), g.double()
    gp = g64 + wd * p64
    b = gp if buf is None else momentum * buf.double() + gp
    return (p64 - lr * b).float(), b.float()


def _cv_rotation_matrix(center, angle_deg: float, scale: float) -> np.ndarray:
    """cv2.getRotationMatrix2D (OpenCV imgproc/imgwarp.cpp): alpha = s*cos, beta = s*sin (degrees, positive =
    counter-clockwise for a top-left origin)."""
    a = scale * math.cos(angle_deg * math.pi / 180.0)
    b = scale * math.sin(angle_deg * math.pi / 180.0)
    return np.array([[a, b, (1 - a) * center[0] - b * center[1]],
                     [-b, a, b * center[0] + (1 - a) * center[1]]], dtype=np.float64)


def scale_n_rotate(img: np.ndarray, rot: float, sc: float, flip: bool, nearest: bool) -> np.ndarray:
    """RandomHorizontalFlip then ScaleNRotate on one [C, H, W] fp32 array (reference
    dataloaders/custom_transforms.py:87-100 then :7-54; the reference holds HWC arrays at that point and ToTensor
    transposes afterwards - per-channel arithmetic is identical).  ``cv2.flip(tmp, 1)``; ``M =
    cv2.getRotationMatrix2D((w/2, h/2), rot, sc)``; ``cv2.warpAffine(tmp, M, (w, h), flags)`` with INTER_NEAREST for
    0/1 masks, INTER_CUBIC otherwise, BORDER_CONSTANT 0.
    cv2 is a third-party dependency the reference does not vendor or pin; this restates OpenCV's published algorithm
    and is PINNED against outputs of the reference's own transforms run with the image's cv2 4.13
    (tests/golden/make_golden_augment.py -> reference_augment.npz, tests/test_oracle.py::
    test_scale_n_rotate_matches_the_reference_transforms: masks bit-exact, cubic pixels to 9.2e-5 of 255-scale values).
    Algorithm (imgwarp.cpp WarpAffineInvoker + remap): the inverse matrix in fp64; source coordinates in fixed point with AB_BITS = 10,
    ``X = (cvRound((m1*y + m2)*1024) + round_delta + cvRound(m0*x*1024)) >> shift`` with round_delta 16 / shift 5
    (1/32-pixel positions) for cubic and 512 / 10 for nearest; cubic weights ``interpolateCubic`` with A = -0.75
    in fp32 at the 1/32 position, the 4x4 window anchored one pixel up-left; out-of-image taps read 0."""
    x = np.asarray(img, dtype=np.float32)
    c, h, w = x.shape
    if flip:
        x = x[:, :, ::-1]
    m = _cv_rotation_matrix((w / 2, h / 2), rot, sc)
    full = np.vstack([m, [0.0, 0.0, 1.0]])
    inv = np.linalg.inv(full)[:2]                      # == OpenCV's explicit 2x3 inversion up to fp64 rounding
    # OpenCV's own inversion, restated (keeps the same rounding as the library)
    d = m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]
    d = 1.0 / d if d != 0 else 0.0
    i00, i11 = m[1, 1] * d, m[0, 0] * d
    i01, i10 = -m[0, 1] * d, -m[1, 0] * d
    i02 = -i00 * m[0, 2] - i01 * m[1, 2]
    i12 = -i10 * m[0, 2] - i11 * m[1, 2]
    assert np.allclose(inv, [[i00, i01, i02], [i10, i11, i12]], rtol=1e-9, atol=1e-9)
    xs = np.arange(w, dtype=np.float64)
    ys = np.arange(h, dtype=np.float64)
    rd = 512 if nearest else 16
    X0 = np.rint((i01 * ys + i02) * 1024.0).astype(np.int64) + rd
    Y0 = np.rint((i11 * ys + i12) * 1024.0).astype(np.int64) + rd
    ad = np.rint(i00 * xs * 1024.0).astype(np.int64)
    bd = np.rint(i10 * xs * 1024.0).astype(np.int64)
    Xf = X0[:, None] + ad[None, :]
    Yf = Y0[:, None] + bd[None, :]
    out = np.zeros((c, h, w), dtype=np.float32)
    if nearest:
        sx, sy = Xf >> 10, Yf >> 10
        ok = (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
        out[:, ok] = x[:, sy[ok], sx[ok]]
        return out
    X, Y = Xf >> 5, Yf >> 5
    sx, sy = (X >> 5) - 1, (Y >> 5) - 1
    fx = ((X & 31).astype(np.float32) * np.float32(1.0 / 32.0))
    fy = ((Y & 31).astype(np.float32) * np.float32(1.0 / 32.0))

    def coeffs(t):
        a = np.float32(-0.75)
        one = np.float32(1.0)
        c0 = ((a * (t + one) - np.float32(5) * a) * (t + one) + np.float32(8) * a) * (t + one) - np.float32(4) * a
        c1 = ((a + np.float32(2)) * t - (a + np.float32(3))) * t * t + one
        u = one - t
        c2 = ((a + np.float32(2)) * u - (a + np.float32(3))) * u * u + one
        return [c0, c1, c2, one - c0 - c1 - c2]
    cx, cy = coeffs(fx), coeffs(fy)
    acc = np.zeros((c, h, w), dtype=np.float32)
    for ky in range(4):
        yy = sy + ky
        for kx in range(4):
            xx = sx + kx
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            wgt = (cy[ky] * cx[kx]).astype(np.float32)
            vals = x[:, np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
            acc += np.where(ok[None], vals * wgt[None], np.float32(0)).astype(np.float32)
    return acc

"""OSVOS network with the reference's module surface and a native H100 forward.

Mirrors networks/vgg_osvos.py of the reference: same constructor
(``OSVOS(pretrained=0|1|2)``, :17), same parameter containers ``stages``,
``side_prep``, ``score_dsn``, ``upscale``, ``upscale_``, ``fuse`` (:48-54) and
therefore the same 52-tensor state_dict, same ``forward(x) -> list of 5 logit
maps`` (:59-74).  The containers only hold parameters: ``forward`` never calls
them, it hands the tensors to the CUDA engine (``..engine``).
"""
import math
import os

import numpy as np
import torch
import torch.nn as nn

from ..engine import OSVOSEngine
from ..layers.osvos_layers import bilinear_deconv_weight

# (has_pool, out_channels...) per stage, networks/vgg_osvos.py:19-24 of the reference
_STAGES = ((False, 64, 64), (True, 128, 128), (True, 256, 256, 256), (True, 512, 512, 512), (True, 512, 512, 512))
_SIDE = 16


def _make_stage(has_pool, cin, widths):
    mods = [nn.MaxPool2d(kernel_size=2, stride=2, ceil_mode=True)] if has_pool else []
    for cout in widths:
        mods += [nn.Conv2d(cin, cout, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
        cin = cout
    return nn.Sequential(*mods), cin


class OSVOS(nn.Module):
    """Drop-in for the reference ``OSVOS`` module.

    Extra keywords (not in the reference): ``precision`` = "exact" (default; split
    bf16, three tensor-core passes, fp32-class results) or "fast" (one bf16 pass);
    ``learn_upsampling`` (default False, also a plain attribute that may be set after
    load_state_dict): backward writes the gradients of the eight deconvolution weights
    (upscale / upscale_), as the reference's autograd does.  Deconvolution weights other
    than interp_surgery's bilinear taps run with or without it (DESIGN.md §20).
    """

    def __init__(self, pretrained=1, precision="exact", verbose=True, learn_upsampling=False):
        super().__init__()
        if verbose:
            print("Constructing OSVOS architecture..")
        stages, side_prep, score_dsn = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        upscale, upscale_ = nn.ModuleList(), nn.ModuleList()
        cin = 3
        for i, (has_pool, *widths) in enumerate(_STAGES):
            stage, cin = _make_stage(has_pool, cin, widths)
            stages.append(stage)
            if i > 0:
                side_prep.append(nn.Conv2d(cin, _SIDE, kernel_size=3, padding=1))
                score_dsn.append(nn.Conv2d(_SIDE, 1, kernel_size=1, padding=0))
                upscale_.append(nn.ConvTranspose2d(1, 1, kernel_size=2 ** (1 + i), stride=2 ** i, bias=False))
                upscale.append(nn.ConvTranspose2d(_SIDE, _SIDE, kernel_size=2 ** (1 + i), stride=2 ** i, bias=False))
        # same registration order as the reference (:48-54) so state_dict / parameters() order match
        self.upscale = upscale
        self.upscale_ = upscale_
        self.stages = stages
        self.side_prep = side_prep
        self.score_dsn = score_dsn
        self.fuse = nn.Conv2d(4 * _SIDE, 1, kernel_size=1, padding=0)
        if verbose:
            print("Initializing weights..")
        self._initialize_weights(pretrained, verbose)
        self.precision = precision
        self.learn_upsampling = bool(learn_upsampling)
        self._engine = OSVOSEngine(self)

    # ------------------------------------------------------------------ forward
    def forward(self, x):
        return self._engine.forward(x)

    def forward_objective(self, x, gts, loss_weights=(0.0, 0.0, 0.0, 0.0, 1.0), size_average=False, batch_average=True,
                          void=False):
        """Extension (not in the reference): forward + the weighted sum of the five class-balanced BCE losses as ONE
        autograd node whose tail (upsample + crop + fuse + loss) is a single kernel forward and a single kernel
        backward.  Equivalent to
            outs = net(x); total = sum(w_k * class_balanced_cross_entropy_loss(outs[k], gts, size_average, batch_average))
        with loss_weights = (0,0,0,0,1) for the online objective (train_online.py:127) and (s,s,s,s,1),
        s = 1 - epoch/nEpochs, for the parent objective (train_parent.py:143-147).
        ``void``: gts < 0 marks void pixels, which the losses leave out (class_balanced_cross_entropy_loss(..., void=True);
        not with size_average or learn_upsampling).
        -> (outs: list of 5 logit maps, detached; total: 0-dim loss to call .backward() on; per_map: [5] losses)."""
        return self._engine.forward_objective(x, gts, loss_weights, size_average, batch_average, void)

    # ------------------------------------------------------------- initialisation
    def _initialize_weights(self, pretrained, verbose=True):
        """Reference init (:76-125): conv ~ N(0, 1e-3), zero bias; deconvs = fixed bilinear taps;
        then optionally VGG-16 weights from vgg_pytorch.pth (1) or vgg_caffe.mat (2)."""
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, 0.0, 0.001)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.ConvTranspose2d):
                with torch.no_grad():
                    m.weight.copy_(bilinear_deconv_weight(m.weight.shape[0], m.weight.shape[1], m.weight.shape[2]))
        if pretrained == 1:
            self._load_torchvision_vgg(verbose)
        elif pretrained == 2:
            self._load_caffe_vgg(verbose)

    def trunk_convs(self):
        """The 13 trunk convs grouped by stage (2, 2, 3, 3, 3), in VGG-16 order."""
        return [[m for m in stage if isinstance(m, nn.Conv2d)] for stage in self.stages]

    def _load_torchvision_vgg(self, verbose):
        from mypath import Path  # same config hook as the reference (:13,99)
        if verbose:
            print("Loading weights from PyTorch VGG")
        sd = torch.load(os.path.join(Path.models_dir(), "vgg_pytorch.pth"), map_location="cpu")
        feats = sorted({int(k.split(".")[1]) for k in sd if k.startswith("features.") and k.endswith(".weight")})
        convs = [c for stage in self.trunk_convs() for c in stage]
        assert len(feats) >= len(convs)
        with torch.no_grad():
            for conv, idx in zip(convs, feats):
                conv.weight.copy_(sd[f"features.{idx}.weight"])
                conv.bias.copy_(sd[f"features.{idx}.bias"])

    def _load_caffe_vgg(self, verbose):
        import scipy.io
        from mypath import Path
        if verbose:
            print("Loading weights from Caffe VGG")
        mat = scipy.io.loadmat(os.path.join(Path.models_dir(), "vgg_caffe.mat"))
        with torch.no_grad():
            for k, conv in enumerate(c for stage in self.trunk_convs() for c in stage):
                w = torch.from_numpy(np.ascontiguousarray(mat["weights"][0][k].transpose()))
                b = torch.from_numpy(np.ascontiguousarray(mat["biases"][0][k][:, 0]))
                assert conv.weight.shape == w.shape and conv.bias.shape == b.shape  # reference :119,123
                conv.weight.copy_(w)
                conv.bias.copy_(b)


def he_init_(net, seed=0):
    """Seeded He-normal weights (benchmarks / tests; the stock N(0,1e-3) init gives ~1e-12 logits)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if name.startswith("upscale"):
                continue
            if name.endswith("weight"):
                fan_in = p.shape[1] * p.shape[2] * p.shape[3]
                p.copy_((torch.randn(p.shape, generator=g) * math.sqrt(2.0 / fan_in)).to(p.device))
            else:
                p.copy_((torch.randn(p.shape, generator=g) * 0.01).to(p.device))
    return net

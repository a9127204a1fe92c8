"""The halo convolution at shapes that give CTAs three tiles or more (ping-pong schedule: the CTA's tiles alternate between
the two consumer warpgroups, which share one operand ring) and an uneven number left over, so the second warpgroup's path
and the ring hand-off between the warpgroups are exercised.  132 SMs: 544 tiles of 64 channels = 4.1 per CTA, 490 tiles
of 128 = 3.7, 336 tiles of 128 in two N blocks = 2.5.
Run on the GPU:  pytest -m gpu."""
import math

import pytest
import torch
import torch.nn.functional as F

from gpu_util import maxrel, rmsrel, split_round

pytestmark = pytest.mark.gpu

EXACT_TOL = 3e-5    # split-bf16 three-pass products: ~2^-16 relative operand error
FAST_TOL = 3e-2     # single bf16 pass

SHAPES = [
    # n, h, w, cin, cout
    (1, 256, 272, 64, 64),
    (1, 160, 392, 128, 128),
    (1, 64, 336, 128, 256),
]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


def _problem(n, h, w, cin, cout, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cin, h, w, generator=g) * 3.0
    wt = torch.randn(cout, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
    b = torch.randn(cout, generator=g) * 0.1
    return x, wt, b


@pytest.mark.parametrize("n,h,w,cin,cout", SHAPES)
def test_conv3x3_several_tiles_per_cta(dev, n, h, w, cin, cout):
    from osvos_pytorch_b200 import ops
    x, wt, b = _problem(n, h, w, cin, cout, 300 + h + cin)
    lin = F.conv2d(x.double(), wt.double(), b.double(), padding=1)
    wp = ops.pack_conv3x3_weights(wt.to(dev))
    for fast in (False, True):
        a = ops.nchw_to_act(x.to(dev), fast)
        for relu in (True, False):
            ref = lin.relu() if relu else lin
            y, yf, _ = ops.conv3x3(a, wp, b.to(dev), cout, relu=relu, fast=fast, out_act=True, out_f32=True)
            torch.cuda.synchronize()
            got_f32 = yf.permute(0, 3, 1, 2).cpu()
            tol = FAST_TOL if fast else EXACT_TOL
            assert maxrel(got_f32, ref) < tol, (fast, relu, maxrel(got_f32, ref), rmsrel(got_f32, ref))
            want_act = split_round(got_f32) if not fast else got_f32.to(torch.bfloat16).float()
            assert torch.equal(ops.act_to_nchw(y).cpu(), want_act), (fast, relu)
            # act output only: the lean epilogue of plain forward launches, bit-identical to the general one
            y_lean, _, _ = ops.conv3x3(a, wp, b.to(dev), cout, relu=relu, fast=fast, out_act=True)
            assert torch.equal(ops.act_to_nchw(y_lean).cpu(), want_act), (fast, relu)
            # CUDA-core cross-check on identical operands
            _, ys, _ = ops.conv3x3(a, wp, b.to(dev), cout, relu=relu, fast=fast, out_act=False, out_f32=True, simt=True)
            assert maxrel(got_f32, ys.permute(0, 3, 1, 2).cpu()) < 2e-5, (fast, relu)


@pytest.mark.parametrize("n,h,w,cin,cout", SHAPES[:2])
def test_conv3x3_relu_mask_several_tiles_per_cta(dev, n, h, w, cin, cout):
    """dgrad-style launch: fp32 output masked by the sign of another act, no bias."""
    from osvos_pytorch_b200 import ops
    x, wt, _ = _problem(n, h, w, cin, cout, 400 + h)
    g = torch.Generator().manual_seed(401 + h)
    mk = torch.randn(n, cout, h, w, generator=g)
    a = ops.nchw_to_act(x.to(dev))
    mact = ops.nchw_to_act(mk.clamp(min=0).to(dev))
    _, yf, _ = ops.conv3x3(a, ops.pack_conv3x3_weights(wt.to(dev)), None, cout, out_act=False, out_f32=True,
                           mask=mact.hi)
    ref = F.conv2d(x.double(), wt.double(), None, padding=1) * (mk > 0)
    assert maxrel(yf.permute(0, 3, 1, 2).cpu(), ref) < EXACT_TOL


@pytest.mark.parametrize("n,h,w,cin,cout", SHAPES[:2])
def test_conv3x3_fused_pool_and_bias_gradient_sum_several_tiles_per_cta(dev, n, h, w, cin, cout):
    """Epilogue fusions: MaxPool2d(2,2,ceil_mode) of the output and the per-channel output sum."""
    from osvos_pytorch_b200 import ops
    x, wt, b = _problem(n, h, w, cin, cout, 500 + h)
    a = ops.nchw_to_act(x.to(dev))
    wp = ops.pack_conv3x3_weights(wt.to(dev))
    colsum = torch.zeros(cout, device=dev)
    y, yp = ops.conv3x3(a, wp, b.to(dev), cout, relu=True, pool=True, colsum=colsum)
    full = ops.act_to_nchw(y).cpu()
    assert torch.equal(ops.act_to_nchw(yp).cpu(), F.max_pool2d(full, 2, 2, ceil_mode=True))   # selection: bit exact
    ref = F.conv2d(x.double(), wt.double(), b.double(), padding=1).relu()
    assert maxrel(full, ref) < EXACT_TOL
    assert maxrel(colsum.cpu(), ref.sum((0, 2, 3))) < 5e-5
    none, yp2 = ops.conv3x3(a, wp, b.to(dev), cout, relu=True, pool=True, out_act=False)
    assert none is None and torch.equal(ops.act_to_nchw(yp2).cpu(), ops.act_to_nchw(yp).cpu())

"""The engine's opt-in stage-1 path against the default path (and through it the oracle): separate conv1_1 and conv1_2
kernels (OSVOS_FUSE_STAGE1=0, the default) and the fused stage-1 kernel (OSVOS_FUSE_STAGE1=1).

The engine reads the switch on every eager pass, so one process can flip it; CUDA graphs are off for the comparison.  The
fused kernel sums conv1_1 in another fp32 order, so the outputs agree within float reassociation noise.
"""
import os

import pytest
import torch

from oracle import osvos_oracle as oc
from gpu_util import maxrel

pytestmark = [pytest.mark.gpu]

VARIANTS = [("OSVOS_FUSE_STAGE1", "0", 1e-4), ("OSVOS_FUSE_STAGE1", "1", 1e-4)]


@pytest.fixture(scope="module")
def net():
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS
    m = OSVOS(pretrained=0, verbose=False)
    m.load_state_dict(oc.he_params(seed=0), strict=False)
    m = m.cuda()
    m._engine.use_cuda_graph = False
    return m


@pytest.mark.parametrize("var,value,tol", VARIANTS)
@pytest.mark.parametrize("n,h,w", [(1, 240, 427), (2, 33, 45), (1, 480, 854)])
def test_variant_forward_matches_default(net, monkeypatch, var, value, tol, n, h, w):
    net.eval()
    x, _ = oc.synthetic_frame(n, h, w, 77)
    x = x.cuda()
    monkeypatch.delenv(var, raising=False)
    with torch.no_grad():
        ref = [o.clone() for o in net(x)]
        monkeypatch.setenv(var, value)
        got = [o.clone() for o in net(x)]
    for i, (g, r) in enumerate(zip(got, ref)):
        err = maxrel(g, r)
        print(f"{var}={value} {n}x{h}x{w} out{i}: max-rel difference to the default path {err:.2e}")
        assert err <= tol


@pytest.mark.parametrize("var,value,tol", VARIANTS)
def test_variant_backward_matches_default(net, monkeypatch, var, value, tol):
    """fwd + online loss + bwd at 240x427: dgrad (ReLU masks, fused bias sums), pooled and full-resolution outputs."""
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    net.train()
    x, gt = oc.synthetic_frame(1, 240, 427, 78)
    x, gt = x.cuda(), gt.cuda()

    def grads():
        net.zero_grad(set_to_none=True)
        loss = cbce(net(x)[-1], gt, size_average=False)
        loss.backward()
        torch.cuda.synchronize()
        return float(loss), {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
    monkeypatch.delenv(var, raising=False)
    loss0, g0 = grads()
    monkeypatch.setenv(var, value)
    loss1, g1 = grads()
    assert abs(loss1 - loss0) <= max(tol, 1e-6) * abs(loss0)
    for k in g0:
        rel = float((g1[k] - g0[k]).norm() / (g0[k].norm() + 1e-30))
        # atomics (wgrad workspace, fused bias sums) reorder between runs: 1e-5 of noise even for identical kernels; a
        # variant that changes the fp32 SUMMATION ORDER of the forward (tol > 0) moves a few ReLU masks / pool argmax
        # and with them the trunk gradients (6e-3 measured for the three-pass accumulator; the controlled comparison
        # is tests/test_gpu_backward.py::test_backward_with_injected_gates_*)
        assert rel <= (2e-2 if tol > 0 else 1e-4), f"{k}: {rel:.2e}"

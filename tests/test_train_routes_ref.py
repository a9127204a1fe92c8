"""Pins tests/train_routes_ref.py, the fp64 reference of a training step, before it judges the CUDA routes
(tests/test_gpu_train_routes.py).  CPU only."""
import pytest
import torch

from oracle import osvos_oracle as oc
from train_routes_ref import WEIGHTS, conv_outputs, expected_keys, gates_of, map_losses, reference_step, relnorm
from upsampling_ref import deconv_weights
from void_loss_ref import void_loss_torch


def _params(seed=0, general=False):
    p = oc.he_params(seed=seed, dtype=torch.float64, include_upscale=True)
    if general:
        p.update({k: v.double() for k, v in deconv_weights(seed + 100, "dense").items()})
    return p


def _frame(n, h, w, seed, void=False):
    x, gt = oc.synthetic_frame(n, h, w, seed)
    if void:
        g = torch.Generator().manual_seed(seed + 1)
        gt = torch.where(torch.rand(gt.shape, generator=g) < 0.2, torch.full_like(gt, -1.0), gt)
        if n > 1:
            gt[-1] = -1.0
    return x.double(), gt.double()


@pytest.mark.parametrize("weights", ["online", "parent", "mixed"])
@pytest.mark.parametrize("void", [False, True])
def test_own_gates_reproduce_the_ungated_oracle(weights, void):
    params = _params(1)
    x, gt = _frame(2, 40, 56, 3, void)
    gates = gates_of(conv_outputs(params, x))
    free = reference_step(params, x, gt, WEIGHTS[weights], 0.5, void=void, want_dx=True)
    gated = reference_step(params, x, gt, WEIGHTS[weights], 0.5, void=void, gates=gates, want_dx=True)
    assert abs(float(free["loss"]) - float(gated["loss"])) <= 1e-13 * abs(float(free["loss"]))
    assert free["grads"].keys() == gated["grads"].keys()
    for k, g in free["grads"].items():
        assert relnorm(gated["grads"][k], g) < 1e-12, k
    assert relnorm(gated["dx"], free["dx"]) < 1e-12
    if not void and weights != "mixed":              # and the oracle's own forward_backward on the same objective
        loss, _, og = oc.forward_backward(params, x, gt, "online" if weights == "online" else "parent",
                                          side_weight=WEIGHTS[weights][0], grad_scale=0.5)
        assert abs(0.5 * float(loss) - float(free["loss"])) <= 1e-13 * abs(float(free["loss"]))
        assert og.keys() == free["grads"].keys()
        for k, g in og.items():
            assert relnorm(free["grads"][k], g) < 1e-12, k


def test_void_loss_without_void_pixels_is_the_reference_loss():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(3, 1, 17, 9, generator=g, dtype=torch.float64) * 3
    y = (torch.rand(3, 1, 17, 9, generator=g) > 0.6).double()
    for divisor, ba in ((3.0, True), (1.0, False)):
        a = void_loss_torch(x, y, divisor)
        b = oc.class_balanced_cross_entropy_loss(x, y, size_average=False, batch_average=ba)
        assert abs(float(a) - float(b)) <= 1e-14 * abs(float(b))
    xr = x.clone().requires_grad_(True)
    void_loss_torch(xr, y, 3.0).backward()
    want = oc.class_balanced_cross_entropy_grad(x, y, size_average=False)
    assert relnorm(xr.grad, want) < 1e-14
    # the void route of map_losses leaves void pixels out and keeps the class balance of the others
    yv = y.clone()
    yv[0] = -1.0
    lv = map_losses([x], yv, void=True)[0]
    keep = yv >= 0
    pos = float((yv >= 0.5).sum())
    neg = float(keep.sum()) - pos
    sp = torch.nn.functional.softplus(x)
    want = (neg / (pos + neg) * (sp - x)[yv >= 0.5].sum() + pos / (pos + neg) * sp[(yv >= 0) & (yv < 0.5)].sum()) / 3
    assert abs(float(lv) - float(want)) <= 1e-13 * abs(float(want))


@pytest.mark.parametrize("weights", ["parent", "mixed"])
def test_literal_tail_on_bilinear_weights_is_the_folded_tail(weights):
    params = _params(2)                                  # he_params(include_upscale) writes interp_surgery's taps
    x, gt = _frame(2, 37, 61, 7)
    gates = gates_of(conv_outputs(params, x))
    folded = reference_step(params, x, gt, WEIGHTS[weights], gates=gates, want_dx=True)
    literal = reference_step(params, x, gt, WEIGHTS[weights], gates=gates, general=True, want_dx=True)
    assert relnorm(literal["per_map"], folded["per_map"]) < 1e-13
    assert folded["grads"].keys() == literal["grads"].keys()
    for k, g in folded["grads"].items():
        assert relnorm(literal["grads"][k], g) < 1e-12, k
    assert relnorm(literal["dx"], folded["dx"]) < 1e-12


@pytest.mark.parametrize("general,void", [(False, False), (False, True), (True, False)])
def test_gated_gradients_match_central_differences(general, void):
    """On a gated 17x9 frame (stage 5 is 2x1) the network is a polynomial in its weights: central differences of the
    fp64 objective match the fp64 gradients for a sample of entries of every parameter."""
    params = _params(3, general)
    x, gt = _frame(2, 17, 9, 11, void)
    weights = (0.5, 0.7, 0.3, 0.9, 1.0)
    gates = gates_of(conv_outputs(params, x))
    ref = reference_step(params, x, gt, weights, void=void, gates=gates, general=general, learn_upsampling=general,
                         want_dx=True)
    assert ref["grads"].keys() == expected_keys(weights, general, general)

    def objective(p, xx=x):
        with torch.no_grad():
            from train_routes_ref import literal_forward
            outs = literal_forward(p, xx, gates) if general else oc.osvos_forward(p, xx, gates=gates)
            return sum(wk * lk for wk, lk in zip(weights, map_losses(outs, gt, void)))
    g = torch.Generator().manual_seed(13)
    for name, grad in ref["grads"].items():
        flat = params[name].view(-1)
        scale = float(grad.abs().max())
        picks = {int(grad.abs().view(-1).argmax())} | {int(i) for i in torch.randint(flat.numel(), (3,), generator=g)}
        for i in picks:
            h = 1e-4 * max(abs(float(flat[i])), 0.05)
            old = float(flat[i])
            flat[i] = old + h
            up = float(objective(params))
            flat[i] = old - h
            down = float(objective(params))
            flat[i] = old
            fd = (up - down) / (2 * h)
            assert abs(fd - float(grad.view(-1)[i])) <= 1e-6 * scale + 1e-10, (name, i, fd, float(grad.view(-1)[i]))
    # the input gradient at a few pixels
    for i in torch.randint(x.numel(), (4,), generator=g).tolist():
        xv = x.clone().view(-1)
        xv[i] += 1e-4
        up = float(objective(params, xv.view(x.shape)))
        xv[i] -= 2e-4
        down = float(objective(params, xv.view(x.shape)))
        fd = (up - down) / 2e-4
        assert abs(fd - float(ref["dx"].view(-1)[i])) <= 1e-6 * float(ref["dx"].abs().max()) + 1e-10, i


@pytest.mark.parametrize("general", [False, True])
@pytest.mark.parametrize("weights", ["online", "parent", "mixed"])
def test_gradient_keys_are_the_expected_ones(weights, general):
    params = _params(4, general)
    x, gt = _frame(1, 17, 9, 17)
    ref = reference_step(params, x, gt, WEIGHTS[weights], general=general, learn_upsampling=general)
    assert set(ref["grads"]) == expected_keys(WEIGHTS[weights], general, general)
    if general:                                          # fixed deconvolution weights receive no gradient
        fixed = reference_step(params, x, gt, WEIGHTS[weights], general=True, learn_upsampling=False)
        assert set(fixed["grads"]) == expected_keys(WEIGHTS[weights], True, False)
        assert not any(k.startswith("upscale") for k in fixed["grads"])
    for k in ref["grads"]:
        assert float(ref["grads"][k].abs().max()) > 0, k

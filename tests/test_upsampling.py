"""CPU checks of the general deconvolution path's arithmetic (DESIGN.md §20): the literal tail pinned to the reference's
own module (tests/golden/reference_upsampling.npz, made by tests/golden/make_golden_upsampling.py), and the V / H
algebra the kernels implement, in float64 against autograd of the literal form."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import osvos_oracle as oc
from upsampling_ref import KINDS, deconv_weights, fold_v, literal_forward, literal_forward_backward, tail_by_taps

HERE = os.path.dirname(os.path.abspath(__file__))
FWD_CASES = {"48x70": (1, 48, 70, 11), "33x45_n2": (2, 33, 45, 12)}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(HERE, "golden", "reference_upsampling.npz")))


def params_for(kind, dtype=torch.float64):
    p = oc.he_params(seed=0, include_upscale=True)
    p.update(deconv_weights(100, kind))
    return {k: v.to(dtype) for k, v in p.items()}


def test_weights_are_not_bilinear():
    for kind in KINDS:
        p = deconv_weights(100, kind)
        for i in range(4):
            assert not torch.equal(p[f"upscale.{i}.weight"], oc.interp_weight(16, 2 ** (i + 1)))
            assert not torch.equal(p[f"upscale_.{i}.weight"], oc.interp_weight(1, 2 ** (i + 1)))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("tag", sorted(FWD_CASES))
def test_literal_forward_matches_reference(golden, kind, tag):
    n, h, w, seed = FWD_CASES[tag]
    x, _ = oc.synthetic_frame(n, h, w, seed)
    with torch.no_grad():
        outs = literal_forward(params_for(kind), x.double())
    for i in range(5):
        ref = golden[f"{kind}.fwd_{tag}.out{i}"]
        err = np.abs(outs[i].numpy() - ref).max() / np.abs(ref).max()
        assert err < 1e-5, (i, err)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("objective", ["online", "parent"])
def test_literal_gradients_match_reference(golden, kind, objective):
    x, gt = oc.synthetic_frame(1, 48, 70, 21)
    loss, _, grads = literal_forward_backward(params_for(kind), x.double(), gt.double(), objective, 0.75)
    ref_loss = float(golden[f"{kind}.bwd.{objective}.loss"])
    assert abs(float(loss) - ref_loss) < 1e-5 * abs(ref_loss)
    none_ref = {k.split(".none.")[1] for k in golden if k.startswith(f"{kind}.bwd.{objective}.none.")}
    assert none_ref == set(params_for(kind)) - set(grads)
    assert len(grads) + len(none_ref) == len(oc.param_shapes()) == 52
    for name, g in grads.items():
        ref_norm = float(golden[f"{kind}.bwd.{objective}.norm.{name}"])
        assert abs(float(g.norm()) - ref_norm) <= 1e-4 * ref_norm, name
        idx = golden[f"{kind}.bwd.{objective}.idx.{name}"]
        val = golden[f"{kind}.bwd.{objective}.val.{name}"]
        np.testing.assert_allclose(g.flatten()[idx].numpy(), val, rtol=0, atol=1e-4 * ref_norm)
    for i in range(4):      # the deconvolutions take part: their gradients are pinned too
        assert f"upscale.{i}.weight" in grads
        assert (f"upscale_.{i}.weight" in grads) == (objective == "parent")


def test_v_and_h_identities_in_float64():
    """fused = b + sum_k sum_src V_k[t] . F_k(src) with V_k[t][ci] = sum_co f[16k+co] U_k[ci][co][t], and
    d U_k[ci][co][t] = f[16k+co] H_k[t][ci], d f[16k+co] = sum U_k[ci][co][t] H_k[t][ci] with H_k = dL/dV_k."""
    g = torch.Generator().manual_seed(4)
    n, h, w = 2, 9, 13
    p = deconv_weights(7, "dense")
    fw = torch.randn(64, generator=g, dtype=torch.float64)
    hk, wk = h, w
    gfused = torch.randn(n, 1, h, w, generator=g, dtype=torch.float64)
    for k in range(4):
        s = 2 ** (k + 1)
        hk, wk = (hk + 1) // 2, (wk + 1) // 2
        feat = torch.randn(n, 16, hk, wk, generator=g, dtype=torch.float64)
        pk = torch.randn(n, 1, hk, wk, generator=g, dtype=torch.float64)
        u = p[f"upscale.{k}.weight"].double().requires_grad_(True)
        a = p[f"upscale_.{k}.weight"].double()
        f = fw[16 * k:16 * k + 16].clone().requires_grad_(True)
        lit_side = oc.center_crop(F.conv_transpose2d(pk, a, stride=s), h, w)
        lit_fused = F.conv2d(oc.center_crop(F.conv_transpose2d(feat, u, stride=s), h, w), f.view(1, 16, 1, 1))
        v = fold_v(u.detach(), f.detach()).requires_grad_(True)
        side, fused = tail_by_taps(feat, pk, a.flatten(), v, s, h, w)
        assert float((side - lit_side).abs().max()) < 1e-12
        assert float((fused - lit_fused).abs().max()) < 1e-12
        (lit_fused * gfused).sum().backward()
        (fused * gfused).sum().backward()
        hmat = v.grad                                           # [T, 16]
        du = f.detach().view(1, 16, 1) * hmat.t().unsqueeze(1)  # [ci, co, t]
        assert float((u.grad.flatten(2) - du).abs().max()) < 1e-10
        df = torch.einsum("iot,ti->o", u.detach().flatten(2), hmat)
        assert float((f.grad - df).abs().max()) < 1e-10

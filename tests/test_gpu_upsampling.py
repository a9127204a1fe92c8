"""The general deconvolution path (csrc/tail_general.cu, DESIGN.md §20): forward, backward and the eight deconvolution
gradients with weights that are not interp_surgery's bilinear taps, against the reference's literal tail in float64."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import maxrel
from oracle import osvos_oracle as oc
from upsampling_ref import deconv_weights, literal_forward, literal_forward_backward

pytestmark = pytest.mark.gpu
GATED_TOL = 5e-4      # per-parameter gradient bound with the CUDA pass's ReLU masks / pool argmax injected into the oracle
GRAD_TOL_TINY = 4e-2  # ungated bound on tiny maps, as tests/test_gpu_backward.py (ReLU / argmax flips, not arithmetic)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_upsampling.npz")


def relnorm(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def make_net(kind="dense", learn=False, seed=0, bilinear=False, precision="exact"):
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS
    params = oc.he_params(seed=seed, include_upscale=True)
    if not bilinear:
        params.update(deconv_weights(seed + 100, kind))
    net = OSVOS(pretrained=0, verbose=False, precision=precision)
    net.load_state_dict(params)
    net.learn_upsampling = learn
    return net.cuda(), params


def literal64(params, x, gates=None):
    p64 = {k: v.double().cuda() for k, v in params.items()}
    with torch.no_grad():
        return [o.cpu() for o in literal_forward(p64, x.double().cuda(), gates)]


@pytest.mark.parametrize("n,h,w,kind", [(1, 48, 70, "noisy"), (2, 33, 45, "dense"), (1, 480, 854, "dense")])
def test_forward_matches_literal_tail(n, h, w, kind):
    net, params = make_net(kind)
    x, _ = oc.synthetic_frame(n, h, w, 7)
    assert net._engine.uses_general_tail()
    ref = literal64(params, x)
    with torch.no_grad():
        eager = net._engine.forward_inference(x.cuda())
        graphed = net(x.cuda())
        graphed2 = net(x.cuda())                      # replay
    for k in range(5):
        err = maxrel(eager[k], ref[k])
        assert err <= 1e-3, (k, err)
        band = 1e-3 * float(ref[k].abs().max())
        flips = (eager[k].cpu() > 0) != (ref[k] > 0)
        assert bool((ref[k][flips].abs() <= band).all()), k
        assert torch.equal(graphed[k], eager[k]) and torch.equal(graphed2[k], eager[k])


@pytest.mark.parametrize("n,h,w", [(1, 48, 70), (2, 33, 45), (1, 480, 854)])
def test_general_path_on_bilinear_weights_matches_folded_path(n, h, w):
    net, _ = make_net(bilinear=True)
    x, _ = oc.synthetic_frame(n, h, w, 9)
    with torch.no_grad():
        assert not net._engine.uses_general_tail()
        folded = net(x.cuda())
        net.learn_upsampling = True
        assert net._engine.uses_general_tail()
        general = net(x.cuda())
    for k in range(5):
        assert maxrel(general[k], folded[k]) <= 1e-4, k


def test_tail_kernels_are_the_adjoint():
    """tail_general_fwd / tail_general_bwd / upsampling_grads_finish against float64 conv_transpose2d autograd."""
    from osvos_pytorch_b200 import ops
    torch.manual_seed(3)
    n, h, w = 2, 37, 53
    dev = torch.device("cuda")
    net, params = make_net("dense")
    hk, wk, feats, ps = h, w, [], []
    for k in range(4):
        hk, wk = (hk + 1) // 2, (wk + 1) // 2
        feats.append(torch.randn(n, hk, wk, 16))
        ps.append(torch.randn(n, hk, wk, 1))
    pqs = [torch.cat([p, torch.zeros_like(p)], 3).contiguous().to(dev) for p in ps]
    table = net._engine._upsampling_table()
    fb = torch.tensor([0.3], device=dev)
    out, _ = ops.tail_general_fwd([f.to(dev) for f in feats], pqs, table, fb, n, h, w)
    # float64 literal tail on leaves
    lf = [f.double().permute(0, 3, 1, 2).requires_grad_(True) for f in feats]
    lp = [p.double().permute(0, 3, 1, 2).requires_grad_(True) for p in ps]
    u16 = [params[f"upscale.{k}.weight"].double().requires_grad_(True) for k in range(4)]
    u1 = [params[f"upscale_.{k}.weight"].double().requires_grad_(True) for k in range(4)]
    fw = params["fuse.weight"].double().requires_grad_(True)
    side, sides = [], []
    for k in range(4):
        s = 2 ** (k + 1)
        sides.append(oc.center_crop(F.conv_transpose2d(lf[k], u16[k], stride=s), h, w))
        side.append(oc.center_crop(F.conv_transpose2d(lp[k], u1[k], stride=s), h, w))
    fused = F.conv2d(torch.cat(sides, 1), fw) + 0.3
    ref = side + [fused]
    for k in range(5):
        assert maxrel(out[k], ref[k]) <= 1e-5, k
    grads = [torch.randn(n, 1, h, w, dtype=torch.float64) for _ in range(5)]
    torch.autograd.backward(ref, grads)
    sw = [torch.zeros(16, device=dev) for _ in range(4)]      # score_dsn weight 0: dF is the tail's adjoint alone
    dfs, reds, _ = ops.tail_general_bwd([f.to(dev) for f in feats], pqs, sw, table, n, h, w,
                                        grads=[g.float().to(dev) for g in grads])
    d_up = [torch.empty_like(net.upscale[k].weight) for k in range(4)]
    d_up1 = [torch.empty_like(net.upscale_[k].weight) for k in range(4)]
    d_fw = torch.empty(64, device=dev)
    ops.upsampling_grads_finish(reds, [l.weight for l in net.upscale], net.fuse.weight, d_up, d_up1, d_fw)
    for k in range(4):
        df = ops.act_to_nchw(dfs[k])
        assert float(df[:, 16:].abs().max()) == 0.0
        assert maxrel(df[:, :16], lf[k].grad) <= 3e-5, k
        assert maxrel(d_up[k], u16[k].grad) <= 3e-5, k
        assert maxrel(d_up1[k], u1[k].grad) <= 3e-5, k
    assert maxrel(d_fw, fw.grad.flatten()) <= 3e-5


def _gated(net, params, x, gt, objective, side_weight=0.5):
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    cap = {}
    net._engine.debug_capture = cap
    try:
        net.zero_grad()
        outs = net(x.cuda())
        if objective == "online":
            loss = cbce(outs[-1], gt.cuda(), size_average=False)
        else:
            ls = [cbce(o, gt.cuda(), size_average=False) for o in outs]
            loss = side_weight * sum(ls[:-1]) + ls[-1]
        loss.backward()
    finally:
        net._engine.debug_capture = None
    gates = oc.gates_from_activations([ops.act_to_nchw(a).cpu() for stage in cap["acts"] for a in stage])
    g64 = {"relu": [g.cuda() for g in gates["relu"]], "pool": [p.cuda() for p in gates["pool"]]}
    p64 = {k: v.double().cuda() for k, v in params.items()}
    ref_loss, _, ograds = literal_forward_backward(p64, x.double().cuda(), gt.double().cuda(), objective, side_weight,
                                                   gates=g64)
    return float(loss), float(ref_loss), {n: relnorm(p.grad, ograds[n]) for n, p in net.named_parameters()
                                          if n in ograds}


@pytest.mark.parametrize("n,h,w,objective", [(1, 40, 56, "online"), (2, 40, 56, "parent"), (1, 64, 96, "parent"),
                                             (1, 480, 854, "online")])
def test_gated_gradients_match_literal_tail(n, h, w, objective):
    net, params = make_net("dense", learn=True)
    x, gt = oc.synthetic_frame(n, h, w, 311)
    loss, ref_loss, errs = _gated(net, params, x, gt, objective)
    assert abs(loss - ref_loss) < 1e-4 * abs(ref_loss)
    for i in range(4):
        assert f"upscale.{i}.weight" in errs and (f"upscale_.{i}.weight" in errs) == (objective == "parent")
    worst = max(errs, key=errs.get)
    print(f"general tail, gated {objective} {n}x{h}x{w}: worst {errs[worst]:.2e} ({worst})")
    assert errs[worst] < GATED_TOL, (worst, errs[worst])


def test_upsampling_grads_only_with_the_flag():
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    x, gt = oc.synthetic_frame(1, 40, 56, 5)
    for bilinear in (True, False):
        net, _ = make_net(bilinear=bilinear)
        cbce(net(x.cuda())[-1], gt.cuda(), size_average=False).backward()
        assert all(p.grad is None for n, p in net.named_parameters() if n.startswith("upscale"))
        assert net.side_prep[0].weight.grad is not None
    grads = {}
    for upstream in (1.0, 2.0):              # scales with the upstream gradient ...
        net, _ = make_net(learn=True)
        (upstream * cbce(net(x.cuda())[-1], gt.cuda(), size_average=False)).backward()
        grads[upstream] = net.upscale[2].weight.grad.clone()
        (upstream * cbce(net(x.cuda())[-1], gt.cuda(), size_average=False)).backward()
        assert maxrel(net.upscale[2].weight.grad, 2 * grads[upstream]) <= 1e-5     # ... and accumulates
    assert maxrel(grads[2.0], 2 * grads[1.0]) <= 1e-5
    with pytest.raises(ValueError, match="learn_upsampling"):
        from osvos_pytorch_b200 import training
        training.make_optimizer(make_net()[0], "online", upsampling_lr=1e-3)


@pytest.mark.parametrize("objective", ["online", "parent"])
def test_objective_matches_reference_call_sequence(objective):
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    weights = (0.0,) * 4 + (1.0,) if objective == "online" else (0.5,) * 4 + (1.0,)
    x, gt = oc.synthetic_frame(2, 48, 70, 17)
    x, gt = x.cuda(), gt.cuda()
    res = {}
    for fused in (False, True):
        net, _ = make_net(learn=True)
        if fused:
            outs, total, _ = net.forward_objective(x, gt, weights)
        else:
            outs = net(x)
            total = sum(wk * cbce(o, gt, size_average=False) for wk, o in zip(weights, outs) if wk != 0.0)
        total.backward()
        res[fused] = (float(total), {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None})
    assert abs(res[True][0] - res[False][0]) <= 1e-5 * abs(res[False][0])
    assert res[True][1].keys() == res[False][1].keys()
    for n, g in res[False][1].items():
        assert relnorm(res[True][1][n], g) <= 1e-4, n


def test_graphed_train_step_and_fused_sgd_move_the_deconvolutions():
    from osvos_pytorch_b200 import training
    x, gt = oc.synthetic_frame(1, 48, 70, 23)
    sample = {"image": x.cuda(), "gt": gt.cuda()}
    weights = (0.5,) * 4 + (1.0,)
    eager, _ = make_net(learn=True)
    _, total, _ = eager.forward_objective(sample["image"], sample["gt"], weights)
    total.backward()
    net, _ = make_net(learn=True)
    step = training.GraphedTrainStep(net, weights, sample)
    step.graph.replay()
    for (n, p), q in zip(net.named_parameters(), eager.parameters()):
        assert relnorm(p.grad, q.grad) <= 1e-5, n
    # one optimizer step: FusedSGD against torch.optim.SGD, the deconvolution groups at a nonzero lr
    ref, _ = make_net(learn=True)
    for p, q in zip(ref.parameters(), net.parameters()):
        p.grad = q.grad.clone()
    before = net.upscale[1].weight.detach().clone()
    table = net._engine._upsampling_table().clone()
    training.make_optimizer(net, "parent", lr=1e-8, fused=True, upsampling_lr=1e-4).step()
    training.make_optimizer(ref, "parent", lr=1e-8, upsampling_lr=1e-4).step()
    assert not torch.equal(net.upscale[1].weight, before)
    for (n, p), q in zip(net.named_parameters(), ref.parameters()):
        assert float((p - q).abs().max()) <= 1e-6 * float(q.abs().max()) + 1e-9, n
    # the folded table follows the update, and the next forward equals a fresh net's with these weights
    from osvos_pytorch_b200 import ops
    now = net._engine._upsampling_table()
    assert not torch.equal(now, table)
    assert torch.equal(now, ops.upsampling_fold([l.weight for l in net.upscale], [l.weight for l in net.upscale_],
                                                net.fuse.weight))
    fresh, _ = make_net(learn=True)
    fresh.load_state_dict(net.state_dict())
    with torch.no_grad():
        a, b = net(sample["image"]), fresh(sample["image"])
    for k in range(5):
        assert maxrel(a[k], b[k]) <= 1e-5, k


def test_deterministic_runs_are_bit_identical():
    from osvos_pytorch_b200 import training
    x, gt = oc.synthetic_frame(2, 48, 70, 29)
    x, gt = x.cuda(), gt.cuda()
    runs = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            net, _ = make_net(learn=True)
            opt = training.make_optimizer(net, "parent", lr=1e-8, upsampling_lr=1e-6)
            seen = []
            for _ in range(3):
                _, total, _ = net.forward_objective(x, gt, (0.5,) * 4 + (1.0,))
                total.backward()
                seen += [total.detach().clone()] + [p.grad.clone() for p in net.parameters()]
                opt.step()
                opt.zero_grad()
            runs.append(seen + [p.detach().clone() for p in net.parameters()])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(bool(torch.isfinite(a).all()) for a in runs[0])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_online_finetune_graphed_fused_equals_eager():
    """online_finetune's default path (graphed step with external packed layouts + FusedSGD) on the general tail over
    several optimizer steps: side_prep's packed layouts must follow every update (FusedSGD re-emits them), so the
    trajectory equals the eager loop with torch.optim.SGD, and the layouts in the cache equal a fresh pack."""
    from osvos_pytorch_b200 import ops, training
    x, gt = oc.synthetic_frame(1, 40, 56, 11)
    sample = {"image": x.cuda(), "gt": gt.cuda()}
    hist, nets = {}, {}
    init = {n: p.detach().clone() for n, p in make_net("dense", learn=True, seed=1)[0].named_parameters()}
    for graphed in (False, True):
        net, _ = make_net("dense", learn=True, seed=1)
        with torch.no_grad():
            for m in list(net.side_prep) + [net.fuse]:
                m.weight.mul_(0.1)
        hist[graphed] = training.online_finetune(net, lambda it: sample, 30, n_ave_grad=5, lr=1e-7, log_every=5,
                                                 log=lambda s: None, use_graph=graphed, fused_optimizer=graphed,
                                                 upsampling_lr=1e-5)
        nets[graphed] = net
    net = nets[True]
    for i, sp in enumerate(net.side_prep):
        for flip in (False, True):
            cached = net._engine._packed_layouts[(sp, flip)][1]
            assert torch.equal(cached, ops.pack_conv3x3_weights(sp.weight, flip, 64)), (i, flip)
    for a, b in zip(hist[False], hist[True]):
        assert abs(a - b) <= 3e-4 * abs(a), (hist[False], hist[True])
    for (n, p), q in zip(nets[True].named_parameters(), nets[False].parameters()):
        step = float((q.detach() - init[n]).double().norm())
        # the online objective (fused map only) reaches neither score_dsn nor upscale_
        assert (step > 0) != n.startswith(("score_dsn", "upscale_")), n
        if step > 0:
            assert float((p.detach() - q.detach()).double().norm()) <= 5e-2 * step, n


def test_sequence_segmenter_with_general_weights():
    """SequenceSegmenter (graphed, bytescale and logits) on general weights: the eager forward's maps and bytes."""
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net, _ = make_net("dense")
    frames = [oc.synthetic_frame(1, 33, 45, 40 + i)[0] for i in range(5)]
    with torch.no_grad():
        want = [net._engine.forward_inference(f.cuda())[-1] for f in frames]
    got = [r.clone() for r in SequenceSegmenter(net, output="logits")(frames)]
    for a, b in zip(got, want):
        assert torch.equal(a.cuda(), b)
    got = [r.clone() for r in SequenceSegmenter(net, output="bytescale")(frames)]
    for a, b in zip(got, want):
        assert torch.equal(a.cuda(), ops.logits_to_u8(b, "bytescale"))


@pytest.mark.parametrize("kind", ["noisy", "dense"])
def test_forward_and_gradients_match_reference_fixture(kind):
    """Against the reference module's own outputs and gradients (tests/golden/make_golden_upsampling.py)."""
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    golden = dict(np.load(GOLDEN))
    net, params = make_net(kind, learn=True)
    for tag, (n, h, w, seed) in {"48x70": (1, 48, 70, 11), "33x45_n2": (2, 33, 45, 12)}.items():
        x, _ = oc.synthetic_frame(n, h, w, seed)
        with torch.no_grad():
            outs = net(x.cuda())
        for i in range(5):
            ref = torch.from_numpy(golden[f"{kind}.fwd_{tag}.out{i}"])
            assert maxrel(outs[i], ref) <= 1e-3, (tag, i)
            flips = (outs[i].cpu() > 0) != (ref > 0)
            assert bool((ref[flips].abs() <= 1e-3 * float(ref.abs().max())).all()), (tag, i)
    x, gt = oc.synthetic_frame(1, 48, 70, 21)
    for obj in ("online", "parent"):
        net.zero_grad()
        outs = net(x.cuda())
        if obj == "online":
            loss = cbce(outs[-1], gt.cuda(), size_average=False)
        else:
            ls = [cbce(o, gt.cuda(), size_average=False) for o in outs]
            loss = 0.75 * sum(ls[:-1]) + ls[-1]
        loss.backward()
        ref_loss = float(golden[f"{kind}.bwd.{obj}.loss"])
        assert abs(float(loss) - ref_loss) < 1e-4 * abs(ref_loss)
        for name, p in net.named_parameters():
            if f"{kind}.bwd.{obj}.none.{name}" in golden:
                assert p.grad is None, name
                continue
            assert p.grad is not None, name
            ref_norm = float(golden[f"{kind}.bwd.{obj}.norm.{name}"])
            assert abs(float(p.grad.double().norm()) - ref_norm) < GRAD_TOL_TINY * ref_norm, (obj, name)
            idx = torch.from_numpy(golden[f"{kind}.bwd.{obj}.idx.{name}"])
            got = p.grad.detach().double().flatten().cpu()[idx].numpy()
            val = golden[f"{kind}.bwd.{obj}.val.{name}"]
            bound = 3 * GRAD_TOL_TINY * max(np.abs(val).max(), ref_norm / math.sqrt(p.numel()))
            assert np.abs(got - val).max() < bound, (obj, name)

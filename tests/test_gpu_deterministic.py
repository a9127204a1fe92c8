"""torch.use_deterministic_algorithms(True): every float reduction of the training path takes its fixed-order form
(OSVOS_FLAG_DETERMINISTIC, DESIGN.md §16).  Two runs give bit-identical results; the results agree with the default
(atomic) kernels within fp32 reassociation and with fp64 references within the per-kernel tolerances."""
import pytest
import torch
import torch.nn.functional as F

from oracle import osvos_oracle as oc
from gpu_util import maxrel

pytestmark = pytest.mark.gpu


@pytest.fixture
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _net(seed=0):
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS
    m = OSVOS(pretrained=0, verbose=False)
    m.load_state_dict(oc.he_params(seed=seed), strict=False)
    return m.cuda().train()


def _same(a, b):
    return torch.equal(a, b)


# conv1_2 at 480x854 (tap rows, ~100 splits), batch 4 at an odd size, stage-4 / stage-5 shapes (tap groups, many tiles)
@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 480, 854, 64, 64), (4, 67, 93, 128, 128), (4, 67, 93, 64, 128),
                                            (1, 60, 107, 512, 512), (1, 30, 54, 512, 512)])
@pytest.mark.parametrize("fast", [False, True])
def test_wgrad_two_calls_bit_identical(deterministic, n, h, w, cin, cout, fast):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(h * w + cin + cout)
    x = torch.randn(n, cin, h, w, generator=g)
    dz = torch.randn(n, cout, h, w, generator=g) * 0.1
    xa, dza = ops.nchw_to_act(x.cuda(), fast), ops.nchw_to_act(dz.cuda(), fast)
    a = ops.conv3x3_wgrad(xa, dza, cout, fast=fast, deterministic=True)
    b = ops.conv3x3_wgrad(xa, dza, cout, fast=fast, deterministic=True)
    assert _same(a, b)
    ref = ops.conv3x3_wgrad(xa, dza, cout, fast=fast)                     # default kernel: same products, atomics
    assert maxrel(a, ref) < 1e-5, maxrel(a, ref)
    # deferred form: per-split slices summed by the finish, accumulated onto an existing gradient
    dst = [torch.full((cout, cin, 3, 3), 0.25, device="cuda") for _ in range(2)]
    for d in dst:
        ws = torch.empty(ops.wgrad_workspace_floats(cout, cin, (n, h, w), True), device="cuda")
        it = ops.conv3x3_wgrad(xa, dza, cout, fast=fast, deferred_ws=ws, deterministic=True)
        it["dw"], it["accumulate"] = d, True
        ops.wgrad_finish([it])
    assert _same(dst[0], dst[1])
    assert maxrel(dst[0] - 0.25, a) < 1e-6
    if not fast and n * h * w * cin * cout < 2e9:
        wt = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, requires_grad=True)
        F.conv2d(xa_ref(xa), wt, None, padding=1).backward(xa_ref(dza))
        assert maxrel(a, wt.grad) < 3e-5, maxrel(a, wt.grad)


def xa_ref(act):
    from osvos_pytorch_b200 import ops
    return ops.act_to_nchw(act).double().cpu()


def test_deterministic_wgrad_workspace_figures():
    """The deterministic workspace of every trunk layer at 480x854, batch 1 (printed; DESIGN.md §16 quotes them)."""
    from osvos_pytorch_b200 import _native as nat
    lib = nat.load()
    layers = [(64, 64, 1), (64, 128, 2), (128, 128, 2), (128, 256, 4), (256, 256, 4), (256, 256, 4), (256, 512, 8),
              (512, 512, 8), (512, 512, 8), (512, 512, 16), (512, 512, 16), (512, 512, 16)]
    total = 0
    for cin, cout, s in layers:
        h, w = -(-480 // s), -(-854 // s)
        nb = lib.osvos_wgrad_workspace_bytes(1, h, w, cin, cout, nat.FLAG_DETERMINISTIC)
        assert nb == lib.osvos_wgrad_deterministic_splits(1, h, w, cin, cout) * lib.osvos_wgrad_workspace_bytes(1, h, w, cin,
                                                                                                              cout, 0)
        total += nb
        print(f"{cin}->{cout} at {h}x{w}: {lib.osvos_wgrad_deterministic_splits(1, h, w, cin, cout)} splits, "
              f"{nb / 2**20:.1f} MiB")
    print(f"total {total / 2**20:.1f} MiB")
    assert total < 1 << 30


def _backward(net, x, gt, objective, direct):
    """Gradients of every parameter after one fwd+bwd (plain mode: a fixed linear functional of the five maps)."""
    for p in net.parameters():
        p.grad = torch.full_like(p, 0.5) if direct else None
    if objective:
        _, loss, _ = net.forward_objective(x, gt, [0.3, 0.3, 0.3, 0.3, 1.0])
    else:
        outs = net(x)
        loss = sum((o * gt).sum() * (k + 1) * 1e-3 for k, o in enumerate(outs))
    if direct:
        with net._engine.direct_grad_accumulation():
            loss.backward()
    else:
        loss.backward()
    return float(loss), {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("objective", [False, True])
@pytest.mark.parametrize("direct", [False, True])
def test_whole_backward_bit_identical(objective, direct):
    net = _net(0)
    x, gt = oc.synthetic_frame(2, 64, 96, 77)
    x, gt = x.cuda(), gt.cuda()
    ref_loss, ref = _backward(net, x, gt, objective, direct)          # default (atomic) kernels
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_backward(net, x, gt, objective, direct) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(prev)
    (l0, g0), (l1, g1) = runs
    assert l0 == l1 and abs(l0 - ref_loss) <= 1e-5 * abs(ref_loss)
    assert g0.keys() == g1.keys() == ref.keys()
    for n in g0:
        assert _same(g0[n], g1[n]), n
        err = float((g0[n] - ref[n]).double().norm() / ref[n].double().norm().clamp(min=1e-30))
        assert err < 5e-4, (n, err)


def _finetune(h, w, iters=50):
    from osvos_pytorch_b200 import training
    net = _net(1)
    with torch.no_grad():
        for m in list(net.side_prep) + [net.fuse]:
            m.weight.mul_(0.1)
    x, gt = oc.synthetic_frame(1, h, w, 11)
    sample = {"image": x.cuda(), "gt": gt.cuda()}
    hist = training.online_finetune(net, lambda it: sample, iters, n_ave_grad=5, lr=1e-9, log_every=5,
                                    log=lambda s: None, use_graph=True, fused_optimizer=True)
    return hist, {k: v.clone() for k, v in net.state_dict().items()}


@pytest.mark.parametrize("h,w", [(40, 56), (480, 854)])
def test_online_finetune_runs_are_identical(deterministic, h, w):
    h0, s0 = _finetune(h, w)
    h1, s1 = _finetune(h, w)
    assert h0 == h1
    for k in s0:
        assert _same(s0[k], s1[k]), k


def test_parent_epoch_runs_are_identical(deterministic):
    from osvos_pytorch_b200 import training
    from osvos_pytorch_b200.parallel import GradientBucket, trainable_parameters
    out = []
    for _ in range(2):
        net = _net(2)
        opt = training.make_optimizer(net, "parent", lr=1e-9)
        bucket = GradientBucket(trainable_parameters(net))
        batches = [training.synthetic_batch(2, 64, 96, seed, "cuda") for seed in range(6)]
        totals = training.parent_epoch(net, opt, bucket, batches, 0, 240, n_ave_grad=2)
        out.append((totals.clone(), {k: v.clone() for k, v in net.state_dict().items()}))
    assert _same(out[0][0], out[1][0])
    for k in out[0][1]:
        assert _same(out[0][1][k], out[1][1][k]), k


def test_graphed_step_refuses_a_toggled_flag():
    from osvos_pytorch_b200 import training
    net = _net(3)
    x, gt = oc.synthetic_frame(1, 40, 56, 5)
    step = training.GraphedTrainStep(net, training.ONLINE_WEIGHTS, {"image": x.cuda(), "gt": gt.cuda()})
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not prev)
    try:
        with pytest.raises(RuntimeError, match="captured with torch.use_deterministic_algorithms"):
            step()
    finally:
        torch.use_deterministic_algorithms(prev)
    step()                                                   # the capture mode replays


def test_reference_style_loss_is_deterministic(deterministic):
    """class_balanced_cross_entropy_loss (osvos_cbce_fwd) adds its block sums in a fixed order under the flag."""
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    g = torch.Generator().manual_seed(4)
    x = (torch.randn(2, 1, 480, 854, generator=g) * 4).cuda()
    y = (torch.rand(2, 1, 480, 854, generator=g) > 0.7).float().cuda()
    a, b = cbce(x, y, size_average=False), cbce(x, y, size_average=False)
    assert _same(a, b)
    torch.use_deterministic_algorithms(False)
    ref = cbce(x, y, size_average=False)
    torch.use_deterministic_algorithms(True)
    assert abs(float(a) - float(ref)) <= 1e-6 * abs(float(ref))
    xr = x.double().cpu()
    yr = y.double().cpu()
    sp = torch.nn.functional.softplus(xr)
    pos = yr >= 0.5
    s_pos, s_neg = float((sp - xr)[pos].sum()), float(sp[~pos].sum())
    p, tot = float(pos.sum()), float(xr.numel())
    want = ((tot - p) / tot * s_pos + p / tot * s_neg) / x.shape[0]          # batch_average: divided by the batch
    assert abs(float(a) - want) <= 3e-5 * abs(want)

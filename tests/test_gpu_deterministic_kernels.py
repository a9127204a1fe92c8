"""Per-kernel checks of the deterministic forms (OSVOS_FLAG_DETERMINISTIC, DESIGN.md §16): two calls of each converted
entry point give bit-identical outputs, which equal the default (atomic) kernels' outputs within fp32 reassociation and
fp64 references within the per-kernel tolerance (3e-5)."""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import maxrel

pytestmark = pytest.mark.gpu


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def _act(t, fast=False):
    from osvos_pytorch_b200 import ops
    return ops.nchw_to_act(t.cuda(), fast)


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 40, 56, 128, 64), (2, 67, 93, 256, 128), (1, 240, 427, 128, 128),
                                            (1, 30, 54, 512, 512)])
@pytest.mark.parametrize("fast", [False, True])
def test_dgrad_column_sums(n, h, w, cin, cout, fast):
    """colsum of the dgrad epilogue: per-tile partial rows + ordered reduction."""
    from osvos_pytorch_b200 import ops
    x = _act(_rand((n, cin, h, w), 1, 0.1), fast)
    mask = _act(_rand((n, cout, h, w), 2), fast)
    wt = ops.pack_conv3x3_weights(_rand((cout, cin, 3, 3), 3, 0.05).cuda())
    sums = []
    for det in (True, True, False):
        cs = torch.zeros(cout, device="cuda")
        _, yf, _ = ops.conv3x3(x, wt, None, cout, fast=fast, mask=mask.hi, colsum=cs, out_f32=True, deterministic=det)
        sums.append(cs)
    assert torch.equal(sums[0], sums[1])
    assert maxrel(sums[0], sums[2]) < 1e-5, maxrel(sums[0], sums[2])
    assert maxrel(sums[0], yf.double().sum(dim=(0, 1, 2))) < 3e-5


@pytest.mark.parametrize("n,h,w,c", [(1, 40, 56, 64), (2, 67, 93, 128), (1, 120, 214, 256), (1, 31, 55, 512)])
@pytest.mark.parametrize("side", [False, True])
@pytest.mark.parametrize("pool", [True, False])
def test_unpool_mask_column_sums(n, h, w, c, side, pool):
    from osvos_pytorch_b200 import ops
    if not side and not pool:
        pytest.skip("without the side branch the call needs a pooling consumer")
    x = _act(_rand((n, c, h, w), 4))
    dpool = _act(_rand((n, c, (h + 1) // 2, (w + 1) // 2), 5, 0.1)) if pool else None
    dpq = _rand((n, h, w, 2), 6, 0.1).cuda() if side else None
    wfold = _rand((9, 2, c), 7, 0.1).cuda() if side else None
    outs = []
    for det in (True, True, False):
        cs = torch.zeros(c, device="cuda")
        dz = ops.unpool_mask(dpool, x, dpq=dpq, wfold=wfold, colsum=cs, deterministic=det)
        outs.append((cs, ops.act_to_nchw(dz)))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[2][1])   # dz itself is unchanged
    assert maxrel(outs[0][0], outs[2][0]) < 1e-5
    assert maxrel(outs[0][0], outs[0][1].double().sum(dim=(0, 2, 3))) < 3e-5


def test_side_g_and_s():
    """G/S of the four side scales: per-block partial rows + ordered reduction."""
    from osvos_pytorch_b200 import ops
    n, h, w = 2, 120, 214
    shapes = [(128, 1), (256, 2), (512, 4), (512, 8)]
    xs, dpqs = [], []
    for k, (c, s) in enumerate(shapes):
        hs, ws = -(-h // s), -(-w // s)
        xs.append(_act(_rand((n, c, hs, ws), 10 + k)))
        dpqs.append(_rand((n, hs, ws, 2), 20 + k, 0.1).cuda())
    res = []
    for det in (True, True, False):
        gs = [torch.zeros((ops.side_folded_wgrad_floats(c) + 3) // 4 * 4, device="cuda") for c, _ in shapes]
        ops.side_folded_wgrad_multi(xs, dpqs, gs, deterministic=det)
        res.append(gs)
    for k, (c, _) in enumerate(shapes):
        a, b, ref = res[0][k], res[1][k], res[2][k]
        assert torch.equal(a, b), k
        assert maxrel(a, ref) < 1e-5, (k, maxrel(a, ref))
        # S = sum of dpq (fp64), and one tap of G against its fp64 definition: G[4][o][c] = sum_px dpq[px][o] x[px][c]
        assert maxrel(a[18 * c:18 * c + 2], dpqs[k].double().sum(dim=(0, 1, 2))) < 3e-5
        xv = ops.act_to_nchw(xs[k]).double().permute(0, 2, 3, 1).reshape(-1, c)
        g4 = dpqs[k].double().reshape(-1, 2).t() @ xv
        assert maxrel(a[8 * c:10 * c].view(2, c), g4) < 3e-5, k


@pytest.mark.parametrize("n,h,w", [(1, 480, 854), (2, 67, 93)])
def test_conv1_1_backward(n, h, w):
    from osvos_pytorch_b200 import ops
    x = _rand((n, 3, h, w), 30, 50.0).cuda()
    dz = _act(_rand((n, 64, h, w), 31, 0.01))
    wt = _rand((64, 3, 3, 3), 32, 0.1).cuda()
    a, _ = ops.conv_first_bwd(x, dz, wt, False, deterministic=True)
    b, _ = ops.conv_first_bwd(x, dz, wt, False, deterministic=True)
    ref, _ = ops.conv_first_bwd(x, dz, wt, False)
    assert torch.equal(a, b)
    assert maxrel(a, ref) < 1e-5
    w64 = torch.zeros(64, 3, 3, 3, dtype=torch.float64, requires_grad=True)
    F.conv2d(x.double().cpu(), w64, None, padding=1).backward(ops.act_to_nchw(dz).double().cpu())
    assert maxrel(a, w64.grad) < 3e-5, maxrel(a, w64.grad)


@pytest.mark.parametrize("n,h,w", [(1, 480, 854), (3, 67, 93)])
def test_tail_forward_and_backward_with_the_loss(n, h, w):
    from osvos_pytorch_b200 import ops
    pqs, hk, wk = [], h, w
    for k in range(4):
        hk, wk = (hk + 1) // 2, (wk + 1) // 2
        pqs.append(_rand((n, hk, wk, 2), 40 + k, 3.0).cuda())
    fb = torch.tensor([0.3], device="cuda")
    label = (_rand((n, 1, h, w), 45) > 0.5).float().cuda()
    wts = [0.3, 0.3, 0.3, 0.3, 1.0]
    runs = []
    for det in (True, True, False):
        out, sums, losses = ops.tail_fwd(pqs, fb, n, h, w, label=label, loss_weights=wts, divisor=float(n),
                                         deterministic=det)
        dpq, fbg = ops.tail_loss_bwd(out, label, sums, wts, float(n), None, n, h, w, deterministic=det)
        plain = ops.tail_bwd([o.clone() for o in out], n, h, w, deterministic=det)
        runs.append((sums[:15].clone(), losses.clone(), dpq, fbg.clone(), plain))
    a, b, ref = runs
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[3], b[3])
    for k in range(4):
        assert torch.equal(a[2][k], b[2][k]) and torch.equal(a[4][k], b[4][k]), k
        assert maxrel(a[2][k], ref[2][k]) < 1e-5 and maxrel(a[4][k], ref[4][k]) < 1e-5, k
    assert maxrel(a[0], ref[0]) < 1e-9 and maxrel(a[1], ref[1]) < 1e-6
    assert abs(float(a[0][10]) - float((label >= 0.5).sum())) == 0.0      # the positive count is exact
    assert maxrel(a[3], ref[3]) < 1e-5


@pytest.mark.parametrize("numel", [1, 1000, 409920, 12 * 409920 + 3])
def test_sum_f32(numel):
    from osvos_pytorch_b200 import ops
    x = _rand((numel,), 50).cuda()
    a, b, ref = ops.sum_f32(x, deterministic=True), ops.sum_f32(x, deterministic=True), ops.sum_f32(x)
    assert torch.equal(a, b)
    want = float(x.double().sum())
    scale = float(x.abs().double().sum())
    assert abs(float(a) - want) <= 1e-6 * scale and abs(float(a) - float(ref)) <= 1e-6 * scale

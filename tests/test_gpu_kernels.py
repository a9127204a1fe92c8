"""Per-kernel parity tests of the CUDA path (through the C ABI) against CPU fp64 restatements.
Run on the GPU:  pytest -m gpu."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import osvos_oracle as oc
from gpu_util import maxrel, rmsrel, split_round

pytestmark = pytest.mark.gpu

EXACT_TOL = 3e-5    # split-bf16 three-pass products: ~2^-16 relative operand error
FAST_TOL = 3e-2     # single bf16 pass


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


def test_layout_round_trip(dev):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 64, 9, 7, generator=g) * 50
    y = ops.act_to_nchw(ops.nchw_to_act(x.to(dev))).cpu()
    assert torch.equal(y, split_round(x))
    assert maxrel(y, x) < 2e-5


@pytest.mark.parametrize("transpose_flip", [False, True])
def test_weight_packing(dev, transpose_flip):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(2)
    w = torch.randn(128, 64, 3, 3, generator=g)
    packed = ops.pack_conv3x3_weights(w.to(dev), transpose_flip).cpu().float()
    rows, cols = (64, 128) if transpose_flip else (128, 64)
    planes = packed.view(2, 9, rows, cols)
    got = planes[0] + planes[1]
    if transpose_flip:
        want = w.flip(2, 3).permute(2, 3, 1, 0).reshape(9, 64, 128)
    else:
        want = w.permute(2, 3, 0, 1).reshape(9, 128, 64)
    assert torch.equal(got, split_round(want))


CONV_CASES = [
    # n, h, w, cin, cout, relu
    (1, 16, 8, 64, 64, True),       # exactly one tile
    (1, 20, 13, 64, 64, True),      # ragged tile edges
    (2, 17, 9, 128, 128, False),    # batch, two K chunks
    (1, 33, 45, 64, 128, True),     # several tiles, n_block = 1 of 128
    (1, 9, 11, 256, 256, True),     # two N blocks, four K chunks
    (1, 3, 5, 512, 512, True),      # image smaller than the TMA box
]


def _conv_f32_case(dev, n, h, w, cin, cout, relu, fast, out_act):
    """Seeded conv problem through osvos_conv3x3 with an fp32 output, checked against fp64 and against the CUDA-core
    kernel on identical operands.  Returns (operands, act output or None, fp32 output as NCHW)."""
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(100 + h * w + cin)
    x = torch.randn(n, cin, h, w, generator=g) * 3.0
    wt = torch.randn(cout, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
    b = torch.randn(cout, generator=g) * 0.1
    ref = F.conv2d(x.double(), wt.double(), b.double(), padding=1)
    if relu:
        ref = ref.relu()
    a = ops.nchw_to_act(x.to(dev), fast)
    wp = ops.pack_conv3x3_weights(wt.to(dev))
    y, yf, _ = ops.conv3x3(a, wp, b.to(dev), cout, relu=relu, fast=fast, out_act=out_act, out_f32=True)
    torch.cuda.synchronize()
    got_f32 = yf.permute(0, 3, 1, 2).cpu()
    tol = FAST_TOL if fast else EXACT_TOL
    assert maxrel(got_f32, ref) < tol, (maxrel(got_f32, ref), rmsrel(got_f32, ref))
    _, ys, _ = ops.conv3x3(a, wp, b.to(dev), cout, relu=relu, fast=fast, out_act=False, out_f32=True, simt=True)
    assert maxrel(got_f32, ys.permute(0, 3, 1, 2).cpu()) < 2e-5
    return (a, wp, b.to(dev)), y, got_f32


@pytest.mark.parametrize("n,h,w,cin,cout,relu", CONV_CASES)
@pytest.mark.parametrize("fast", [False, True])
def test_conv3x3_tensor_core(dev, n, h, w, cin, cout, relu, fast):
    from osvos_pytorch_b200 import ops
    (a, wp, b), y, got_f32 = _conv_f32_case(dev, n, h, w, cin, cout, relu, fast, out_act=True)
    # the act output is the split rounding of the fp32 result
    want_act = split_round(got_f32) if not fast else got_f32.to(torch.bfloat16).float()
    assert torch.equal(ops.act_to_nchw(y).cpu(), want_act)
    # act output only: the lean epilogue of plain forward launches, bit-identical to the general one
    y_lean, _, _ = ops.conv3x3(a, wp, b, cout, relu=relu, fast=fast, out_act=True)
    assert torch.equal(y_lean.hi, y.hi)
    assert y.lo is None or torch.equal(y_lean.lo, y.lo)


@pytest.mark.parametrize("fast", [False, True])
def test_conv3x3_side_prep_fp32_output(dev, fast):
    """side_prep shape (16 outputs, no ReLU, side-branch kernel): fp32 features only; an act output is refused."""
    from osvos_pytorch_b200 import _native as nat, ops
    (a, wp, b), _, _ = _conv_f32_case(dev, 1, 30, 27, 128, 16, False, fast, out_act=False)
    with pytest.raises(nat.NativeLibraryError, match="invalid argument"):
        ops.conv3x3(a, wp, b, 16, fast=fast, out_act=True, out_f32=True)


def test_conv3x3_outputs_need_only_element_pair_alignment(dev):
    """The epilogue stores channel pairs (4-byte bf16x2 words, 8-byte float2), so output planes that start 4 / 8 bytes past
    a 32-byte boundary are valid and must give the same result as the allocator-aligned call."""
    from ctypes import byref
    from osvos_pytorch_b200 import _native as nat, ops
    n, h, w, cin, cout = 1, 20, 13, 64, 128
    g = torch.Generator().manual_seed(7)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
    b = (torch.randn(cout, generator=g) * 0.1).to(dev)
    a = ops.nchw_to_act(x.to(dev))
    wp = ops.pack_conv3x3_weights(wt.to(dev))
    y, yf, _ = ops.conv3x3(a, wp, b, cout, relu=True, out_act=True, out_f32=True)
    numel = n * h * w * cout
    hi = torch.zeros(numel + 2, dtype=torch.bfloat16, device=dev)      # planes at +4 bytes
    lo = torch.zeros(numel + 2, dtype=torch.bfloat16, device=dev)
    f32 = torch.zeros(numel + 2, dtype=torch.float32, device=dev)      # plane at +8 bytes
    args = nat.Conv3x3Args()
    args.x_hi, args.x_lo, args.w_packed, args.bias = a.hi.data_ptr(), a.lo.data_ptr(), wp.data_ptr(), b.data_ptr()
    args.y_hi, args.y_lo, args.y_f32 = hi[2:].data_ptr(), lo[2:].data_ptr(), f32[2:].data_ptr()
    args.n, args.h, args.w, args.cin, args.cout, args.flags = n, h, w, cin, cout, nat.FLAG_RELU
    nat.check(nat.load().osvos_conv3x3(byref(args), torch.cuda.current_stream().cuda_stream), "osvos_conv3x3")
    torch.cuda.synchronize()
    assert torch.equal(f32[2:].view(n, h, w, cout), yf)
    assert torch.equal(hi[2:].view(n, h, w, cout), y.hi) and torch.equal(lo[2:].view(n, h, w, cout), y.lo)


@pytest.mark.parametrize("n,h,w", [(1, 16, 8), (1, 33, 45), (2, 40, 56), (1, 5, 3), (1, 480, 854), (3, 97, 131)])
def test_stage1_fused_equals_conv1_1_then_conv1_2(dev, n, h, w):
    """osvos_stage1_fused (conv1_1 evaluated inside conv1_2's kernel on its halo patch) against the two-kernel route and
    the fp64 reference: full-resolution and pooled outputs, ragged tiles, frames smaller than a tile, batches."""
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(h * 7 + w)
    x = torch.rand(n, 3, h, w, generator=g) * 255.0 - 110.0
    w1 = torch.randn(64, 3, 3, 3, generator=g) * math.sqrt(2.0 / 27)
    b1 = torch.randn(64, generator=g) * 0.1
    w2 = torch.randn(64, 64, 3, 3, generator=g) * math.sqrt(2.0 / 576)
    b2 = torch.randn(64, generator=g) * 0.1
    a1 = ops.conv_first(x.to(dev), w1.to(dev), b1.to(dev), relu=True)
    w2p = ops.pack_conv3x3_weights(w2.to(dev))
    full0, pool0 = ops.conv3x3(a1, w2p, b2.to(dev), 64, relu=True, pool=True)
    full1, pool1 = ops.stage1_fused(x.to(dev), w1.to(dev), b1.to(dev), w2p, b2.to(dev), pool=True, out_act=True)
    _, pool2 = ops.stage1_fused(x.to(dev), w1.to(dev), b1.to(dev), w2p, b2.to(dev), pool=True, out_act=False)
    torch.cuda.synchronize()
    ref1 = F.conv2d(x.double(), w1.double(), b1.double(), padding=1).relu()
    ref = F.conv2d(ref1, w2.double(), b2.double(), padding=1).relu()
    got = ops.act_to_nchw(full1).cpu()
    assert maxrel(got, ref) < EXACT_TOL, maxrel(got, ref)
    assert maxrel(got, ops.act_to_nchw(full0).cpu()) < 2e-5
    want_pool = F.max_pool2d(got, 2, 2, ceil_mode=True)            # selection of the stored (split-rounded) values
    assert torch.equal(ops.act_to_nchw(pool1).cpu(), want_pool)
    assert torch.equal(ops.act_to_nchw(pool2).cpu(), want_pool)
    assert maxrel(ops.act_to_nchw(pool1).cpu(), ops.act_to_nchw(pool0).cpu()) < 2e-5


def test_side_branch_multi_fold_is_one_conv(dev):
    """side_prep (no ReLU) + score_dsn + fuse slice == ONE 3x3 conv C -> 2 (osvos_fold_side_weights_multi): same pq as the
    16-feature kernel with fused projections, to fp32 reassociation."""
    from osvos_pytorch_b200 import ops
    for n, h, w, cin in [(1, 30, 27, 128), (2, 17, 13, 256), (1, 60, 107, 512), (1, 5, 3, 512), (1, 120, 214, 128)]:
        g = torch.Generator().manual_seed(h + cin)
        x = torch.randn(n, cin, h, w, generator=g) * 3.0
        wt = torch.randn(16, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
        bs = torch.randn(16, generator=g) * 0.1
        proj = torch.randn(32, generator=g) * 0.3
        pb = torch.randn(1, generator=g)
        a = ops.nchw_to_act(x.to(dev))
        _, _, pq16 = ops.conv3x3(a, ops.pack_conv3x3_weights(wt.to(dev)), bs.to(dev), 16, out_act=False, proj_w=proj.to(dev),
                                 proj_b=pb.to(dev))
        (packed, bias2, _), = ops.fold_side_weights_multi([(wt.to(dev), bs.to(dev), proj.to(dev), pb.to(dev))],
                                                          want_f32=False)
        pq2 = ops.side_folded(a, packed, bias2)
        torch.cuda.synchronize()
        feat = F.conv2d(x.double(), wt.double(), bs.double(), padding=1)
        want_p = (feat * proj[:16].double().view(1, 16, 1, 1)).sum(1) + pb.double()
        want_q = (feat * proj[16:].double().view(1, 16, 1, 1)).sum(1)
        want = torch.stack([want_p, want_q], dim=-1)
        assert maxrel(pq2, want) < EXACT_TOL, (n, h, w, cin, maxrel(pq2, want))
        assert maxrel(pq2, pq16) < 2e-5, (n, h, w, cin, maxrel(pq2, pq16))
        # fast mode: one bf16 pass
        pqf = ops.side_folded(ops.nchw_to_act(x.to(dev), True), packed, bias2, fast=True)
        assert maxrel(pqf, want) < FAST_TOL


def test_side_branch_folded_multi_scale_launch(dev):
    """osvos_side_folded_multi: the folded side convs of several scales in one launch give bit-identical pq to one launch
    per scale (same tiles, same arithmetic; only the tile -> CTA assignment differs), in any order of the scales."""
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(21)
    shapes = [(1, 30, 53, 128), (1, 15, 27, 256), (1, 8, 14, 512), (1, 4, 7, 512)]
    for fast in (False, True):
        acts, folded, single = [], [], []
        for n, h, w, cin in shapes:
            x = torch.randn(n, cin, h, w, generator=g) * 2.0
            wt = torch.randn(16, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
            bs = torch.randn(16, generator=g) * 0.1
            proj = torch.randn(32, generator=g) * 0.3
            pb = torch.randn(1, generator=g)
            a = ops.nchw_to_act(x.to(dev), fast)
            (f,) = ops.fold_side_weights_multi([(wt.to(dev), bs.to(dev), proj.to(dev), pb.to(dev))])
            acts.append(a)
            folded.append(f)
            single.append(ops.side_folded(a, f[0], f[1], fast=fast))
        multi = ops.side_folded_multi(acts, folded, fast=fast)
        for k in range(len(shapes)):
            assert torch.equal(multi[k], single[k]), (fast, k)
        rev = ops.side_folded_multi(acts[::-1], folded[::-1], fast=fast)[::-1]
        for k in range(len(shapes)):
            assert torch.equal(rev[k], single[k]), (fast, k)
        two = ops.side_folded_multi(acts[1:3], folded[1:3], fast=fast)
        assert torch.equal(two[0], single[1]) and torch.equal(two[1], single[2])


def test_conv3x3_relu_mask_and_projection(dev):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(7)
    n, h, w, cin = 1, 21, 19, 64
    x = torch.randn(n, cin, h, w, generator=g)
    a = ops.nchw_to_act(x.to(dev))
    # dgrad-style: output masked by the sign of another act
    wt = torch.randn(64, cin, 3, 3, generator=g) * 0.05
    mk = torch.randn(n, 64, h, w, generator=g)
    mact = ops.nchw_to_act(mk.clamp(min=0).to(dev))
    _, yf, _ = ops.conv3x3(a, ops.pack_conv3x3_weights(wt.to(dev)), None, 64, out_act=False, out_f32=True,
                           mask=mact.hi)
    ref = F.conv2d(x.double(), wt.double(), None, padding=1) * (mk > 0)
    assert maxrel(yf.permute(0, 3, 1, 2).cpu(), ref) < EXACT_TOL
    # side_prep with the fused 1x1 projections
    w16 = torch.randn(16, cin, 3, 3, generator=g) * 0.05
    b16 = torch.randn(16, generator=g) * 0.1
    pw = torch.randn(32, generator=g)
    pb = torch.randn(1, generator=g)
    _, feat, pq = ops.conv3x3(a, ops.pack_conv3x3_weights(w16.to(dev)), b16.to(dev), 16, out_act=False, out_f32=True,
                              proj_w=pw.to(dev), proj_b=pb.to(dev))
    ref16 = F.conv2d(x.double(), w16.double(), b16.double(), padding=1)
    assert maxrel(feat.permute(0, 3, 1, 2).cpu(), ref16) < EXACT_TOL
    refp = (ref16 * pw[:16].double().view(1, 16, 1, 1)).sum(1) + pb.double()
    refq = (ref16 * pw[16:].double().view(1, 16, 1, 1)).sum(1)
    assert maxrel(pq[..., 0].cpu(), refp) < EXACT_TOL and maxrel(pq[..., 1].cpu(), refq) < EXACT_TOL
    pq2 = ops.side_project(feat, pw.to(dev), pb.to(dev))
    assert maxrel(pq2.cpu(), pq.cpu()) < 1e-6


@pytest.mark.parametrize("n,h,w,cin,cout", [(1, 16, 8, 64, 64), (2, 21, 13, 64, 128), (1, 33, 45, 128, 256), (1, 7, 5, 64, 64)])
def test_conv3x3_fused_pool_and_bias_gradient_sum(dev, n, h, w, cin, cout):
    """Epilogue fusions: MaxPool2d(2,2,ceil_mode) of the output and the per-channel output sum."""
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(17 + h)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
    b = torch.randn(cout, generator=g) * 0.1
    a = ops.nchw_to_act(x.to(dev))
    wp = ops.pack_conv3x3_weights(wt.to(dev))
    colsum = torch.zeros(cout, device=dev)
    y, yp = ops.conv3x3(a, wp, b.to(dev), cout, relu=True, pool=True, colsum=colsum)
    full = ops.act_to_nchw(y).cpu()
    assert torch.equal(ops.act_to_nchw(yp).cpu(), F.max_pool2d(full, 2, 2, ceil_mode=True))   # selection: bit exact
    y2, _, _ = ops.conv3x3(a, wp, b.to(dev), cout, relu=True)
    assert torch.equal(ops.act_to_nchw(y2).cpu(), full)
    ref = F.conv2d(x.double(), wt.double(), b.double(), padding=1).relu()
    assert maxrel(colsum.cpu(), ref.sum((0, 2, 3))) < 5e-5
    # pooled output only (inference of stage 1 needs no full-resolution map)
    none, yp2 = ops.conv3x3(a, wp, b.to(dev), cout, relu=True, pool=True, out_act=False)
    assert none is None and torch.equal(ops.act_to_nchw(yp2).cpu(), ops.act_to_nchw(yp).cpu())


@pytest.mark.parametrize("n,h,w", [(1, 16, 130), (2, 7, 5), (1, 33, 45)])
def test_conv_first(dev, n, h, w):
    from osvos_pytorch_b200 import ops
    x, _ = oc.synthetic_frame(n, h, w, 5)
    g = torch.Generator().manual_seed(9)
    wt = torch.randn(64, 3, 3, 3, generator=g) * math.sqrt(2.0 / 27)
    b = torch.randn(64, generator=g) * 0.01
    ref = F.conv2d(x.double(), wt.double(), b.double(), padding=1).relu()
    y = ops.act_to_nchw(ops.conv_first(x.to(dev), wt.to(dev), b.to(dev))).cpu()
    assert maxrel(y, ref) < 3e-5


@pytest.mark.parametrize("n,h,w,c", [(1, 8, 8, 64), (2, 7, 5, 64), (1, 33, 45, 128), (1, 1, 1, 64)])
def test_maxpool_ceil_mode(dev, n, h, w, c):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(11)
    x = split_round(torch.randn(n, c, h, w, generator=g).clamp(min=0) * 10)
    ref = F.max_pool2d(x, 2, 2, ceil_mode=True)
    y = ops.act_to_nchw(ops.maxpool2x2(ops.nchw_to_act(x.to(dev)))).cpu()
    assert torch.equal(y, ref)      # selection only: bit exact


@pytest.mark.parametrize("n,h,w", [(1, 48, 70), (2, 33, 45), (1, 240, 427), (1, 17, 3)])
def test_tail_forward_and_loss_sums(dev, n, h, w):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(13)
    pqs, hk, wk = [], h, w
    for k in range(4):
        hk, wk = oc.pooled_size(hk), oc.pooled_size(wk)
        pqs.append(torch.randn(n, hk, wk, 2, generator=g) * 5)
    fb = torch.randn(1, generator=g)
    label = torch.rand(n, 1, h, w, generator=g)
    out, sums = ops.tail_fwd([p.to(dev) for p in pqs], fb.to(dev), n, h, w, label=label.to(dev))
    out = out.cpu()
    fused = fb.double().view(1, 1, 1, 1)
    for k in range(4):
        p = pqs[k][..., 0].unsqueeze(1).double()
        q = pqs[k][..., 1].unsqueeze(1).double()
        s = 2 ** (k + 1)
        refp = oc.center_crop(oc.upsample_zero_padded(p, s), h, w)
        assert maxrel(out[k], refp) < 2e-6
        fused = fused + oc.center_crop(oc.upsample_zero_padded(q, s), h, w)
    assert maxrel(out[4], fused) < 2e-6
    sums = sums.cpu().numpy()
    y = (label >= 0.5).double()
    assert sums[10] == float(y.sum()) and sums[11] == n * h * w
    for k in range(5):
        x = out[k].double()
        sp = torch.clamp(x, min=0) + torch.log1p(torch.exp(-x.abs()))
        assert abs(sums[2 * k] - float((y * (sp - x)).sum())) <= 2e-5 * max(1.0, abs(float((y * (sp - x)).sum())))
        assert abs(sums[2 * k + 1] - float(((1 - y) * sp).sum())) <= 2e-5 * max(1.0, float(((1 - y) * sp).sum()))


def test_loss_matches_oracle_and_reference(dev, golden):
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    g = torch.Generator().manual_seed(5)
    lo = torch.randn(2, 1, 9, 13, generator=g) * 4.0
    la = torch.rand(2, 1, 9, 13, generator=g)
    for key, kw in (("sa", {}), ("ba", dict(size_average=False)),
                    ("none", dict(size_average=False, batch_average=False))):
        got = float(cbce(lo.to(dev), la.to(dev), **kw))
        assert abs(got - float(golden[f"loss.rand.{key}"])) <= 1e-5 * abs(float(golden[f"loss.rand.{key}"]))
    x = lo.to(dev).requires_grad_(True)
    loss = cbce(x, la.to(dev), size_average=False)
    (loss / 5).backward()
    assert maxrel(x.grad.cpu() * 5, golden["loss.rand.grad"]) < 1e-5
    # known answers (SURVEY.md 8c)
    z = torch.zeros(1, 1, 4, 5, device=dev)
    lab = torch.zeros(1, 1, 4, 5)
    lab.view(-1)[:10] = 1
    assert abs(float(cbce(z, lab.to(dev), size_average=False)) - 6.931472) < 1e-5
    assert abs(float(cbce(torch.full((1, 1, 2, 2), -100.0, device=dev),
                          torch.tensor([1.0, 0, 0, 0]).view(1, 1, 2, 2).to(dev), size_average=False)) - 75.0) < 1e-4
    assert float(cbce(torch.full((1, 1, 2, 2), 100.0, device=dev), torch.ones(1, 1, 2, 2, device=dev),
                      size_average=False)) == 0.0
    assert float(cbce(torch.randn(1, 1, 3, 3, device=dev), torch.zeros(1, 1, 3, 3, device=dev),
                      size_average=False)) == 0.0
    # odd element count (tail path) and python sum()/scalar multiply on the result
    xo = torch.randn(1, 1, 7, 9, generator=g)
    lo_ = torch.rand(1, 1, 7, 9, generator=g)
    got = cbce(xo.to(dev), lo_.to(dev), size_average=False)
    want = oc.class_balanced_cross_entropy_loss(xo.double(), lo_.double(), size_average=False)
    assert abs(float(got) - float(want)) < 1e-5 * abs(float(want))
    total = 0.5 * sum([got, got]) + got
    assert abs(float(total) - 2 * float(want)) < 1e-4 * abs(float(want))

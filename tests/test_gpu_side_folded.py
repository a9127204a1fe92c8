"""Side branch backward in folded (rank-2) form (csrc/side_bwd_folded.cu, unpool_add_mask_kernel's dpq/wfold path,
osvos_fold_side_weights_multi) against torch CPU fp64 autograd of the LITERAL branch the reference runs
(networks/vgg_osvos.py:67,69,72: side_prep 3x3 C -> 16 without ReLU, score_dsn 1x1, this scale's slice of fuse).  The whole
network's gradients through this route are held to the reference's golden gradients and to the oracle by
tests/test_gpu_backward.py."""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import maxrel, split_round

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _literal_branch(x, side_w, side_b, ws, bs, wf, dp, dq):
    """fp64 autograd of the literal branch: returns grads of (x, side_w, side_b, ws, bs, wf)."""
    xs = x.double().requires_grad_(True)
    p = [t.double().requires_grad_(True) for t in (side_w, side_b, ws, bs, wf)]
    feat = F.conv2d(xs, p[0], p[1], padding=1)
    pp = (feat * p[2].view(1, 16, 1, 1)).sum(1) + p[3]
    qq = (feat * p[4].view(1, 16, 1, 1)).sum(1)
    ((pp * dp.double()).sum() + (qq * dq.double()).sum()).backward()
    return [xs.grad] + [t.grad for t in p]


@pytest.mark.parametrize("n,h,w,c", [(1, 9, 14, 128), (2, 7, 5, 128), (1, 33, 45, 256), (1, 4, 6, 512), (1, 40, 70, 128)])
def test_folded_side_backward(dev, n, h, w, c):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(h * w + c)
    x = split_round(torch.randn(n, c, h, w, generator=g).clamp(min=0) * 2)       # a post-ReLU stage output
    side_w = torch.randn(16, c, 3, 3, generator=g) * 0.05
    side_b = torch.randn(16, generator=g) * 0.1
    ws, wf = torch.randn(16, generator=g), torch.randn(16, generator=g)
    bs = torch.randn(1, generator=g)
    dp, dq = torch.randn(n, h, w, generator=g), torch.randn(n, h, w, generator=g)
    dpool = split_round(torch.randn(n, c, (h + 1) // 2, (w + 1) // 2, generator=g))
    dx_ref, dsw, dsb, dws, dbs, dwf = _literal_branch(x, side_w, side_b, ws, bs, wf, dp, dq)

    proj = torch.cat([ws, wf]).to(dev)
    (packed, bias2, wfold), = ops.fold_side_weights_multi([(side_w.to(dev), side_b.to(dev), proj, bs.to(dev))])
    # the fold itself: W'[t][o][c] = sum_f proj[o][f] side_w[f][c][t]; the packed operand is the split-bf16 packing of
    # that same fp32 fold (as OIHW [2, c, 3, 3]), bit for bit
    want_fold = torch.einsum("of,fct->toc", torch.stack([ws, wf]).double(), side_w.double().reshape(16, c, 9))
    assert maxrel(wfold, want_fold) < 1e-6
    assert torch.equal(packed, ops.pack_conv3x3_weights(wfold.permute(1, 2, 0).reshape(2, c, 3, 3)))
    # b'[o] = (o == 0 ? proj_b : 0) + sum_f proj[o][f] side_b[f]: 16 fp32 FMAs after the proj_b term
    terms = torch.stack([ws, wf]).double() * side_b.double()
    want_b = terms.sum(1) + torch.cat([bs.double(), torch.zeros(1, dtype=torch.float64)])
    b_bound = 17 * 2.0 ** -24 * (terms.abs().sum(1) + torch.cat([bs.double().abs(), torch.zeros(1, dtype=torch.float64)]))
    assert bool(((bias2.cpu().double() - want_b).abs() <= b_bound).all()), (bias2, want_b)

    xa = ops.nchw_to_act(x.to(dev))
    dpq = torch.stack([dp, dq], dim=-1).contiguous().to(dev)
    # (1) G and the parameter gradients
    gbuf = torch.zeros(ops.side_folded_wgrad_floats(c), device=dev)
    ops.side_folded_wgrad_multi([xa], [dpq], [gbuf])
    G = gbuf[:18 * c].view(9, 2, c).cpu().double()
    xpad = F.pad(x.double(), (1, 1, 1, 1))
    for t in range(9):
        r, s = t // 3, t % 3
        win = xpad[:, :, r:r + h, s:s + w]                                         # x[q + (r-1, s-1)]
        assert maxrel(G[t, 0], (win * dp.double().unsqueeze(1)).sum((0, 2, 3))) < 2e-5, t
        assert maxrel(G[t, 1], (win * dq.double().unsqueeze(1)).sum((0, 2, 3))) < 2e-5, t
    assert abs(float(gbuf[18 * c]) - float(dp.double().sum())) < 1e-3 and abs(float(gbuf[18 * c + 1]) - float(dq.double().sum())) < 1e-3
    out = {k: torch.full(shape, 7.0, device=dev) for k, shape in
           (("d_side_w", (16, c, 3, 3)), ("d_side_b", (16,)), ("d_score_w", (16,)), ("d_score_b", (1,)), ("d_fuse_w", (16,)))}
    entry = dict(out, g=gbuf, side_w=side_w.to(dev), side_b=side_b.to(dev), proj_w=proj, c=c)
    ops.side_grads_finish([entry], accumulate=False)
    for k, ref in (("d_side_w", dsw), ("d_side_b", dsb), ("d_score_w", dws), ("d_score_b", dbs), ("d_fuse_w", dwf)):
        assert maxrel(out[k], ref) < 3e-5, (k, maxrel(out[k], ref))
    ops.side_grads_finish([entry], accumulate=True)                                # adds to what is there
    for k, ref in (("d_side_w", dsw), ("d_fuse_w", dwf)):
        assert maxrel(out[k], 2 * ref) < 3e-5, k
    # unsupervised side map / fused map: NULL outputs are skipped
    entry2 = {k: v for k, v in entry.items() if k not in ("d_score_w", "d_score_b", "d_fuse_w")}
    ops.side_grads_finish([entry2], accumulate=False)
    assert maxrel(out["d_side_b"], dsb) < 3e-5

    # (2) dz = ReLU'(x) * (unpool(dpool) + dX) with dX formed on the fly; and the deepest-stage form without pooling
    xr = x.clone().double().requires_grad_(True)
    F.max_pool2d(xr, 2, 2, ceil_mode=True).backward(dpool.double())
    for pooled in (True, False):
        want = ((xr.grad if pooled else 0) + dx_ref) * (x > 0)
        colsum = torch.zeros(c, device=dev)
        dz = ops.unpool_mask(ops.nchw_to_act(dpool.to(dev)) if pooled else None, xa, dpq=dpq, wfold=wfold,
                             colsum=colsum)
        got = ops.act_to_nchw(dz).cpu()
        assert maxrel(got, want) < 3e-5, (pooled, maxrel(got, want))
        assert maxrel(colsum.cpu(), want.sum((0, 2, 3))) < 3e-5


def test_folded_wgrad_scales_in_one_launch(dev):
    """osvos_side_folded_wgrad_multi: the four scales' G in one launch (block ranges per scale) equals one launch per scale
    (the same entry point with one item) up to the order of the fp32 atomics."""
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(31)
    shapes = [(1, 30, 53, 128), (1, 15, 27, 256), (1, 8, 14, 512), (1, 4, 7, 512)]
    for fast in (False, True):
        xs, dpqs = [], []
        for n, h, w, c in shapes:
            xs.append(ops.nchw_to_act((torch.randn(n, c, h, w, generator=g).clamp(min=0) * 2).to(dev), fast))
            dpqs.append(torch.randn(n, h, w, 2, generator=g).to(dev))
        single = []
        for x, d in zip(xs, dpqs):
            gb = torch.zeros(ops.side_folded_wgrad_floats(x.shape[3]), device=dev)
            ops.side_folded_wgrad_multi([x], [d], [gb])
            single.append(gb)
        multi = [torch.zeros_like(s) for s in single]
        ops.side_folded_wgrad_multi(xs, dpqs, multi)
        for k in range(len(shapes)):
            assert maxrel(multi[k], single[k]) < 1e-5, (fast, k, maxrel(multi[k], single[k]))
        two = [torch.zeros_like(single[2]), torch.zeros_like(single[0])]
        ops.side_folded_wgrad_multi([xs[2], xs[0]], [dpqs[2], dpqs[0]], two)
        assert maxrel(two[0], single[2]) < 1e-5 and maxrel(two[1], single[0]) < 1e-5

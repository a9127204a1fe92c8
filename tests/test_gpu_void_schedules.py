"""Every launch regime of the void loss kernels (OSVOS_FLAG_VOID_LABELS, DESIGN.md §26), at the running device's SM
count, against fp64 of the operands the kernels read - the regimes tests/train_dispatch_ref.py finds for their plain
twins, under the bounds of tests/test_gpu_train_schedules.py (its module docstring derives them).  torch.profiler
confirms that each call ran the void kernel, once.

- tail_bwd2_void_kernel<DET>: atomic and deterministic over train_dispatch_ref.find_tail_bwd_widths() - every reachable
  (scale, row groups) pair, an idle-thread width, full and short segments at scales 0 and 1 (a width past 510: two
  segments per low-res row at scale 0, as at 854) - with labels of -1 / 0 / 0.5 / 1 and the upstream gradient null and
  set; and every pixel void (N = 0: every output exactly 0).
- cbce_fwd_void_kernel<DET> and cbce_bwd_void_kernel: numel 1 - 3 (no vector), one block, and a capped grid, each
  with numel % 4 = 1, 2, 3 and 0, labels -1 / 0 / 0.5 / 1; and all void, and positives with void only (one class:
  loss and gradient exactly 0)."""
import pytest
import torch

import train_dispatch_ref as tdr
from conv_dispatch_ref import parse_kernel_name
from test_gpu_conv_schedules import KernelsRan
from test_gpu_train_schedules import U, _adjoint, _gen, _stream, check_bound

pytestmark = pytest.mark.gpu

VOID_KERNELS = {"tail_bwd2_void_kernel": 0, "cbce_fwd_void_kernel": 0}


def parse_void_kernel_name(name):
    p = parse_kernel_name(name, VOID_KERNELS)
    if p is not None:
        return p
    return ("cbce_bwd_void_kernel", ()) if "cbce_bwd_void_kernel(" in name else None


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


def ran(fn, expected):
    """fn() with the void kernels it launched, which must be exactly ``expected`` ({(kernel, args): launches}); a
    window that lost a record is run again, at most twice, and a window with no device record at all is not judged."""
    for _ in range(3):
        with KernelsRan(parse_void_kernel_name) as k:
            out = fn()
        if sum(k.counts.values()) >= sum(expected.values()):
            break
    if not k.counts and not any(d == "CUDA" for _, d, _ in k.seen):
        return out
    assert k.counts == expected, (k.counts, k.seen[:12])
    return out


def _void_labels(shape, g, kind="mixed"):
    if kind == "all_void":
        return -torch.ones(shape)
    if kind == "pos_void":
        return torch.where(torch.rand(shape, generator=g) < 0.5, 1.0, -1.0)
    y = torch.randint(-1, 3, shape, generator=g).float()
    return torch.where(y < 0, -1.0, y * 0.5)                    # -1, 0, 0.5 and 1


# ------------------------------------------------------------------------------------------------ tail backward
TAIL_WIDTHS = tdr.find_tail_bwd_widths()
TAIL_TARGETS = [(w, det, up, "mixed") for w in TAIL_WIDTHS for det in (False, True) for up in (False, True)] + \
    [(TAIL_WIDTHS[0], det, True, "all_void") for det in (False, True)]


@pytest.mark.parametrize("target", TAIL_TARGETS,
                         ids=[f"w{w}-{'det' if d else 'atomic'}{'-upstream' if u else ''}-{k}"
                              for w, d, u, k in TAIL_TARGETS])
def test_tail_loss_bwd_void(dev, target):
    """dpq of the five void gradient maps g_k = c_k w (sigmoid(x_k) - [y >= .5]), w = Nn/N, P/N or 0 on void, and
    fuse_bias_grad = c_4 (Nn/N A_pos + P/N A_neg) from the sums as given; N = the non-void count."""
    from osvos_pytorch_b200 import ops
    w, det, with_upstream, kind = target
    assert max(TAIL_WIDTHS) > 2 * tdr.TAIL_SEG_LO[0]             # the regime of 854-wide frames is in the set
    n, h = 2, 13
    scales, _ = tdr.tail_bwd_scales(n, h, w)
    items = tdr.tail_bwd_row_items(w)
    depth = [max(tdr.tail_bwd_depth(it) for it in items if it.scale == k) for k in range(4)]
    g = _gen(5000 + w + det)
    logits = torch.randn(5, n, 1, h, w, generator=g) * 4.0
    label = _void_labels((n, 1, h, w), g, kind)
    pos, neg = label >= 0.5, (label >= 0) & (label < 0.5)
    P, N = float(pos.sum()), float(pos.sum() + neg.sum())
    sums = torch.zeros(tdr.TAIL_SUMS, dtype=torch.float64)
    sums[10], sums[11], sums[12], sums[13] = P, N, 37.25, -11.5
    weights, divisor = (0.5, 0.0, 0.75, 1.0, 1.5), 2.0
    upstream = torch.tensor([0.7], device=dev) if with_upstream else None
    up = float(torch.tensor(0.7, dtype=torch.float32)) if with_upstream else 1.0
    d_logits, d_label, d_sums = logits.to(dev), label.to(dev), sums.to(dev)

    def call():
        return ops.tail_loss_bwd(d_logits, d_label, d_sums, weights, divisor, upstream, n, h, w, want_fuse_bias=True,
                                 deterministic=det, void=True)
    dpq, fb = ran(call, {("tail_bwd2_void_kernel", (det,)): 1})
    if det:
        again, fb2 = call()
        assert all(torch.equal(a, b) for a, b in zip(dpq, again)) and torch.equal(fb, fb2), \
            "deterministic dpq differs between runs"
    if N == 0:
        assert all(bool((t == 0).all()) for t in dpq) and float(fb) == 0.0
        return
    xd = logits.double()
    sg = torch.sigmoid(xd)
    cls = torch.where(pos, (N - P) / N, torch.where(neg, P / N, 0.0)).double()
    yv = pos.double()
    maps, mags = [], []
    for k in range(5):
        c = weights[k] * up / divisor
        maps.append(c * cls * (sg[k] - yv))
        mags.append(abs(c) * cls * (sg[k] + 1.0))
    extra = 3 + 8 + 1.2 * xd.abs().max().item()
    c4 = weights[4] * up / divisor
    fb_ref = c4 * ((N - P) / N * 37.25 + P / N * -11.5)
    fb_mag = abs(c4) * ((N - P) / N * 37.25 + P / N * 11.5)
    check_bound("tail bwd void fuse bias", fb, torch.tensor([fb_ref]), torch.tensor([8 * U * fb_mag]), "fuse_bias_grad")
    family = f"tail bwd void {'det' if det else 'atomic'}"
    for k, sc in enumerate(scales):
        got = dpq[k].cpu().double()
        steps = depth[k] + extra
        for ch, src in ((0, k), (1, 4)):
            check_bound(family, got[..., ch], _adjoint(maps[src], sc, h, w),
                        steps * U * _adjoint(mags[src], sc, h, w), f"scale {k} channel {ch}")


# ------------------------------------------------------------------------------------------------ loss
CBCE_TARGETS = [(regime, i, det, "mixed") for regime in tdr.CBCE_REGIMES
                for i in range(4 if regime != "tiny" else 3) for det in (False, True)] + \
    [(regime, 0, det, kind) for regime in ("one_block", "capped") for kind in ("all_void", "pos_void")
     for det in (False, True)]


def _cbce_id(regime, i, det, kind):
    numel = tdr.find_cbce_numels(regime, 132)[i]
    return f"{regime}-mod{numel % 4}-{kind}-{'det' if det else 'atomic'}"


@pytest.mark.parametrize("target", CBCE_TARGETS, ids=[_cbce_id(*t) for t in CBCE_TARGETS])
def test_cbce_void_fwd_bwd(dev, sms, target):
    """Sums over the non-void pixels, P and N exact, the loss, and the backward with and without an upstream gradient
    (void pixels exactly 0), under test_gpu_train_schedules' cbce bounds."""
    from osvos_pytorch_b200 import _native as nat
    lib = nat.load()
    regime, i, det, kind = target
    numel = tdr.find_cbce_numels(regime, sms)[i]
    g = _gen(6000 + numel)
    x = torch.randn(numel, generator=g) * 4.0
    y = _void_labels((numel,), g, kind)
    if kind == "mixed" and numel >= 2:
        y[:2] = torch.tensor([0.5, -1.0])
    d_x, d_y = x.to(dev), y.to(dev)
    grid = tdr.loss_grid(numel, sms)
    flags = nat.FLAG_VOID_LABELS | (nat.FLAG_DETERMINISTIC if det else 0)
    assert lib.osvos_cbce_fwd_sums(numel, flags) == (5 + 4 * grid if det else 5)
    sums = torch.zeros(lib.osvos_cbce_fwd_sums(numel, flags), dtype=torch.float64, device=dev)
    loss = torch.empty(1, device=dev)
    divisor = 3.0
    ran(lambda: nat.check(lib.osvos_cbce_fwd(d_x.data_ptr(), d_y.data_ptr(), numel, divisor, sums.data_ptr(),
                                             loss.data_ptr(), flags, _stream()), "cbce fwd"),
        {("cbce_fwd_void_kernel", (det,)): 1})
    if det:
        s2, l2 = sums.clone(), loss.clone()
        nat.check(lib.osvos_cbce_fwd(d_x.data_ptr(), d_y.data_ptr(), numel, divisor, s2.data_ptr(), l2.data_ptr(),
                                     flags, _stream()), "cbce fwd")
        assert torch.equal(s2[:4], sums[:4]) and torch.equal(l2, loss), "deterministic cbce differs between runs"
    xd = x.double()
    pos, neg = y >= 0.5, (y >= 0) & (y < 0.5)
    sp = xd.clamp(min=0) + torch.log1p(torch.exp(-xd.abs()))
    e_terms = 8 + 1.2 * xd.abs().max().item()
    ordered = -(-grid // 256) + 256
    depth = 4 * tdr.loss_vectors_per_thread(numel, sms) + 1 + 5 + 8 + (ordered if det else grid) + e_terms
    term = sp + xd.abs()
    want = torch.stack([(sp - xd)[pos].sum(), sp[neg].sum()])
    bound = torch.stack([depth * U * term[pos].sum(), depth * U * term[neg].sum()])
    s = sums.cpu()
    check_bound("cbce void sums", s[:2], want, bound, f"sums of {numel}")
    P, N = float(pos.sum()), float(pos.sum() + neg.sum())
    assert s[2].item() == P and s[3].item() == N, (s[:4], P, N)
    if N > 0:
        lref = ((N - P) / N * want[0] + P / N * want[1]) / divisor
        lb = ((N - P) / N * bound[0] + P / N * bound[1]) / divisor + 2 * U * abs(lref)
    else:
        lref, lb = torch.tensor(0.0, dtype=torch.float64), torch.tensor(0.0, dtype=torch.float64)
    check_bound("cbce void loss", loss.cpu(), lref.view(1), lb.view(1), f"loss of {numel}")
    for gout in (None, 0.625):
        buf = torch.full((numel + 8,), float("nan"), device=dev)
        dx = buf[:numel]
        d_g = None if gout is None else torch.tensor([gout], device=dev)
        ran(lambda: nat.check(lib.osvos_cbce_bwd_void(d_x.data_ptr(), d_y.data_ptr(), sums.data_ptr(), nat.ptr(d_g),
                                                      divisor, numel, dx.data_ptr(), _stream()), "cbce bwd void"),
            {("cbce_bwd_void_kernel", ()): 1})
        assert bool(torch.isnan(buf[numel:]).all()), "cbce backward wrote past numel"
        gg = (1.0 if gout is None else gout) * float(torch.tensor(1.0 / divisor, dtype=torch.float32))
        if N > 0:
            wcls = torch.where(pos, (N - P) / N, torch.where(neg, P / N, 0.0)).double() * gg
        else:
            wcls = torch.zeros(numel, dtype=torch.float64)
        sg = torch.sigmoid(xd)
        ref = wcls * (sg - pos.double())
        check_bound("cbce void bwd", dx, ref, (e_terms + 6) * U * wcls.abs() * (sg + 1), f"dx of {numel}")
        assert bool((dx.cpu()[~(pos | neg)] == 0).all()), "a void pixel got a gradient"

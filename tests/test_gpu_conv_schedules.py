"""Every schedule of the 3x3 convolution kernels, at the running device's SM count, against fp64 of the operands the
kernel reads.

Forward / data gradient: one test per instantiation of conv3x3_halo_kernel<BLOCK_N, PLANES, SPLIT, LEAN, PINGPONG, DET>
the dispatcher can pick (tests/conv_dispatch_ref.py: REACHABLE_HALO), at a small shape that selects it on this device
(find_halo_shape), with more tiles than CTAs so that CTAs also run a second tile.  Weight gradient: {tap rows, tap
pairs, nine taps} x {one pixel-range split, several with a short last one} x {exact, fast} x {atomic, deterministic},
plus nine taps with more items than CTAs and more patches per split than ring stages.  torch.profiler confirms which
kernel instantiation each launch ran.

Reference and bounds.  The kernels form exact bf16 x bf16 products and add them in fp32; exact mode sums the three
products A_hi.B_hi + A_hi.B_lo + A_lo.B_hi of the split operands, fast mode A_hi.B_hi only.  The reference is the fp64
convolution (or weight gradient) of exactly those planes, read back from the Act tensors and the packed weights, so
only the fp32 summation differs from it.  An output is a chain of `steps` fp32 accumulations (one per wgmma of K = 16
that adds into it, plus the epilogue's adds); each rounds by at most 2^-23 of the running sum (a truncating adder's
unit), and for these zero-mean operands the running sums stay within the largest output, so
    max |got - ref| <= steps * 2^-23 * max |ref|.
For a forward with k 64-channel chunks that is steps = 9 * 4 * k * passes + 2 (passes = 3 exact, 1 fast), about 1e-5
at k = 2 exact.  Column sums add the stored fp32 outputs in a tree and then per partial row, D additions deep, so they
are bounded by the outputs' own error plus D * 2^-23 * sum |y| per channel (the standard recursive-summation bound), and
normalised by sum |ref| per channel because the plain sum can cancel."""
import math
import os
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

import conv_dispatch_ref as cdr
from gpu_util import maxrel, split_round

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
EXACT_TOL = 3e-5    # against fp64 of the unsplit fp32 operands (as tests/test_gpu_kernels.py)


@pytest.fixture(scope="module")
def dev():
    assert "OSVOS_ABLATE" not in os.environ, "OSVOS_ABLATE switches off parts of the kernels: results are meaningless"
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(0).multi_processor_count


class KernelsRan:
    """Counts the conv3x3_halo_kernel / wgrad_tc_kernel instantiations (or those ``parse`` recognises) the device ran
    inside the block, by their demangled names in a torch.profiler trace of CUDA activity; ``seen`` lists every record
    of the window as (name, device type, count)."""
    def __init__(self, parse=cdr.parse_kernel_name):
        self.parse = parse

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        self.counts = Counter()
        self.seen = []
        for ev in self.prof.key_averages():
            self.seen.append((ev.key[:60], ev.device_type.name, ev.count))
            if ev.device_type.name != "CUDA":
                continue
            parsed = self.parse(ev.key)
            if parsed is not None:
                self.counts[parsed] += ev.count
        return False


def profiled(fn, expected, parse=cdr.parse_kernel_name):
    """fn() under KernelsRan(parse); its kernels must be exactly ``expected`` ({(kernel, template args): launches}).
    The profiler occasionally loses a kernel record from a window (a count below the launches made, seen on the H100 at
    about one window in 50); such a window is run again, at most twice.  A wrong instantiation fails either way."""
    for _ in range(3):
        with KernelsRan(parse) as k:
            out = fn()
        if sum(k.counts.values()) >= sum(expected.values()):
            break
    assert k.counts == expected, (k.counts, k.seen[:12])
    return out


def _halo_id(t):
    block_n, planes, split, lean, pingpong, det = t
    return (f"n{block_n}-{'exact' if planes == 2 else 'fast'}{'-split' if split else ''}{'-lean' if lean else ''}"
            f"-{'pingpong' if pingpong else 'coop'}{'-det' if det else ''}")


HALO_TARGETS = sorted(cdr.REACHABLE_HALO)


def _weights_seen(wp, cout, cin):
    """The packed [plane][tap][cout][cin] weights as two fp64 OIHW tensors (hi, lo)."""
    planes = wp[: 2 * 9 * cout * cin].view(2, 3, 3, cout, cin).double()
    return planes[0].permute(2, 3, 0, 1), planes[1].permute(2, 3, 0, 1)


def _nchw(plane):
    return plane.double().permute(0, 3, 1, 2)


class HaloProblem:
    """Seeded operands of one shape, their Act / packed forms and the fp64 references."""
    def __init__(self, s, dev):
        from osvos_pytorch_b200 import ops
        g = torch.Generator().manual_seed(1000 + s.h * 7 + s.w + s.cin + s.cout)
        self.s = s
        x = torch.randn(s.n, s.cin, s.h, s.w, generator=g) * 3.0
        wt = torch.randn(s.cout, s.cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * s.cin))
        self.bias = (torch.randn(s.cout, generator=g) * 0.1).to(dev)
        self.a = ops.nchw_to_act(x.to(dev), s.fast)
        self.wp = ops.pack_conv3x3_weights(wt.to(dev))
        torch.cuda.synchronize()
        w_hi, w_lo = _weights_seen(self.wp, s.cout, s.cin)
        x_hi = _nchw(self.a.hi)
        lin = F.conv2d(x_hi, w_hi, padding=1)
        if not s.fast:
            x_lo = _nchw(self.a.lo)
            lin = lin + F.conv2d(x_hi, w_lo, padding=1) + F.conv2d(x_lo, w_hi, padding=1)
        self.lin = lin                                    # seen-operand product sum, no bias
        self.unsplit = F.conv2d(x.double().to(dev), wt.double().to(dev), padding=1)
        steps = 9 * 4 * (s.cin // 64) * (1 if s.fast else 3) + 2
        self.tol = steps * U

    def ref(self, bias=True, relu=False):
        r = self.lin + self.bias.double().view(1, -1, 1, 1) if bias else self.lin
        return r.relu() if relu else r

    def check_f32(self, yf, bias, relu, what, mask=None):
        got = yf.double().permute(0, 3, 1, 2)
        ref = self.ref(bias, relu)
        if mask is not None:
            ref = ref * mask
        scale = self.ref(bias).abs().max().item()
        err = (got - ref).abs().max().item() / scale
        MEASURED.setdefault(("fast" if self.s.fast else "exact"), []).append((err, self.tol))
        assert err <= self.tol, (what, err, self.tol)
        if not self.s.fast:
            uref = self.unsplit + self.bias.double().view(1, -1, 1, 1) if bias else self.unsplit
            uref = uref.relu() if relu else uref
            if mask is not None:
                uref = uref * mask
            assert maxrel(got, uref) < EXACT_TOL, (what, maxrel(got, uref))
        return got

    def colsum_bound(self, cs, y):
        """|cs - sum ref| per channel over sum |ref|, and the bound it must stay under (module docstring)."""
        ref = self.ref(bias=False)
        m_tiles = -(-self.s.h // 16) * -(-self.s.w // 8) * self.s.n
        depth = 5 + 8 * m_tiles     # 4 in the warp, then one per partial row of 8 per tile, then into the zeroed sum
        sum_abs = ref.abs().sum((0, 2, 3))
        out_err = (y - ref).abs().sum((0, 2, 3))
        err = (cs.double() - ref.sum((0, 2, 3))).abs()
        bound = out_err + depth * U * y.abs().sum((0, 2, 3))
        return err, bound, sum_abs


MEASURED = {}


@pytest.fixture(scope="module", autouse=True)
def _report_measured():
    yield
    for mode, v in sorted(MEASURED.items()):
        print(f"\n{mode}: largest max|got - ref| / max|ref| {max(e for e, _ in v):.2e}, largest share of its bound "
              f"{max(e / t for e, t in v):.3f} ({len(v)} outputs)")


@pytest.mark.parametrize("target", HALO_TARGETS, ids=[_halo_id(t) for t in HALO_TARGETS])
def test_halo_schedule(dev, sms, target):
    from osvos_pytorch_b200 import ops
    block_n, planes, split, lean, pingpong, det = target
    s = cdr.find_halo_shape(target, sms, **cdr.halo_case_args(target))
    assert s is not None, (target, sms)
    assert cdr.halo_plan(s.n, s.h, s.w, s.cin, s.cout, s.fast, s.lean, s.det, sms) == (target, s.total_tiles)
    p = HaloProblem(s, dev)
    b, cout, fast = p.bias, s.cout, s.fast

    if lean:
        general = (block_n, planes, split, False, pingpong, False)

        def lean_launches():
            y_act, _, _ = ops.conv3x3(p.a, p.wp, b, cout, relu=True, out_act=True)
            none, pool_only = ops.conv3x3(p.a, p.wp, b, cout, relu=True, pool=True, out_act=False)
            y_pa, pool_pa = ops.conv3x3(p.a, p.wp, b, cout, relu=True, pool=True, out_act=True)
            return y_act, none, pool_only, y_pa, pool_pa
        y_act, none, pool_only, y_pa, pool_pa = profiled(lean_launches, {("conv3x3_halo_kernel", target): 3})
        _, yf, _ = profiled(lambda: ops.conv3x3(p.a, p.wp, b, cout, relu=True, out_act=False, out_f32=True),
                            {("conv3x3_halo_kernel", general): 1})
        p.check_f32(yf, True, True, "general fp32 output")
        want = split_round(yf.permute(0, 3, 1, 2).cpu())
        stored = ops.act_to_nchw(y_act).cpu()
        assert torch.equal(stored, want)
        assert torch.equal(ops.act_to_nchw(y_pa).cpu(), want)
        want_pool = F.max_pool2d(stored, 2, 2, ceil_mode=True)      # selection of the stored values: bit exact
        assert none is None
        assert torch.equal(ops.act_to_nchw(pool_only).cpu(), want_pool)
        assert torch.equal(ops.act_to_nchw(pool_pa).cpu(), want_pool)
        return

    if det:
        def det_launches():
            rows = []
            for _ in range(2):
                cs = torch.zeros(cout, device=dev)
                _, yf, _ = ops.conv3x3(p.a, p.wp, None, cout, fast=fast, out_act=False, out_f32=True, colsum=cs,
                                       deterministic=True)
                rows.append((cs, yf))
            return rows
        rows = profiled(det_launches, {("conv3x3_halo_kernel", target): 2})
        assert torch.equal(rows[0][0], rows[1][0]), "deterministic column sums differ between two launches"
        assert torch.equal(rows[0][1], rows[1][1])
        y = p.check_f32(rows[0][1], False, False, "det fp32 output")
        err, bound, sum_abs = p.colsum_bound(rows[0][0], y)
        assert bool((err <= bound).all()), ((err - bound).max().item(), (err / sum_abs).max().item())
        cs_atomic = torch.zeros(cout, device=dev)
        ops.conv3x3(p.a, p.wp, None, cout, fast=fast, out_act=False, out_f32=True, colsum=cs_atomic)
        torch.cuda.synchronize()
        depth = 5 + 8 * (s.total_tiles // (cout // block_n))
        reassoc = 2 * depth * U * y.abs().sum((0, 2, 3))
        assert bool(((rows[0][0].double() - cs_atomic.double()).abs() <= reassoc).all())
        return

    g = torch.Generator().manual_seed(77 + s.w)
    mk = torch.randn(s.n, cout, s.h, s.w, generator=g)
    flat = mk.view(-1)
    flat[::5] = 0.0
    flat[1::7] = -0.0
    mact = ops.nchw_to_act(mk.to(dev))
    mask = (mact.hi.double() > 0).permute(0, 3, 1, 2)
    assert bool((mact.hi == 0).any()) and bool((mact.hi < 0).any()) and bool((mact.hi > 0).any())
    def general_launches():
        y_relu, yf_relu, _ = ops.conv3x3(p.a, p.wp, b, cout, relu=True, fast=fast, out_act=True, out_f32=True)
        y_lin, yf_lin, _ = ops.conv3x3(p.a, p.wp, b, cout, relu=False, fast=fast, out_act=True, out_f32=True)
        _, yf_mask, _ = ops.conv3x3(p.a, p.wp, None, cout, fast=fast, out_act=False, out_f32=True, mask=mact.hi)
        cs = torch.zeros(cout, device=dev)
        _, yf_cs, _ = ops.conv3x3(p.a, p.wp, None, cout, fast=fast, out_act=False, out_f32=True, colsum=cs)
        return y_relu, yf_relu, y_lin, yf_lin, yf_mask, cs, yf_cs
    y_relu, yf_relu, y_lin, yf_lin, yf_mask, cs, yf_cs = profiled(general_launches,
                                                                  {("conv3x3_halo_kernel", target): 4})
    for y, yf, relu in ((y_relu, yf_relu, True), (y_lin, yf_lin, False)):
        p.check_f32(yf, True, relu, f"relu={relu}")
        f32 = yf.permute(0, 3, 1, 2).cpu()
        want_act = f32.to(torch.bfloat16).float() if fast else split_round(f32)
        assert torch.equal(ops.act_to_nchw(y).cpu(), want_act), relu
    p.check_f32(yf_mask, False, False, "relu mask", mask=mask)
    y = p.check_f32(yf_cs, False, False, "column-sum launch")
    err, bound, sum_abs = p.colsum_bound(cs, y)
    assert bool((err <= bound).all()), ((err - bound).max().item(), (err / sum_abs).max().item())


# ------------------------------------------------------------------------------------------------ weight gradient
WGRAD_CHANNELS = {(mode, regime): ch for mode, regime, ch in cdr.WGRAD_SHAPES}
WGRAD_TARGETS = [(mode, regime, fast, det) for mode, regime, _ in cdr.WGRAD_SHAPES
                 for fast in (False, True) for det in (False, True)]


def _wgrad_id(t):
    mode, regime, fast, det = t
    return f"{mode}-{regime}-{'fast' if fast else 'exact'}-{'det' if det else 'atomic'}"


class WgradProblem:
    def __init__(self, mode, regime, fast, det, sms, dev, seed=0):
        from osvos_pytorch_b200 import ops
        self.plan_sms = cdr.WGRAD_NOMINAL_SMS if det else sms
        self.cin, self.dz = WGRAD_CHANNELS[(mode, regime)]
        self.n, self.h, self.w = cdr.find_wgrad_shape(mode, regime, self.plan_sms, sms, (self.cin, self.dz))
        self.plan = cdr.wgrad_plan(self.n, self.h, self.w, self.dz, self.cin, self.plan_sms)
        g = torch.Generator().manual_seed(500 + seed + self.h * 3 + self.w + self.dz)
        x = torch.randn(self.n, self.cin, self.h, self.w, generator=g) * 2.0
        dz = torch.randn(self.n, self.dz, self.h, self.w, generator=g) * 0.5
        self.x, self.g = ops.nchw_to_act(x.to(dev), fast), ops.nchw_to_act(dz.to(dev), fast)
        self.fast, self.det = fast, det
        torch.cuda.synchronize()
        shape = (self.dz, self.cin, 3, 3)
        wg = torch.nn.grad.conv2d_weight
        xh, gh = _nchw(self.x.hi), _nchw(self.g.hi)
        ref = wg(xh, shape, gh, padding=1)
        if not fast:
            ref = ref + wg(_nchw(self.x.lo), shape, gh, padding=1) + wg(xh, shape, _nchw(self.g.lo), padding=1)
        self.ref = ref
        # an output element: patches_per_split K blocks of 4 wgmma steps per pass, then one add per split, then the finish
        steps = 4 * self.plan.patches_per_split * (1 if fast else 3) + self.plan.splits + 1
        self.tol = steps * U

    def run(self, **kw):
        from osvos_pytorch_b200 import ops
        return ops.conv3x3_wgrad(self.x, self.g, self.dz, fast=self.fast, deterministic=self.det, **kw)

    def check(self, dw):
        err = (dw.double() - self.ref).abs().max().item() / self.ref.abs().max().item()
        MEASURED.setdefault("wgrad " + ("fast" if self.fast else "exact"), []).append((err, self.tol))
        assert err <= self.tol, (err, self.tol, self.plan)


@pytest.mark.parametrize("target", WGRAD_TARGETS, ids=[_wgrad_id(t) for t in WGRAD_TARGETS])
def test_wgrad_schedule(dev, sms, target):
    from osvos_pytorch_b200 import _native as nat
    mode, regime, fast, det = target
    p = WgradProblem(mode, regime, fast, det, sms, dev)
    assert p.plan.mode == mode
    if regime == "one_split":
        assert p.plan.splits == 1
    elif regime == "splits":
        assert p.plan.splits > 1 and p.plan.patches_total % p.plan.patches_per_split != 0
    else:   # CTAs run several items, and the operand ring wraps within an item
        assert p.plan.total_items > sms and p.plan.patches_per_split > 6
    if det:
        assert nat.load().osvos_wgrad_deterministic_splits(p.n, p.h, p.w, p.cin, p.dz) == p.plan.splits
    dw = profiled(p.run, {("wgrad_tc_kernel", (128, 1 if fast else 2, det)): 1})
    p.check(dw)
    if det:
        assert torch.equal(dw, p.run()), "deterministic weight gradient differs between two launches"


def test_wgrad_deferred_finish_accumulates(dev, sms):
    """Deferred launches of several mixed layers plus ONE ops.wgrad_finish with accumulate=True equal the direct calls
    plus the prior contents: bit-exact for deterministic layers, within fp32 reassociation for atomic ones."""
    from osvos_pytorch_b200 import ops
    layers = [WgradProblem("tap_rows", "splits", False, True, sms, dev, 1),
              WgradProblem("tap_pairs", "splits", False, False, sms, dev, 2),
              WgradProblem("nine_taps", "splits", True, True, sms, dev, 3),
              WgradProblem("nine_taps", "one_split", False, False, sms, dev, 4),
              WgradProblem("nine_taps", "many_items", False, False, sms, dev, 5)]
    g = torch.Generator().manual_seed(9)
    items, direct, prior = [], [], []
    for p in layers:
        direct.append(p.run())
        ws = torch.zeros(ops.wgrad_workspace_floats(p.dz, p.cin, (p.n, p.h, p.w), p.det), device=dev)
        item = p.run(deferred_ws=ws)
        pr = torch.randn(p.dz, p.cin, 3, 3, generator=g).to(dev)
        item["dw"], item["accumulate"] = pr.clone(), True
        items.append(item)
        prior.append(pr)
    ops.wgrad_finish(items)
    torch.cuda.synchronize()
    for p, it, d, pr in zip(layers, items, direct, prior):
        p.check(d)
        if p.det:
            assert torch.equal(it["dw"], d + pr)
        else:
            want = d.double() + pr.double()
            slack = 2 * p.tol * p.ref.abs().max().item() + U * want.abs().max().item()
            assert (it["dw"].double() - want).abs().max().item() <= slack


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("fast", [False, True])
def test_wgrad_refuses_192_output_channels(dev, fast, det):
    """192 output channels are not a whole number of 128-row m blocks.  With a workspace present the launch reaches
    plan_wgrad, which refuses it as OSVOS_ERR_UNSUPPORTED (status 3) before anything is enqueued: no kernel runs and
    the workspace keeps its contents.  The deterministic workspace size of such a shape is 0
    (osvos_wgrad_workspace_bytes with OSVOS_FLAG_DETERMINISTIC), so the immediate deterministic call has no workspace
    and is refused earlier, as an invalid argument (status 1)."""
    from osvos_pytorch_b200 import _native as nat, ops
    g = torch.Generator().manual_seed(3)
    x = ops.nchw_to_act(torch.randn(1, 128, 9, 11, generator=g).to(dev), fast)
    dz = ops.nchw_to_act(torch.randn(1, 192, 9, 11, generator=g).to(dev), fast)
    assert nat.load().osvos_wgrad_workspace_bytes(1, 9, 11, 128, 192, nat.FLAG_DETERMINISTIC) == 0
    ws = torch.full((ops.wgrad_workspace_floats(192, 128, (1, 9, 11)),), 7.0, device=dev)
    with KernelsRan() as k:
        with pytest.raises(nat.NativeLibraryError, match="failed with status 3"):
            ops.conv3x3_wgrad(x, dz, 192, fast=fast, deferred_ws=ws, deterministic=det)
        with pytest.raises(nat.NativeLibraryError, match=f"failed with status {1 if det else 3}"):
            ops.conv3x3_wgrad(x, dz, 192, fast=fast, deterministic=det)
    assert not any(name == "wgrad_tc_kernel" for name, _ in k.counts), k.counts
    assert bool((ws == 7.0).all())

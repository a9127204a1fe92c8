"""Every launch regime of the side-branch, unpool and tail kernels, at the running device's SM count, against fp64 of the
operands the kernels read.  tests/side_dispatch_ref.py restates the plans and finds a small shape for each regime;
torch.profiler confirms which instantiation each launch ran and how many times.

- side_conv_kernel<PLANES, NCO>: {exact, fast} x {NCO 2 (folded side branch), NCO 16 (side_prep)} x {tiles <= SMs,
  tiles > 2 SMs with CTAs running both odd and even tile counts}, and NCO = 2 launches of 2, 3 and 4 scales in which a
  CTA's tile walk crosses from one scale (and chunk count) into the next.
- side_folded_wgrad_kernel<DET>: {atomic, deterministic} x {exact, fast} x {one chunk per block, a ring that wraps with
  uneven chunk counts, a multi-scale launch with a scale clamped to one block per slab, rows narrower than a chunk}.
- unpool_add_mask_kernel<POOL, SIDE, DET>: all eight through osvos_unpool_mask, with the folded weights in global
  and in shared memory, at c = 64 .. 512, more tiles than CTAs, odd sizes, tied window maxima, +-0 and negative x.
- tail_fwd_kernel<DET>: more rows than blocks, odd width, with and without a label, output and label planes 16-byte
  aligned and 4 bytes off.

Bounds.  U = 2^-23 is the unit of one fp32 rounding.  An output that the kernel forms by `steps` fp32 roundings of
running sums of terms t_i is within steps * U * sum |t_i| of the exact sum of the terms it read (each rounding errs by at
most U of its result, and every partial result is at most sum |t_i|).  Each check normalises by sum |t_i| per output,
computed in fp64 from the absolute values of the operands, so it also holds where the output cancels.  Step counts:
- side convolution: the wgmma K steps of 16 that add into the accumulator (4 per 64-channel chunk and pass; passes = 3
  exact, 1 fast), + 9 for the shift-add of the taps, + 1 for the bias; pq of NCO = 16 adds 16 FMAs of the projections,
  over the terms |proj_w| x (sum |t_i| of the features).
- folded G and S: 4 FMAs per chunk a block walks (a compute warp takes 4 pixels of a chunk), + 7 for the warps'
  partials, + one per block of the slab (atomics into G), + the ordered row reduction's depth under DET.
- unpool with SIDE: the 18 FMAs of W' x dpq and the add of the selected dpool, 19; the store then splits the value into
  bf16 hi + lo (relative error 2^-16; fast mode stores bf16 hi only, half a bf16 unit), which the check allows on top of
  the bound (_store_rounding).  Without SIDE the kernel adds two fp32 values once, which host fp32 arithmetic
  reproduces: that dz is compared bit for bit.
- column sums: a recursive sum of the fp32 pre-store values, depth = (window positions x tiles per block) + the block's
  pixel lanes + the grid's atomics (or the ordered row reduction under DET); the bound is the values' own error plus
  depth * U * sum |value| per channel.
- tail maps: the two-tap vertical and horizontal blends, 4 roundings; the fused map adds the four scales' q blends to the
  bias, 5 roundings per scale.  The bilinear weights are positive, so the maps of |pq| and |bias| are sum |t_i|.
- tail sums: depth = pixels per thread + 5 shuffle levels + 2, plus E = 8 + 1.2 max |x| for the terms themselves:
  __expf(x) errs by up to 2 + 1.173 |x| units (CUDA programming guide), log1pf, the division and the subtractions by a
  few more.  Each term is normalised by |softplus(x)| + |x| (the loss terms) or |sigmoid(x)| + 1 (the bias-gradient
  terms), which bound its partial results.
At module end each family reports its largest share of the bound."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import side_dispatch_ref as sdr
from test_gpu_conv_schedules import KernelsRan, _nchw, _weights_seen

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
MEASURED = {}
BLIND = []          # launches whose profiler window held no device record at all


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


@pytest.fixture(scope="module", autouse=True)
def _report_measured():
    yield
    for family, v in sorted(MEASURED.items()):
        print(f"\n{family}: largest share of its bound {max(v):.3f} ({len(v)} checks)")
    if BLIND:
        print(f"\nprofiler windows without any device record (instantiation not confirmed): {len(BLIND)}")


def ran(fn, expected):
    """fn() under KernelsRan with the kernels of tests/side_dispatch_ref.py: they must be exactly ``expected``
    ({(kernel, template args): launches}).  A window that loses a record is run again, at most twice, as in
    test_gpu_conv_schedules.profiled.  Late in a long process (the whole GPU suite, after other files have captured and
    replayed CUDA graphs) torch.profiler can go blind: a window records the launch calls but no device activity at all.
    Such a window cannot tell which kernel ran; it is counted in BLIND and reported at module end, and the results
    are still checked.  A window that records a wrong instantiation fails."""
    for _ in range(3):
        with KernelsRan(sdr.parse_side_kernel_name) as k:
            out = fn()
        if sum(k.counts.values()) >= sum(expected.values()):
            break
    if not k.counts and not any(dev == "CUDA" for _, dev, _ in k.seen):
        BLIND.append(sorted(expected))
        return out
    assert k.counts == expected, (k.counts, k.seen[:12])
    return out


def check_bound(family, got, ref, bound, what, slack=None):
    """max (|got - ref| - slack) / bound <= 1 elementwise (bound > 0, or got == ref exactly where bound == 0).
    ``slack``: a known rounding of the stored output, outside the share the family reports."""
    got, ref, bound = got.double(), ref.double(), bound.double()
    err = (got - ref).abs()
    if slack is not None:
        err = (err - slack.double()).clamp(min=0)
    exact = bound == 0
    assert bool((err[exact] == 0).all()), (what, "outputs with a zero bound differ")
    share = (err[~exact] / bound[~exact]).max().item() if bool((~exact).any()) else 0.0
    MEASURED.setdefault(family, []).append(share)
    assert share <= 1.0, (what, share)
    return share


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------ side convolution
def _side_terms(a, wp, nco, cin, fast):
    """(fp64 convolution of the seen planes, fp64 convolution of their absolute values) of one scale, NCHW."""
    w_hi, w_lo = _weights_seen(wp, nco, cin)
    x_hi = _nchw(a.hi)
    lin = F.conv2d(x_hi, w_hi, padding=1)
    mag = F.conv2d(x_hi.abs(), w_hi.abs(), padding=1)
    if not fast:
        x_lo = _nchw(a.lo)
        lin = lin + F.conv2d(x_hi, w_lo, padding=1) + F.conv2d(x_lo, w_hi, padding=1)
        mag = mag + F.conv2d(x_hi.abs(), w_lo.abs(), padding=1) + F.conv2d(x_lo.abs(), w_hi.abs(), padding=1)
    return lin, mag


def _side_steps(cin, fast):
    return 4 * (cin // 64) * (1 if fast else 3) + 9 + 1


class SideScale:
    """Seeded stage output and side-branch weights of one scale, folded (NCO = 2) or literal (NCO = 16)."""
    def __init__(self, n, h, w, cin, nco, fast, dev, seed):
        from osvos_pytorch_b200 import ops
        g = _gen(seed)
        self.n, self.h, self.w, self.cin, self.nco, self.fast = n, h, w, cin, nco, fast
        x = torch.randn(n, cin, h, w, generator=g) * 2.0
        side_w = torch.randn(16, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
        side_b = torch.randn(16, generator=g) * 0.1
        self.proj = (torch.randn(32, generator=g) * 0.5).to(dev)
        self.proj_b = (torch.randn(1, generator=g) * 0.1).to(dev)
        self.a = ops.nchw_to_act(x.to(dev), fast)
        if nco == 2:
            (self.wp, self.bias, _), = ops.fold_side_weights_multi(
                [(side_w.to(dev), side_b.to(dev), self.proj, self.proj_b)], want_f32=False)
        else:
            self.wp, self.bias = ops.pack_conv3x3_weights(side_w.to(dev)), side_b.to(dev)
        torch.cuda.synchronize()
        lin, mag = _side_terms(self.a, self.wp, nco, cin, fast)
        b = self.bias.double().view(1, -1, 1, 1)
        self.ref, self.mag = lin + b, mag + b.abs()        # [n, nco, h, w]
        self.steps = _side_steps(cin, fast)

    def check_pq(self, pq, family):
        got = pq.permute(0, 3, 1, 2)
        if self.nco == 2:
            return check_bound(family, got, self.ref, self.steps * U * self.mag, "pq")
        pw = self.proj.double().view(2, 16)
        ref = torch.einsum("of,nfhw->nohw", pw, self.ref)
        ref[:, 0] += self.proj_b.double()
        mag = torch.einsum("of,nfhw->nohw", pw.abs(), self.mag)
        mag[:, 0] += self.proj_b.double().abs()
        return check_bound(family, got, ref, (self.steps + 16) * U * mag, "pq of the features")


SIDE_TARGETS = [(nco, fast, regime) for nco in (2, 16) for fast in (False, True) for regime in sdr.SIDE_REGIMES]


@pytest.mark.parametrize("target", SIDE_TARGETS,
                         ids=[f"nco{c}-{'fast' if f else 'exact'}-{r}" for c, f, r in SIDE_TARGETS])
def test_side_conv_schedule(dev, sms, target):
    from osvos_pytorch_b200 import ops
    nco, fast, regime = target
    n, h, w = sdr.find_side_shape(regime, sms)
    cin = 128
    plan = sdr.side_conv_plan([(n, h, w, cin, nco)], fast, sms)
    counts = {len(t) for t in plan.cta_tiles}
    assert counts == {1} if regime == "one_wave" else {c % 2 for c in counts} == {0, 1}
    s = SideScale(n, h, w, cin, nco, fast, dev, 100 + nco + w)
    family = f"side conv nco{nco} {'fast' if fast else 'exact'}"
    if nco == 2:
        pq = ran(lambda: ops.side_folded(s.a, s.wp, s.bias, fast), {("side_conv_kernel", plan.inst): 1})
        s.check_pq(pq, family)
        return
    _, feat, pq = ran(lambda: ops.conv3x3(s.a, s.wp, s.bias, 16, fast=fast, out_act=False, out_f32=True,
                                          proj_w=s.proj, proj_b=s.proj_b),
                      {("side_conv_kernel", plan.inst): 1})
    check_bound(family, feat.permute(0, 3, 1, 2), s.ref, s.steps * U * s.mag, "features")
    s.check_pq(pq, family)


SIDE_MULTI_TARGETS = [(count, fast) for count in (2, 3, 4) for fast in (False, True)]


@pytest.mark.parametrize("target", SIDE_MULTI_TARGETS,
                         ids=[f"{c}scales-{'fast' if f else 'exact'}" for c, f in SIDE_MULTI_TARGETS])
def test_side_conv_scales_in_one_launch(dev, sms, target):
    """The scales are passed shallowest first (the network's order); the launch runs them deepest first."""
    from osvos_pytorch_b200 import ops
    count, fast = target
    n, h, w = sdr.find_side_multi_shape(count, sms)
    shapes = sdr.multi_scale_shapes(h, w, count)[::-1]
    plan = sdr.side_conv_plan([(n, hh, ww, c, 2) for hh, ww, c in shapes], fast, sms)
    assert sdr.crossing_ctas(plan) and [s[3] for s in plan.scales] == sorted((c for _, _, c in shapes), reverse=True)
    scales = [SideScale(n, hh, ww, c, 2, fast, dev, 300 + 7 * k + ww) for k, (hh, ww, c) in enumerate(shapes)]
    pqs = ran(lambda: ops.side_folded_multi([s.a for s in scales], [(s.wp, s.bias) for s in scales], fast),
              {("side_conv_kernel", plan.inst): 1})
    for s, pq in zip(scales, pqs):
        s.check_pq(pq, f"side conv nco2 {'fast' if fast else 'exact'}")


# ------------------------------------------------------------------------------------------------ folded side G
SW_TARGETS = [(det, fast, regime) for det in (False, True) for fast in (False, True) for regime in sdr.SW_REGIMES]


def _g_reference(a, dpq):
    """G [9][2][c] and S [2] in fp64 of what the kernel reads, x = fp32(hi + lo), and the same over absolute values."""
    x = a.hi.float() + (a.lo.float() if a.lo is not None else 0.0)
    x = x.double()
    d = dpq.double()
    n, h, w, _ = x.shape
    dpad = F.pad(d, (0, 0, 1, 1, 1, 1))
    G, M = [], []
    for r in range(3):
        for s in range(3):
            win = dpad[:, 2 - r:2 - r + h, 2 - s:2 - s + w]          # dpq[y + 1 - r][x + 1 - s]
            G.append(torch.einsum("nhwo,nhwc->oc", win, x))
            M.append(torch.einsum("nhwo,nhwc->oc", win.abs(), x.abs()))
    return torch.stack(G), torch.stack(M), d.sum((0, 1, 2)), d.abs().sum((0, 1, 2))


@pytest.mark.parametrize("target", SW_TARGETS,
                         ids=[f"{'det' if d else 'atomic'}-{'fast' if f else 'exact'}-{r}" for d, f, r in SW_TARGETS])
def test_side_folded_wgrad(dev, sms, target):
    from osvos_pytorch_b200 import ops
    det, fast, regime = target
    items = sdr.find_sw_items(regime, sms)
    plan = sdr.side_wgrad_plan(items, sms)
    g = _gen(700 + len(regime) + items[0][1])
    xs, dpqs = [], []
    for n, h, w, c in items:
        xs.append(ops.nchw_to_act((torch.randn(n, c, h, w, generator=g) * 2.0).to(dev), fast))
        dpqs.append(torch.randn(n, h, w, 2, generator=g).to(dev))

    def launch():
        gs = [torch.zeros(ops.side_folded_wgrad_floats(c), device=dev) for _, _, _, c in items]
        ops.side_folded_wgrad_multi(xs, dpqs, gs, deterministic=det)
        return gs
    gs = ran(launch, {("side_folded_wgrad_kernel", (det,)): 1})
    if det:
        assert all(torch.equal(a, b) for a, b in zip(gs, launch())), "deterministic G differs between two launches"
    family = f"folded G {'det' if det else 'atomic'} {'fast' if fast else 'exact'}"
    for (n, h, w, c), sc, x, dpq, gb in zip(items, plan.scales, xs, dpqs, gs):
        steps = 4 * sc.chunks_per_block[0] + 7 + sc.blocks_per_slab
        if det:
            steps += sdr.reduce_rows_depth(sc.blocks_per_slab)
        G, M, S, MS = _g_reference(x, dpq)
        check_bound(family, gb[:18 * c].view(9, 2, c), G, steps * U * M, f"G of {(n, h, w, c)}")
        check_bound(family, gb[18 * c:], S, steps * U * MS, f"S of {(n, h, w, c)}")


# ------------------------------------------------------------------------------------------------ unpool
UNPOOL_TARGETS = [(t, c) for t in sdr.unpool_targets() for c in sdr.UNPOOL_CHANNELS]


def _unpool_id(t, c):
    pool, side, det, wf = t
    return (f"{'pool' if pool else 'nopool'}-{'side' if side else 'dside'}-{'det' if det else 'atomic'}"
            f"{'-wf_smem' if wf else ''}-c{c}")


def _window_select(x32, h, w):
    """[n,h,w,c] bool: the first maximum in (dy, dx) scan order of each ceil-mode 2x2 window of x32 ([n,h,w,c])."""
    n, _, _, c = x32.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    xp = F.pad(x32, (0, 0, 0, 2 * ow - w, 0, 2 * oh - h), value=float("-inf")).view(n, oh, 2, ow, 2, c)
    vals = [xp[:, :, q >> 1, :, q & 1] for q in range(4)]
    best = torch.stack(vals).amax(0)
    first = torch.full_like(best, 4, dtype=torch.int64)
    for q in (3, 2, 1, 0):
        first = torch.where(vals[q] == best, q, first)
    sel = torch.empty(n, oh, 2, ow, 2, c, dtype=torch.bool, device=x32.device)
    for q in range(4):
        sel[:, :, q >> 1, :, q & 1] = first == q
    return sel.view(n, 2 * oh, 2 * ow, c)[:, :h, :w]


def _upsample(t, h, w):
    return t.repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :h, :w]


class UnpoolProblem:
    def __init__(self, pool, side, det, c, n, h, w, fast, dev, seed):
        from osvos_pytorch_b200 import ops
        g = _gen(seed)
        self.n, self.h, self.w, self.c, self.pool, self.side, self.fast = n, h, w, c, pool, side, fast
        # x: half tie-prone values (a few levels, so windows often hold equal maxima, +-0 among them), half random
        levels = (torch.randint(-2, 4, (n, c, h, w), generator=g).float() * 0.5)
        x = torch.where(torch.rand(n, c, h, w, generator=g) < 0.5, levels, torch.randn(n, c, h, w, generator=g))
        flat = x.view(-1)
        flat[::13] = -0.0
        flat[5::17] = 0.0
        self.x = ops.nchw_to_act(x.to(dev), fast)
        oh, ow = (h + 1) // 2, (w + 1) // 2
        self.dpool = ops.nchw_to_act(torch.randn(n, c, oh, ow, generator=g).to(dev), fast) if pool else None
        dside = torch.randn(n, h, w, c, generator=g)
        dside.view(-1)[::11] = -0.0
        self.dside = dside.to(dev)
        self.dpq = (torch.randn(n, h, w, 2, generator=g) * 0.5).to(dev)
        self.wfold = (torch.randn(9, 2, c, generator=g) * 0.1).to(dev)
        torch.cuda.synchronize()
        zero = torch.zeros((), device=dev)
        x32 = self.x.hi.float() + (self.x.lo.float() if self.x.lo is not None else zero)
        self.mask = x32 > 0
        if pool:
            dpv = self.dpool.hi.float() + (self.dpool.lo.float() if self.dpool.lo is not None else zero)
            self.sel_dpool = torch.where(_window_select(x32, h, w), _upsample(dpv, h, w), zero)
        else:
            self.sel_dpool = torch.zeros(n, h, w, c, device=dev)

    def value(self, dside):
        """SIDE = false: the fp32 value the kernel stores (split) - fp32(dside + selected dpool), masked."""
        ds = dside if dside is not None else torch.zeros_like(self.sel_dpool)
        return torch.where(self.mask, ds + self.sel_dpool, torch.zeros((), device=ds.device))

    def side_ref(self):
        """SIDE = true: (fp64 reference, fp64 sum |terms|) of the pre-store value, masked."""
        wt = self.wfold.double().view(3, 3, 2, self.c).permute(2, 3, 0, 1)       # [o][c][r][s]
        d = self.dpq.double().permute(0, 3, 1, 2)
        dx = F.conv_transpose2d(d, wt, padding=1).permute(0, 2, 3, 1)
        mag = F.conv_transpose2d(d.abs(), wt.abs(), padding=1).permute(0, 2, 3, 1)
        sel = self.sel_dpool.double()
        m = self.mask
        return (dx + sel) * m, (mag + sel.abs()) * m

    def colsum_depth(self, plan, det):
        per_thread = (4 if self.pool else 1) * -(-plan.tiles // plan.grid)
        return per_thread + plan.ppb + (sdr.reduce_rows_depth(plan.grid) if det else plan.grid)


def _split_planes(v, fast):
    hi = v.to(torch.bfloat16)
    lo = None if fast else (v - hi.float()).to(torch.bfloat16)
    return hi, lo


def _store_rounding(got, fast):
    """A bound on |v - got| for a stored dz = got of a value v: half a bf16 unit of got in fast mode (v rounds to got,
    and no value of a lower binade rounds up by more); in exact mode 2^-16 |v| for hi + lo, |v| <= |got| / (1 - 2^-16)."""
    if fast:
        _, ex = torch.frexp(got)                        # got = m 2^ex, 0.5 <= |m| < 1: unit 2^(ex - 8)
        return torch.where(got == 0, torch.zeros_like(got), torch.ldexp(torch.ones_like(got), ex - 9))
    return got.abs() * (2.0 ** -16 / (1 - 2.0 ** -16))


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("fast", [False, True], ids=["exact", "fast"])
@pytest.mark.parametrize("target,c", UNPOOL_TARGETS, ids=[_unpool_id(t, c) for t, c in UNPOOL_TARGETS])
def test_unpool_mask(dev, sms, target, c, fast):
    from osvos_pytorch_b200 import ops
    pool, side, det, wf = target
    n, h, w = sdr.find_unpool_shape(pool, side, det, wf, c, sms)
    plan = sdr.unpool_plan(n, h, w, c, pool, side, det, sms)
    assert plan.tiles > plan.grid and plan.wf_in_smem == wf
    p = UnpoolProblem(pool, side, det, c, n, h, w, fast, dev, 900 + c + h + 2 * pool + side)
    dpool = p.dpool if pool else None
    inst = ("unpool_add_mask_kernel", (pool, side, det))
    family = f"unpool {'side' if side else 'dside'} {'fast' if fast else 'exact'}"

    def zeros():
        return torch.zeros(c, device=dev)

    if side:
        def launches():
            cs = zeros()
            return [(ops.unpool_mask(dpool, p.x, dpq=p.dpq, wfold=p.wfold, colsum=cs, deterministic=det), cs)]
    else:
        def launches():                 # with and without the fp32 side map; without dpool the map is the only consumer
            runs = []
            for ds in ((p.dside, None) if pool else (p.dside,)):
                cs = zeros()
                runs.append((ops.unpool_mask(dpool, p.x, dside=ds, colsum=cs, deterministic=det), cs, ds))
            return runs
    runs = ran(launches, {inst: 2 if pool and not side else 1})
    depth = p.colsum_depth(plan, det)
    for run in runs:
        dz, cs = run[0], run[1]
        if side:
            ref, mag = p.side_ref()
            vb = 19 * U * mag                               # bound of the pre-store value v
            got = dz.hi.float() + (dz.lo.float() if dz.lo is not None else 0.0)
            check_bound(family, got, ref, vb, "dz", slack=_store_rounding(got, fast))
            cs_ref, cs_bound = ref.sum((0, 1, 2)), vb.sum((0, 1, 2)) + depth * U * (ref.abs() + vb).sum((0, 1, 2))
        else:
            v = p.value(run[2])
            hi, lo = _split_planes(v, fast)
            assert torch.equal(_bits(dz.hi), _bits(hi)), "dz hi differs from bf16(fp32(dside + selected dpool))"
            assert (dz.lo is None) == fast and (fast or torch.equal(_bits(dz.lo), _bits(lo)))
            cs_ref, cs_bound = v.double().sum((0, 1, 2)), depth * U * v.double().abs().sum((0, 1, 2))
        check_bound("unpool column sums", cs, cs_ref, cs_bound, "column sums")
    if det:
        again = launches()
        assert all(torch.equal(a[1], b[1]) for a, b in zip(runs, again)), "deterministic column sums differ"


# ------------------------------------------------------------------------------------------------ tail forward
TAIL_TARGETS = [("nolabel", False, off) for off in (0, 4)] + \
    [("label", det, off) for det in (False, True) for off in (0, 4)]


@pytest.mark.parametrize("target", TAIL_TARGETS,
                         ids=[f"{m}{'-det' if d else ''}-offset{o}" for m, d, o in TAIL_TARGETS])
def test_tail_fwd(dev, sms, target):
    from oracle import osvos_oracle as oc
    from osvos_pytorch_b200 import ops
    from test_gpu_objective import _ref_maps
    mode, det, off = target
    n, h, w = sdr.find_tail_shape(sms)
    blocks = sdr.tail_fwd_blocks(n, h, sms)
    assert n * h > blocks and w % 2 == 1
    g = _gen(1234 + off + 2 * det)
    pqs, hk, wk = [], h, w
    for _ in range(4):
        hk, wk = oc.pooled_size(hk), oc.pooled_size(wk)
        pqs.append(torch.randn(n, hk, wk, 2, generator=g) * 4.0)
    fb = torch.randn(1, generator=g)
    npix = n * h * w
    per = (npix + 3) // 4 * 4
    obuf = torch.empty(5, per + 4, device=dev)
    out = obuf[:, off // 4:off // 4 + npix].view(5, n, 1, h, w)
    assert all(out[k].data_ptr() % 16 == off for k in range(5))
    label = None
    if mode == "label":
        lbuf = torch.empty(npix + 4, device=dev)
        label = lbuf[off // 4:off // 4 + npix].view(n, 1, h, w)
        label.copy_((torch.rand(n, 1, h, w, generator=g) > 0.6).float())
        assert label.data_ptr() % 16 == off
    weights, divisor = (0.5, 0.25, 0.75, 1.0, 1.5), float(n)
    d_pqs, d_fb = [p.to(dev) for p in pqs], fb.to(dev)

    def launch():
        if label is None:
            return ops.tail_fwd(d_pqs, d_fb, n, h, w, out=out, deterministic=det)
        return ops.tail_fwd(d_pqs, d_fb, n, h, w, label=label, out=out, loss_weights=weights, divisor=divisor,
                            deterministic=det)
    res = ran(launch, {("tail_fwd_kernel", (det,)): 1})
    got_maps = out.cpu().double()
    ref = _ref_maps([p.double() for p in pqs], fb.double(), h, w)
    mag = _ref_maps([p.double().abs() for p in pqs], fb.double().abs(), h, w)
    for k in range(5):
        steps = 4 if k < 4 else 20
        check_bound("tail maps", got_maps[k], ref[k], steps * U * mag[k], f"map {k}")
    if label is None:
        assert res[1] is None
        return
    _, sums, losses = res
    if det:
        o2, s2, l2 = launch()
        assert torch.equal(sums[:14], s2[:14]) and torch.equal(losses, l2) and torch.equal(o2.cpu().double(), got_maps)
    sums, losses = sums.cpu(), losses.cpu().double()
    lab = label.cpu().double() >= 0.5
    x = got_maps                                                         # the maps the sums are formed from
    sp = x.clamp(min=0) + torch.log1p(torch.exp(-x.abs()))
    groups = -(-(w + 3) // 4)                                            # pixel groups of four per row, at most
    per_thread = 4 * -(-groups // 256) * -(-(n * h) // blocks)
    e_terms = 8 + 1.2 * x.abs().max().item()
    depth = per_thread + 5 + 2 + e_terms
    want, bound = [], []
    for k in range(5):
        term_mag = sp[k] + x[k].abs()
        want += [(sp[k] - x[k])[lab].sum(), sp[k][~lab].sum()]
        bound += [depth * U * term_mag[lab].sum(), depth * U * term_mag[~lab].sum()]
    P, N = lab.sum().item(), npix
    sg = torch.sigmoid(x[4])
    a_pos, a_neg = (sg - 1)[lab].sum(), sg[~lab].sum()
    a_bound = [depth * U * (sg + 1)[lab].sum(), depth * U * (sg + 1)[~lab].sum()]
    check_bound("tail sums", sums[:10], torch.stack(want), torch.stack(bound), "loss sums")
    assert sums[10].item() == P and sums[11].item() == N
    check_bound("tail sums", sums[12:14], torch.stack([a_pos, a_neg]), torch.stack(a_bound), "bias-gradient sums")
    lw, lb = [], []
    for k in range(5):
        lk = ((N - P) / N * want[2 * k] + P / N * want[2 * k + 1]) / divisor
        lw.append(lk)
        lb.append(((N - P) / N * bound[2 * k] + P / N * bound[2 * k + 1]) / divisor + 2 * U * abs(lk))
    total = sum(wt * l for wt, l in zip(weights, lw))
    tb = sum(wt * b for wt, b in zip(weights, lb)) + U * abs(total)
    check_bound("tail losses", losses, torch.stack(lw + [total]), torch.stack(lb + [tb]), "losses")

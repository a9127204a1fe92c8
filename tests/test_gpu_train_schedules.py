"""Every launch regime of the kernels at both ends of a training step, at the running device's SM count, against fp64 of
the operands the kernels read.  tests/train_dispatch_ref.py restates the plans and finds a small shape for each regime;
torch.profiler confirms which kernels each call ran and how many times.

- conv_first_tc_kernel<PLANES, STAGED>: {exact, fast} x {16-byte aligned output planes (TMA-staged stores), planes 4
  bytes off (direct stores)} x {tiles <= SMs, tiles > 3 SMs dealt unevenly over five images}, ReLU on and off, x about
  +-128 like a normalised frame.
- conv_first_wgrad_kernel<DET> and conv_first_dgrad_kernel: {atomic, deterministic} x {exact, fast} x {tiles < 16,
  tiles <= 4 SMs, tiles > 8 SMs with uneven tiles per block} x {w < 64, w = 64 k, w = 64 k + 1}; n = 2, frame borders
  in every case and w > 128 (several dgrad x-blocks) at w = 64 k and 64 k + 1.
- tail_bwd2_kernel<LOSS, DET>: all four, over a set of widths whose segments reach every reachable (scale, rgroups)
  pair, an idle-thread width (wpad = 96), and full and short segments at scales 0 and 1; zero maps; with LOSS,
  fuse_bias_grad with the upstream gradient both null and set at every width.
- upsampling_fold_kernel: all 17 x 1360 table entries.  tail_general_fwd_kernel: n h <= 8 SMs with w > 256 (threads
  walk the row) and n h > 8 SMs (blocks stride rows), with and without a label; maps, the 13 sums and six losses.
- cbce_fwd_kernel<DET> and cbce_bwd_kernel: numel 1 - 3 (no vector), one block, and a capped grid with three vectors
  per thread, each with numel % 4 = 1, 2, 3 and 0; all-positive, all-negative and exactly-0.5 labels.
- sum_f32 (both forms) and osvos_reduce_rows at nrows 1, 63, 64, 65 and 4100, ncols not a multiple of 32, with
  accumulate.

Bounds.  U = 2^-23 is the unit of one fp32 rounding.  An output the kernel forms by `steps` fp32 roundings of running
sums of terms t_i is within steps * U * sum |t_i| of the exact sum of the terms it read, computed here in fp64 from the
absolute values of the operands, so the check also holds where the output cancels.  Step counts:
- conv1_1 forward: two wgmma K steps of 16 per pass (three passes exact: x_hi w_hi + x_lo w_hi + x_hi w_lo; one fast:
  x_hi w_hi), + 1 for the bias.  The store splits the value into bf16 hi + lo (or hi only in fast mode), which the
  check allows on top (_store_rounding).  The host restates the split: hi = bf16(v), lo = bf16(v - hi).
- conv1_1 weight gradient: 4 mma k-steps per pass and tile (three passes exact: x_hi dz_hi + x_hi dz_lo + x_lo dz_hi;
  two fast: x_hi dz_hi + x_lo dz_hi) times the tiles of the busiest block, + the replica atomics (ceil(grid / 16)) and
  the 16-replica sum, or + the ordered row reduction's depth under DET.
- conv1_1 data gradient: 9 taps x 64 channels of FMAs, 576, over the fp32 weights and dz = hi + lo (exact in fp32).
- tail backward: per scale, the largest depth over its items of ceil(2s / rgroups) phase-1 FMAs + rgroups adds into
  shared memory + ceil(2s / lanes) phase-2 FMAs + log2(lanes) shuffles + 1 for the scaling.  With LOSS the gradient maps
  are formed from logits and label: + 3 for the class weight and coefficient products, and E = 8 + 1.2 max |x| for
  __expf (which errs by up to 2 + 1.173 |x| units) and the division; the terms are normalised by |c| w (sigmoid + 1).
- upsampling fold: V is 16 FMAs over |f| |U|; A is a copy, compared bit for bit.  General tail forward: the side maps
  4 FMAs, the fused map the bias + 4 scales x 4 sources x 16 channels = 257; its sums as the tail forward's, with the
  pixels per thread = ceil(w / 256) x rows per block.
- cbce forward: depth = 4 x vectors per thread + 1 (the scalar tail) + 5 shuffle levels + 8 warps + the blocks (fp64
  atomics, or the ordered sum: ceil(blocks / 256) + 256) + E, over |softplus(x)| + |x| per term; the loss adds 2 U.
  cbce backward: E + 6 roundings of |w g| (sigmoid + 1) per element.
- sum_f32: the elements per thread + 5 shuffle levels + 1 (the fp32 result); deterministic: the elements per thread
  + 256 threads + 256 blocks in order + 1.  reduce_rows: side_dispatch_ref.reduce_rows_depth.
At module end each family reports its largest share of the bound."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import train_dispatch_ref as tdr
from test_gpu_conv_schedules import KernelsRan
from test_gpu_side_schedules import _store_rounding

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
        print(f"\nprofiler windows without any device record (kernels not confirmed): {len(BLIND)}")


def ran(fn, expected):
    """fn() under KernelsRan with the kernels of tests/train_dispatch_ref.py: they must be exactly ``expected``
    ({(kernel, template args): launches}).  As in test_gpu_side_schedules.ran: a window that loses a record is run
    again, at most twice; a window with no device record at all (torch.profiler gone blind late in a long process) is
    counted in BLIND and its results are still checked; a window that records a wrong kernel fails."""
    for _ in range(3):
        with KernelsRan(tdr.parse_train_kernel_name) as k:
            out = fn()
        if sum(k.counts.values()) >= sum(expected.values()):
            break
    if not k.counts and not any(d == "CUDA" for _, d, _ in k.seen):
        BLIND.append(sorted(expected))
        return out
    assert k.counts == expected, (k.counts, k.seen[:12])
    return out


def check_bound(family, got, ref, bound, what, slack=None):
    """max (|got - ref| - slack) / bound <= 1 elementwise (bound > 0, or got == ref exactly where bound == 0).
    ``slack``: a known rounding of the stored output, outside the share the family reports."""
    got, ref, bound = got.double().cpu(), ref.double().cpu(), bound.double().cpu()
    err = (got - ref).abs()
    if slack is not None:
        err = (err - slack.double().cpu()).clamp(min=0)
    assert not bool(torch.isnan(got).any()), (what, "NaN in the output")
    exact = bound == 0
    assert bool((err[exact] == 0).all()), (what, "outputs with a zero bound differ")
    share = (err[~exact] / bound[~exact]).max().item() if bool((~exact).any()) else 0.0
    MEASURED.setdefault(family, []).append(share)
    assert share <= 1.0, (what, share)
    return share


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _split(v):
    """fp32 -> (hi, lo) as the kernels split it: hi = bf16(v), lo = bf16(v - hi), both as fp64."""
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    return hi.double(), lo.double()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ conv1_1 forward
FIRST_TARGETS = [(fast, staged, regime) for fast in (False, True) for staged in (True, False)
                 for regime in tdr.FIRST_REGIMES]


@pytest.mark.parametrize("target", FIRST_TARGETS,
                         ids=[f"{'fast' if f else 'exact'}-{'staged' if s else 'direct'}-{r}" for f, s, r in FIRST_TARGETS])
def test_conv_first_fwd(dev, sms, target):
    from osvos_pytorch_b200 import _native as nat
    fast, staged, regime = target
    n, h, w = tdr.find_first_shape(regime, sms)
    plan = tdr.conv_first_plan(n, h, w, fast, staged, sms)
    g = _gen(40 + w + 2 * fast + staged)
    x = torch.rand(n, 3, h, w, generator=g) * 256.0 - 128.0
    wt = torch.randn(64, 3, 3, 3, generator=g) * math.sqrt(2.0 / 27)
    b = torch.randn(64, generator=g) * 0.1
    d_x, d_w, d_b = x.to(dev), wt.to(dev), b.to(dev)
    numel = n * h * w * 64
    off = 0 if staged else 2                                  # bf16 elements: planes 4 bytes past an aligned address
    bufs = [torch.zeros(numel + 8, dtype=torch.bfloat16, device=dev) for _ in range(2)]
    hi, lo = (t[off:off + numel] for t in bufs)
    assert all((t.data_ptr() % 16 == 0) == staged for t in (hi, lo))
    x_hi, x_lo = _split(x)
    w_hi, w_lo = _split(wt)
    lin = F.conv2d(x_hi, w_hi, padding=1)
    mag = F.conv2d(x_hi.abs(), w_hi.abs(), padding=1)
    if not fast:
        lin = lin + F.conv2d(x_lo, w_hi, padding=1) + F.conv2d(x_hi, w_lo, padding=1)
        mag = mag + F.conv2d(x_lo.abs(), w_hi.abs(), padding=1) + F.conv2d(x_hi.abs(), w_lo.abs(), padding=1)
    bd = b.double().view(1, -1, 1, 1)
    ref, mag = lin + bd, mag + bd.abs()
    steps = 2 * (1 if fast else 3) + 1
    family = f"conv1_1 fwd {'fast' if fast else 'exact'}"
    for relu in (True, False):
        flags = (nat.FLAG_RELU if relu else 0) | (nat.FLAG_FAST if fast else 0)

        def launch():
            nat.check(nat.load().osvos_conv_first_fwd(d_x.data_ptr(), d_w.data_ptr(), d_b.data_ptr(), hi.data_ptr(),
                                                      None if fast else lo.data_ptr(), n, h, w, flags, _stream()),
                      "osvos_conv_first_fwd")
        ran(launch, {("conv_first_tc_kernel", plan.inst): 1})
        got = hi.float() + (0.0 if fast else lo.float())
        got = got.view(n, h, w, 64).permute(0, 3, 1, 2)
        want = ref.relu() if relu else ref
        check_bound(family, got, want, steps * U * mag, f"relu={relu}", slack=_store_rounding(got, fast))
        if fast:
            assert bool((bufs[1] == 0).all()), "fast mode wrote a lo plane"
        assert bool((bufs[0][:off] == 0).all()) and bool((bufs[0][off + numel:] == 0).all()), "wrote outside the planes"


# ------------------------------------------------------------------------------------------------ conv1_1 backward
FW_TARGETS = [(det, fast, regime, width) for det in (False, True) for fast in (False, True)
              for regime, width in tdr.fw_cases()]


def _wgrad_terms(x, dz_hi, dz_lo, fast):
    """(fp64 dW of the planes the kernel reads, the same over absolute values), [64, 3, 3, 3]."""
    x_hi, x_lo = _split(x)
    pairs = [(x_hi, dz_hi), (x_lo, dz_hi)] if fast else [(x_hi, dz_hi), (x_hi, dz_lo), (x_lo, dz_hi)]
    lin = sum(torch.nn.grad.conv2d_weight(a, (64, 3, 3, 3), d, padding=1) for a, d in pairs)
    mag = sum(torch.nn.grad.conv2d_weight(a.abs(), (64, 3, 3, 3), d.abs(), padding=1) for a, d in pairs)
    return lin, mag


@pytest.mark.parametrize("target", FW_TARGETS,
                         ids=[f"{'det' if d else 'atomic'}-{'fast' if f else 'exact'}-{r}-w{wd}"
                              for d, f, r, wd in FW_TARGETS])
def test_conv_first_bwd(dev, sms, target):
    from osvos_pytorch_b200 import ops
    det, fast, regime, width = target
    n, h, w = tdr.find_fw_shape(regime, width, sms)
    plan = tdr.first_wgrad_plan(n, h, w, sms)
    g = _gen(500 + h + w + 2 * fast)
    x = torch.rand(n, 3, h, w, generator=g) * 256.0 - 128.0
    dz = torch.randn(n, 64, h, w, generator=g) * 0.01
    wt = torch.randn(64, 3, 3, 3, generator=g) * math.sqrt(2.0 / 27)
    d_x, d_w = x.to(dev), wt.to(dev)
    a = ops.nchw_to_act(dz.to(dev), fast)
    torch.cuda.synchronize()
    dz_hi = a.hi.double().permute(0, 3, 1, 2).cpu()
    dz_lo = None if fast else a.lo.double().permute(0, 3, 1, 2).cpu()
    expected = {("conv_first_wgrad_kernel", (det,)): 1, ("conv_first_dgrad_kernel", ()): 1}
    if det:
        expected.update({("reduce_rows_segments_kernel", ()): 1, ("reduce_rows_final_kernel", ()): 1})
    dw, dx = ran(lambda: ops.conv_first_bwd(d_x, a, d_w, True, deterministic=det), expected)
    if det:
        dw2, dx2 = ops.conv_first_bwd(d_x, a, d_w, True, deterministic=True)
        assert torch.equal(dw, dw2) and torch.equal(dx, dx2), "deterministic conv1_1 backward differs between runs"
    ref, mag = _wgrad_terms(x, dz_hi, dz_lo, fast)
    per_block = max(len(t) for t in plan.block_tiles)
    steps = 4 * (2 if fast else 3) * per_block
    steps += tdr.reduce_rows_depth(plan.grid) if det else -(-plan.grid // tdr.FW_COPIES) + tdr.FW_COPIES
    check_bound(f"conv1_1 wgrad {'det' if det else 'atomic'} {'fast' if fast else 'exact'}", dw, ref, steps * U * mag,
                "dW")
    d = dz_hi + (dz_lo if dz_lo is not None else 0.0)
    wd = wt.double()
    dx_ref = F.conv_transpose2d(d, wd, padding=1)
    dx_mag = F.conv_transpose2d(d.abs(), wd.abs(), padding=1)
    check_bound("conv1_1 dgrad", dx, dx_ref, 576 * U * dx_mag, "dx")


# ------------------------------------------------------------------------------------------------ tail backward
def _adjoint(gmap, sc, h, w):
    """fp64 dpq channel of one scale from a full-resolution gradient map [n, 1, h, w]: the zero-padded bilinear
    deconvolution's adjoint, cropped as the forward crops."""
    s = sc.s
    f = torch.tensor([1.0 - abs(t - (s - 0.5)) / s for t in range(2 * s)], dtype=torch.float64)
    kern = (f[:, None] * f[None, :]).view(1, 1, 2 * s, 2 * s)
    full = torch.zeros(gmap.shape[0], 1, (sc.hk + 1) * s, (sc.wk + 1) * s, dtype=torch.float64)
    full[:, :, sc.top:sc.top + h, sc.left:sc.left + w] = gmap
    return F.conv2d(full, kern, stride=s)[:, 0]                  # [n, hk, wk]


TAIL_WIDTHS = tdr.find_tail_bwd_widths()
TAIL_TARGETS = [(w, loss, det, up) for w in TAIL_WIDTHS for loss in (False, True) for det in (False, True)
                for up in ((False, True) if loss else (False,))]


def _tail_id(w, loss, det, up):
    return f"w{w}-{'loss' if loss else 'grads'}-{'det' if det else 'atomic'}{'-upstream' if up else ''}"


@pytest.mark.parametrize("target", TAIL_TARGETS, ids=[_tail_id(*t) for t in TAIL_TARGETS])
def test_tail_bwd(dev, target):
    """``up``: LOSS with a device scalar d(total loss) = 0.7 that scales dpq and fuse_bias_grad (else null: 1)."""
    from osvos_pytorch_b200 import ops
    w, loss, det, with_upstream = target
    n, h = 2, 13
    scales, _ = tdr.tail_bwd_scales(n, h, w)
    items = tdr.tail_bwd_row_items(w)
    depth = [max(tdr.tail_bwd_depth(it) for it in items if it.scale == k) for k in range(4)]
    g = _gen(2000 + w + 2 * loss + det)
    npix = n * h * w
    if loss:
        logits = torch.randn(5, n, 1, h, w, generator=g) * 4.0
        label = (torch.randint(0, 3, (n, 1, h, w), generator=g).float() * 0.5)        # 0, 0.5 and 1
        pos = label >= 0.5
        P, N = float(pos.sum()), float(npix)
        sums = torch.zeros(tdr.TAIL_SUMS, dtype=torch.float64)
        sums[10], sums[11], sums[12], sums[13] = P, N, 37.25, -11.5
        weights, divisor = (0.5, 0.0, 0.75, 1.0, 1.5), 2.0
        upstream = torch.tensor([0.7], device=dev) if with_upstream else None
        up = float(torch.tensor(0.7, dtype=torch.float32)) if with_upstream else 1.0
        d_logits, d_label, d_sums = logits.to(dev), label.to(dev), sums.to(dev)
        (dpq, fb) = ran(lambda: ops.tail_loss_bwd(d_logits, d_label, d_sums, weights, divisor, upstream, n, h, w,
                                                  want_fuse_bias=True, deterministic=det),
                        {("tail_bwd2_kernel", (True, det)): 1})
        xd = logits.double()
        sg = torch.sigmoid(xd)
        cls = torch.where(pos, (N - P) / N, P / N).double()
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
        check_bound("tail bwd fuse bias", fb, torch.tensor([fb_ref]), torch.tensor([8 * U * fb_mag]), "fuse_bias_grad")
    else:
        grads = [torch.randn(n, 1, h, w, generator=g) for _ in range(5)]
        grads[1] = None                                                    # a scale without upstream gradient
        dpq = ran(lambda: ops.tail_bwd([None if t is None else t.to(dev) for t in grads], n, h, w, deterministic=det),
                  {("tail_bwd2_kernel", (False, det)): 1})
        maps = [torch.zeros(n, 1, h, w, dtype=torch.float64) if t is None else t.double() for t in grads]
        mags = [m.abs() for m in maps]
        extra = 0
    if det:
        again = (ops.tail_loss_bwd(d_logits, d_label, d_sums, weights, divisor, upstream, n, h, w,
                                   want_fuse_bias=True, deterministic=True)[0] if loss else
                 ops.tail_bwd([None if t is None else t.to(dev) for t in grads], n, h, w, deterministic=True))
        assert all(torch.equal(a_, b_) for a_, b_ in zip(dpq, again)), "deterministic dpq differs between runs"
    family = f"tail bwd {'loss' if loss else 'grads'} {'det' if det else 'atomic'}"
    for k, sc in enumerate(scales):
        got = dpq[k].cpu().double()
        steps = depth[k] + extra
        for ch, src in ((0, k), (1, 4)):
            ref = _adjoint(maps[src], sc, h, w)
            bound = steps * U * _adjoint(mags[src], sc, h, w)
            check_bound(family, got[..., ch], ref, bound, f"scale {k} channel {ch}")
        if k == 1:
            assert bool((got[..., 0] == 0).all()), "a zero-coefficient / absent map gave a non-zero dpq"


# ------------------------------------------------------------------------------------------------ general tail
def _gen_weights(seed, dev):
    """Random upscale[k] [16,16,2s,2s], upscale_[k] [1,1,2s,2s] and fuse.weight [64] (not the bilinear taps)."""
    g = _gen(seed)
    up = [(torch.randn(16, 16, 4 << k, 4 << k, generator=g) * 0.3).to(dev) for k in range(4)]
    up1 = [(torch.randn(1, 1, 4 << k, 4 << k, generator=g) * 0.3).to(dev) for k in range(4)]
    fw = (torch.randn(64, generator=g) * 0.5).to(dev)
    return up, up1, fw


_GEN_OFF = (0, 16, 80, 336)


def test_upsampling_fold(dev):
    """All 17 x 1360 entries: V_k[t][ci] = sum_co f[16k + co] U_k[ci][co][t] (16 FMAs) and A_k[t] copied."""
    from osvos_pytorch_b200 import ops
    up, up1, fw = _gen_weights(71, dev)
    tab = ran(lambda: ops.upsampling_fold(up, up1, fw), {("upsampling_fold_kernel", ()): 1}).cpu()
    V, A = tab[:16 * tdr.GEN_TAPS].view(tdr.GEN_TAPS, 16), tab[16 * tdr.GEN_TAPS:]
    f = fw.cpu().double()
    for k in range(4):
        taps = (4 << k) ** 2
        u = up[k].cpu().double().flatten(2)                                  # [ci][co][t]
        ref = torch.einsum("o,iot->ti", f[16 * k:16 * k + 16], u)
        mag = torch.einsum("o,iot->ti", f[16 * k:16 * k + 16].abs(), u.abs())
        check_bound("upsampling fold", V[_GEN_OFF[k]:_GEN_OFF[k] + taps], ref, 16 * U * mag, f"V of scale {k}")
        assert torch.equal(A[_GEN_OFF[k]:_GEN_OFF[k] + taps], up1[k].cpu().flatten()), f"A of scale {k}"


def _gen_maps(feats, pqs, tab, fb, h, w):
    """fp64 [5, n, 1, h, w] of the general tail from the table as read (side k = A_k on p_k, fused = fb + sum_k V_k
    on F_k), and the same over absolute values."""
    V, A = tab[:16 * tdr.GEN_TAPS].view(tdr.GEN_TAPS, 16).double(), tab[16 * tdr.GEN_TAPS:].double()
    maps, mags = [], []
    fused = torch.full((feats[0].shape[0], 1, h, w), float(fb), dtype=torch.float64)
    fmag = fused.abs()
    for k, (hk, wk, s, top, left) in enumerate(tdr.tail_scales(h, w)):
        taps = 4 * s * s
        wv = V[_GEN_OFF[k]:_GEN_OFF[k] + taps].view(2 * s, 2 * s, 16).permute(2, 0, 1).unsqueeze(1)   # [ci,1,ty,tx]
        wa = A[_GEN_OFF[k]:_GEN_OFF[k] + taps].view(1, 1, 2 * s, 2 * s)
        fk = feats[k].double().permute(0, 3, 1, 2)
        pk = pqs[k][..., :1].double().permute(0, 3, 1, 2)

        def up(x, wt):
            return F.conv_transpose2d(x, wt, stride=s)[:, :, top:top + h, left:left + w]
        maps.append(up(pk, wa))
        mags.append(up(pk.abs(), wa.abs()))
        fused = fused + up(fk, wv)
        fmag = fmag + up(fk.abs(), wv.abs())
    return torch.stack(maps + [fused]), torch.stack(mags + [fmag])


GEN_FWD_TARGETS = [(regime, label) for regime in tdr.GEN_FWD_REGIMES for label in (False, True)]


@pytest.mark.parametrize("target", GEN_FWD_TARGETS,
                         ids=[f"{r}-{'label' if lab else 'nolabel'}" for r, lab in GEN_FWD_TARGETS])
def test_tail_general_fwd(dev, sms, target):
    """Maps (side: 4 FMAs, fused: the bias + 256 FMAs), the 13 sums and six losses against fp64 of the maps written;
    two identical calls are bit-identical (every reduction of the file is fixed-order)."""
    from osvos_pytorch_b200 import ops
    regime, with_label = target
    n, h, w = tdr.find_gen_fwd_shape(regime, sms)
    blocks = tdr.gen_fwd_blocks(n, h, sms)
    up, up1, fw = _gen_weights(90 + h, dev)
    tab = ops.upsampling_fold(up, up1, fw)
    g = _gen(4000 + h + with_label)
    feats, pqs = [], []
    for hk, wk, _, _, _ in tdr.tail_scales(h, w):
        feats.append(torch.randn(n, hk, wk, 16, generator=g))
        pqs.append(torch.randn(n, hk, wk, 2, generator=g) * 2.0)
    fb = torch.randn(1, generator=g)
    d_feats, d_pqs, d_fb = [f.to(dev) for f in feats], [p.to(dev) for p in pqs], fb.to(dev)
    label = (torch.rand(n, 1, h, w, generator=g) > 0.6).float() if with_label else None
    d_label = label.to(dev) if with_label else None
    weights, divisor = (0.5, 0.25, 0.75, 1.0, 1.5), float(n)

    def launch():
        if d_label is None:
            return ops.tail_general_fwd(d_feats, d_pqs, tab, d_fb, n, h, w)
        return ops.tail_general_fwd(d_feats, d_pqs, tab, d_fb, n, h, w, label=d_label, loss_weights=weights,
                                    divisor=divisor)
    res = ran(launch, {("tail_general_fwd_kernel", ()): 1})
    again = launch()
    assert all(torch.equal(a_, b_) for a_, b_ in zip(res, again) if a_ is not None), "two calls differ"
    got = res[0].cpu().double()
    ref, mag = _gen_maps(feats, pqs, tab.cpu(), fb.item(), h, w)
    for k in range(5):
        check_bound("general tail maps", got[k], ref[k], (257 if k == 4 else 4) * U * mag[k], f"map {k}")
    if not with_label:
        assert res[1] is None
        return
    _, sums, losses = res
    sums, losses = sums.cpu(), losses.cpu().double()
    lab = label.double() >= 0.5
    x = got
    sp = x.clamp(min=0) + torch.log1p(torch.exp(-x.abs()))
    per_thread = -(-w // 256) * -(-(n * h) // blocks)
    depth = per_thread + 5 + 2 + 8 + 1.2 * x.abs().max().item()
    want, bound = [], []
    for k in range(5):
        term_mag = sp[k] + x[k].abs()
        want += [(sp[k] - x[k])[lab].sum(), sp[k][~lab].sum()]
        bound += [depth * U * term_mag[lab].sum(), depth * U * term_mag[~lab].sum()]
    P, N = lab.sum().item(), n * h * w
    sg = torch.sigmoid(x[4])
    a_pos, a_neg = (sg - 1)[lab].sum(), sg[~lab].sum()
    a_bound = [depth * U * (sg + 1)[lab].sum(), depth * U * (sg + 1)[~lab].sum()]
    check_bound("general tail sums", sums[:10], torch.stack(want), torch.stack(bound), "loss sums")
    assert sums[10].item() == P and sums[11].item() == N
    check_bound("general tail sums", sums[12:14], torch.stack([a_pos, a_neg]), torch.stack(a_bound), "A sums")
    lw, lb = [], []
    for k in range(5):
        lk = ((N - P) / N * want[2 * k] + P / N * want[2 * k + 1]) / divisor
        lw.append(lk)
        lb.append(((N - P) / N * bound[2 * k] + P / N * bound[2 * k + 1]) / divisor + 2 * U * abs(lk))
    total = sum(wt * lk for wt, lk in zip(weights, lw))
    tb = sum(wt * b for wt, b in zip(weights, lb)) + U * abs(total)
    check_bound("general tail losses", losses, torch.stack(lw + [total]), torch.stack(lb + [tb]), "losses")


# ------------------------------------------------------------------------------------------------ class-balanced loss
def _labels(numel, kind, g):
    """"mixed": 0, 0.5 (positive) and 1 at random, with both classes present whenever numel >= 2."""
    if kind == "all_pos":
        return torch.ones(numel)
    if kind == "all_neg":
        return torch.zeros(numel)
    y = torch.randint(0, 3, (numel,), generator=g).float() * 0.5
    y[:2] = torch.tensor([0.5, 0.0])[:numel]
    return y


CBCE_TARGETS = [(regime, i, det, "mixed") for regime in tdr.CBCE_REGIMES
                for i in range(4 if regime != "tiny" else 3) for det in (False, True)] + \
    [(regime, 0, det, kind) for regime in ("one_block", "capped") for kind in ("all_pos", "all_neg")
     for det in (False, True)]


def _cbce_id(regime, i, det, kind):
    numel = tdr.find_cbce_numels(regime, 132)[i]
    return f"{regime}-mod{numel % 4}-{kind}-{'det' if det else 'atomic'}"


@pytest.mark.parametrize("target", CBCE_TARGETS, ids=[_cbce_id(*t) for t in CBCE_TARGETS])
def test_cbce_fwd_bwd(dev, sms, target):
    """One numel of a regime (its remainder mod 4 does not depend on the SM count).  Labels: 0 / 0.5 / 1 at random,
    all positive or all negative.  With a single class (and so at numel = 1) the class weights make every gradient
    exactly 0, as in the reference loss."""
    from osvos_pytorch_b200 import _native as nat
    lib = nat.load()
    regime, i, det, kind = target
    numel = tdr.find_cbce_numels(regime, sms)[i]
    g = _gen(3000 + numel)
    x = torch.randn(numel, generator=g) * 4.0
    y = _labels(numel, kind, g)
    d_x, d_y = x.to(dev), y.to(dev)
    grid = tdr.loss_grid(numel, sms)
    sums = torch.zeros(tdr.cbce_det_sums(numel, sms) if det else 5, dtype=torch.float64, device=dev)
    loss = torch.empty(1, device=dev)
    divisor = 3.0
    flags = nat.FLAG_DETERMINISTIC if det else 0
    ran(lambda: nat.check(lib.osvos_cbce_fwd(d_x.data_ptr(), d_y.data_ptr(), numel, divisor, sums.data_ptr(),
                                             loss.data_ptr(), flags, _stream()), "cbce fwd"),
        {("cbce_fwd_kernel", (det,)): 1})
    if det:
        s2, l2 = sums.clone(), loss.clone()
        nat.check(lib.osvos_cbce_fwd(d_x.data_ptr(), d_y.data_ptr(), numel, divisor, s2.data_ptr(), l2.data_ptr(),
                                     flags, _stream()), "cbce fwd")
        assert torch.equal(s2[:4], sums[:4]) and torch.equal(l2, loss), "deterministic cbce differs between runs"
    xd = x.double()
    pos = y >= 0.5
    sp = xd.clamp(min=0) + torch.log1p(torch.exp(-xd.abs()))
    e_terms = 8 + 1.2 * xd.abs().max().item()
    ordered = -(-grid // 256) + 256
    depth = 4 * tdr.loss_vectors_per_thread(numel, sms) + 1 + 5 + 8 + (ordered if det else grid) + e_terms
    term = sp + xd.abs()
    want = torch.stack([(sp - xd)[pos].sum(), sp[~pos].sum()])
    bound = torch.stack([depth * U * term[pos].sum(), depth * U * term[~pos].sum()])
    s = sums.cpu()
    check_bound("cbce sums", s[:2], want, bound, f"sums of {numel}")
    P, N = float(pos.sum()), float(numel)
    assert s[2].item() == P and s[3].item() == N, (s[:4], P, N)
    lref = ((N - P) / N * want[0] + P / N * want[1]) / divisor
    lb = ((N - P) / N * bound[0] + P / N * bound[1]) / divisor + 2 * U * abs(lref)
    check_bound("cbce loss", loss.cpu(), lref.view(1), lb.view(1), f"loss of {numel}")
    # backward, with and without an upstream gradient; the guard floats behind the output stay untouched
    for gout in (None, 0.625):
        buf = torch.full((numel + 8,), float("nan"), device=dev)
        dx = buf[:numel]
        d_g = None if gout is None else torch.tensor([gout], device=dev)
        ran(lambda: nat.check(lib.osvos_cbce_bwd(d_x.data_ptr(), d_y.data_ptr(), sums.data_ptr(), nat.ptr(d_g),
                                                 divisor, numel, dx.data_ptr(), _stream()), "cbce bwd"),
            {("cbce_bwd_kernel", ()): 1})
        assert bool(torch.isnan(buf[numel:]).all()), "cbce backward wrote past numel"
        gg = (1.0 if gout is None else gout) * float(torch.tensor(1.0 / divisor, dtype=torch.float32))
        wcls = torch.where(pos, (N - P) / N, P / N).double() * gg
        sg = torch.sigmoid(xd)
        ref = wcls * (sg - pos.double())
        check_bound("cbce bwd", dx, ref, (e_terms + 6) * U * wcls.abs() * (sg + 1), f"dx of {numel}")


# ------------------------------------------------------------------------------------------------ reductions
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
def test_sum_f32(dev, sms, det):
    from osvos_pytorch_b200 import ops
    for numel in (1, 255, 257, 4 * 256 * sms * 3 + 77, 1000003):
        x = torch.randn(numel, generator=_gen(numel)) * 3.0
        kern = "sum_f32_det_kernel" if det else "sum_f32_kernel"
        got = ran(lambda: ops.sum_f32(x.to(dev), deterministic=det), {(kern, ()): 1})
        if det:
            seg = -(-numel // tdr.SUM_BLOCKS)
            depth = -(-seg // 256) + 256 + tdr.SUM_BLOCKS + 1
        else:
            depth = -(-numel // (tdr.sum_grid(numel, sms) * 256)) + 5 + 1
        check_bound(f"sum_f32 {'det' if det else 'atomic'}", got, x.double().sum().view(1),
                    (depth * U * x.double().abs().sum()).view(1), f"sum of {numel}")


@pytest.mark.parametrize("nrows", [1, 63, 64, 65, 4100])
def test_reduce_rows(dev, nrows):
    from osvos_pytorch_b200 import ops
    for ncols in (37, 1000):
        g = _gen(nrows * 7 + ncols)
        rows = torch.randn(nrows, ncols, generator=g)
        base = torch.randn(ncols, generator=g)
        d_rows, d_base = rows.to(dev), base.to(dev)
        for acc in (False, True):
            # a fresh output per call: ran() may call again, and the accumulating form is not idempotent
            out = ran(lambda: ops.reduce_rows(d_rows, d_base.clone(), accumulate=acc),
                      {("reduce_rows_segments_kernel", ()): 1, ("reduce_rows_final_kernel", ()): 1})
            want = rows.double().sum(0) + (base.double() if acc else 0.0)
            mag = rows.double().abs().sum(0) + (base.double().abs() if acc else 0.0)
            check_bound("reduce_rows", out, want, tdr.reduce_rows_depth(nrows) * U * mag, f"{nrows} x {ncols} {acc}")

"""The general tail's backward and the tail's two parameter-gradient finishes, at every segment regime, against fp64 of
what the kernels read.  tests/general_tail_dispatch_ref.py walks tail_general_bwd_kernel's grid and finds the shapes
(find_gen_bwd_shapes: a short, full, one-pixel-last and ragged-last segment at each scale with odd and even w, hk = 1,
n = 1 and 3, and the 480 x 854 frame); torch.profiler confirms which kernels each call ran and how many times.

- tail_general_bwd_kernel<LOSS> + reduce_rows (osvos_tail_general_bwd): every found shape x {maps form, LOSS form} x
  {exact, fast}.  Maps form: all five maps, the four side maps, the fused map alone, one side map.  LOSS form: the
  online weights (0, 0, 0, 0, 1), parent-like weights (all nonzero) and one nonzero side weight, each with mixed,
  all-positive and all-negative labels, the upstream gradient null and 0.7 in turn; logits up to |x| = 20; score_dsn
  weights nonzero.  (A 1 x 1 map holds one class, so there every LOSS-form gradient is exactly 0, as in the loss.)
  Every output starts as NaN, so an entry the call never writes fails.  dF channels 0 - 15, the exact zeros of
  channels 16 - 63 (hi and lo), every column of red[k] (H, gA, sum dp F, sum dp, sum dF) and fuse_bias_grad are
  checked.  The maps of zero-weight losses are passed as NaN: the results are finite and bit-equal to a call with
  finite maps there, so the kernel did not read them; and two calls are bit-identical.
- upsampling_grads_finish_kernel: random reduced rows, U and fuse.weight, with and without accumulate, each output
  kind NULL in turn (its buffer stays as it was).
- side_grads_finish_kernel: tables of 1 - 4 entries with c in the network's order (128, 256, 512, 512), reversed
  (cmax not first), c = 64 (9 c < 1024 threads), 9 c not a multiple of 1024, and c = 1024 (above 48 KB of shared
  memory: the opt-in); side_b NULL, each optional output NULL, accumulate.

Reference.  V and A are the fold's table as the kernel read it (ops.upsampling_fold): V_k as a [16, 1, 2s, 2s]
deconvolution weight (t = ty 2s + tx), A_k as [1, 1, 2s, 2s].  The literal fused_k = crop(conv_transpose2d(F_k, V_k,
stride s)) and side_k = crop(conv_transpose2d(p_k, A_k, stride s)) (oracle.osvos_oracle.center_crop) is differentiated
in fp64 on the GPU against the gradient maps: autograd gives dF, dp, H (V's gradient) and gA (A's gradient); dF gets
dp sw added.  The same computation on the absolute values of every operand gives sum |terms| for each output.

Bounds.  U = 2^-23.  An output formed by `steps` fp32 roundings of running sums of terms t_i is within
steps * U * sum |t_i| of the exact sum of the terms it read.  T = 4 s^2 taps; `depth` = reduce_rows_depth(n hk segs).
- Gradient maps: exact operands in the maps form (e = 0).  In the LOSS form g = c w (sigmoid(x) - y), c = coeff up /
  divisor, formed with __expf: e = E + 7 with the tail backward's E = 8 + 1.2 max |x| (__expf and the division), and
  seven roundings: 1 / divisor, upstream times it, coeff times that, the class weight (fp64 -> fp32), c w, sigmoid - y
  and the product; over the terms |c| w (sigmoid + 1).  The class weights come from the sums read (N - P) / N, P / N.
- dp: T / 16 FMAs per lane + 4 shuffle levels, + e.
- dF: 4 s^2 FMAs + 1 (the fmaf that adds dp sw), + e, over sum |g4 V|; plus dp's error (T / 16 + 4 + e) times |sw|,
  and that product's share of the fmaf, over sum |gk A| |sw|.  The stored hi + lo (or hi alone in fast mode) rounds
  on top (test_gpu_side_schedules._store_rounding).
- H and gA: at most 16 FMAs per item + depth, + e.
- sum dp F and sum dp: as H, plus dp's error carried through: (16 + depth + T / 16 + 4 + e) over sum |dp| |F|;
  sum dF: (16 + depth) over sum |dF| plus the sum of dF's own bounds.
- fuse_bias_grad = c_4 (w_pos S_pos + w_neg S_neg): 1 / divisor, upstream, coeff, the fp32 conversion of the fp64 sum
  and the product: 5, + 1 for the fp64 part.
- upsampling_grads_finish: d_upscale = f H is one fp32 product, so the host restates it bit for bit; with accumulate
  nvcc may contract old + f H into an FMA (--fmad=true), so two roundings of |old| + |f H|.  d_fuse_w: ceil(16 T / 256)
  FMAs + 8 tree levels (+ 1 with accumulate).  d_upscale_, d_score_w, d_score_b and d_side_b are copies of columns of
  red[k]: bit-exact, and with accumulate bit-exact against one fp32 add.
- side_grads_finish: d_side_w = fmaf(ps, g0, pf g1) and d_side_b = fmaf(ps, S0, pf S1): 2 roundings (+ 1 with
  accumulate); d_score_w / d_fuse_w: ceil(9 c / 1024) FMAs + 5 shuffle levels + 32 warps in order + 1 for the side_b
  term (+ 1 with accumulate); d_score_b = S0: a copy.
At module end each family reports its largest share of the bound."""
import os

import pytest
import torch
import torch.nn.functional as F

import general_tail_dispatch_ref as gtr
import train_dispatch_ref as tdr
from oracle import osvos_oracle as oc
from test_gpu_conv_schedules import KernelsRan
from test_gpu_side_schedules import _store_rounding
from test_gpu_train_schedules import BLIND, MEASURED, U, _GEN_OFF, _gen, _gen_weights, _stream, check_bound

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    assert "OSVOS_ABLATE" not in os.environ, "OSVOS_ABLATE switches off parts of the kernels: results are meaningless"
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_measured():
    """The largest share of its bound per family of this module (MEASURED is shared with test_gpu_train_schedules)."""
    before, blind = {f: len(v) for f, v in MEASURED.items()}, len(BLIND)
    yield
    for family, v in sorted(MEASURED.items()):
        mine = v[before.get(family, 0):]
        if mine:
            print(f"\n{family}: largest share of its bound {max(mine):.3f} ({len(mine)} checks)")
    if len(BLIND) > blind:
        print(f"\nprofiler windows that lost device records (kernels not confirmed): {len(BLIND) - blind}")


def ran(fn, expected):
    """test_gpu_train_schedules.ran over this file's kernel names (gtr.parse_general_tail_kernel_name: the training
    step's, and side_grads_finish_kernel): fn() must launch exactly ``expected``.  A window that loses a record is run
    again, at most twice (so fn makes fresh outputs on every call); a window that records a wrong kernel, or more
    launches than expected, fails.  Late in the whole GPU suite torch.profiler can keep losing device records: a window
    holds no device record at all, or fewer than the launch calls it recorded on the host (on the H100: the first
    kernel of the window only, or all but the first).  If the device records it kept are all expected, such a window
    cannot tell whether the rest ran; it is counted in BLIND and its results are still checked."""
    for _ in range(3):
        with KernelsRan(gtr.parse_general_tail_kernel_name) as k:
            out = fn()
        if sum(k.counts.values()) >= sum(expected.values()):
            break
    launches = sum(c for name, d, c in k.seen if d == "CPU" and name.startswith("cudaLaunchKernel"))
    records = sum(c for _, d, c in k.seen if d == "CUDA")
    if records < launches and all(c <= expected.get(key, 0) for key, c in k.counts.items()):
        BLIND.append(sorted(expected))
        return out
    assert k.counts == expected, (k.counts, k.seen[:12])
    return out


def ran_into(make, fn, expected):
    """ran(fn(out), expected) with the outputs of each of its up to three calls made by make() before the profiler
    window opens, so that a window holds the calls' own kernels only."""
    pool = [make() for _ in range(3)]
    return ran(lambda: fn(pool.pop()), expected)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _same_bits(a, b):
    return all((x is None and y is None) or torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def _f32(v):
    """The fp32 value a float argument reaches the kernel as (ctypes c_float), as a Python float."""
    return float(torch.tensor(v, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------ general tail backward
SHAPES = gtr.find_gen_bwd_shapes()
BWD_TARGETS = [(i, loss, fast) for i in range(len(SHAPES)) for loss in (False, True) for fast in (False, True)]
MAP_SETS = ("all", "sides", "fused", "single")
LOSS_WEIGHTS = ("online", "parent", "single")
LABELS = ("mixed", "all_pos", "all_neg")
DIVISOR = 3.0
UPSTREAM = 0.7


def _bwd_id(i, loss, fast):
    n, h, w = SHAPES[i]
    return f"{n}x{h}x{w}-{'loss' if loss else 'maps'}-{'fast' if fast else 'exact'}"


class _Case:
    """Operands of one shape on the device: side features, pq (p in channel 0, channel 1 never read), score_dsn weights
    and the fold's table of random deconvolution weights."""
    def __init__(self, shape, seed, dev):
        from osvos_pytorch_b200 import ops
        self.shape = n, h, w = shape
        self.scales = tdr.tail_scales(h, w)
        self.plan = tdr.gen_bwd_plan(n, h, w)
        up, up1, fw = _gen_weights(seed, dev)
        self.tab = ops.upsampling_fold(up, up1, fw)
        g = _gen(seed)
        self.feats = [torch.randn(n, hk, wk, 16, generator=g).to(dev) for hk, wk, _, _, _ in self.scales]
        self.pqs = [(torch.randn(n, hk, wk, 2, generator=g) * 2.0).to(dev) for hk, wk, _, _, _ in self.scales]
        self.sws = [(torch.randn(16, generator=g) * 0.5).to(dev) for _ in range(4)]

    def outputs(self, fast, loss):
        """NaN-filled outputs and workspace of one call: dF hi [4], lo [4] | None, red [4], fuse_bias_grad | None."""
        from osvos_pytorch_b200 import _native as nat
        dev = self.tab.device
        n, h, w = self.shape
        his, los, reds = [], [], []
        for hk, wk, s, _, _ in self.scales:
            his.append(torch.full((n, hk, wk, 64), NAN, dtype=torch.bfloat16, device=dev))
            los.append(None if fast else torch.full((n, hk, wk, 64), NAN, dtype=torch.bfloat16, device=dev))
            reds.append(torch.full((tdr.gen_row_len(4 * s * s),), NAN, device=dev))
        fb = torch.full((1,), NAN, device=dev) if loss else None
        ws = torch.full(((nat.load().osvos_tail_general_bwd_workspace_bytes(n, h, w) + 3) // 4,), NAN, device=dev)
        return his, los, reds, fb, ws

    def launch(self, fast, maps=None, objective=None, out=None):
        """One osvos_tail_general_bwd into `out` (an outputs() result; fresh ones if None): (dF hi [4], lo [4] | None,
        red [4], fuse_bias_grad | None).  maps: five [n,1,h,w] maps or None; objective: (logits [5], label, sums,
        weights, upstream | None)."""
        from ctypes import byref
        from osvos_pytorch_b200 import _native as nat
        lib = nat.load()
        n, h, w = self.shape
        taps = nat.UPSAMPLING_TAPS
        a = nat.TailGeneralBwdArgs()
        a.vtab, a.atab = self.tab.data_ptr(), self.tab[16 * taps:].data_ptr()
        his, los, reds, fb, ws = out if out is not None else self.outputs(fast, objective is not None)
        for k in range(4):
            a.feat[k], a.pq[k], a.score_w[k] = self.feats[k].data_ptr(), self.pqs[k].data_ptr(), self.sws[k].data_ptr()
            a.df_hi[k], a.df_lo[k], a.red[k] = his[k].data_ptr(), nat.ptr(los[k]), reds[k].data_ptr()
        a.workspace = ws.data_ptr()
        if objective is None:
            for k in range(5):
                a.src[k] = nat.ptr(maps[k])
        else:
            logits, label, sums, weights, upstream = objective
            for k in range(5):
                a.src[k], a.loss_weights[k] = logits[k].data_ptr(), weights[k]
            a.label, a.sums, a.upstream = label.data_ptr(), sums.data_ptr(), nat.ptr(upstream)
            a.divisor, a.fuse_bias_grad = DIVISOR, fb.data_ptr()
        a.n, a.h, a.w = n, h, w
        nat.check(lib.osvos_tail_general_bwd(byref(a), _stream()), "osvos_tail_general_bwd")
        return his, los, reds, fb

    def reference(self, gmaps, gmags):
        """Per scale, fp64: (dF [n,16,hk,wk] without dp sw, dp [n,hk,wk], H [T,16], gA [T]) of the literal tail against
        the maps gmaps [5][n,1,h,w], and the same over |operands| against gmags."""
        n, h, w = self.shape
        tab = self.tab.double()
        V, A = tab[:16 * tdr.GEN_TAPS].view(tdr.GEN_TAPS, 16), tab[16 * tdr.GEN_TAPS:]
        out = []
        for k, (hk, wk, s, _, _) in enumerate(self.scales):
            taps = 4 * s * s
            vk = V[_GEN_OFF[k]:_GEN_OFF[k] + taps].view(2 * s, 2 * s, 16).permute(2, 0, 1).unsqueeze(1)
            ak = A[_GEN_OFF[k]:_GEN_OFF[k] + taps].view(1, 1, 2 * s, 2 * s)
            fk = self.feats[k].double().permute(0, 3, 1, 2)
            pk = self.pqs[k][..., :1].double().permute(0, 3, 1, 2)
            pair = []
            for ops_, g4, gk in (((fk, pk, vk, ak), gmaps[4], gmaps[k]),
                                 (tuple(t.abs() for t in (fk, pk, vk, ak)), gmags[4], gmags[k])):
                leaves = [t.clone().requires_grad_(True) for t in ops_]
                fused = oc.center_crop(F.conv_transpose2d(leaves[0], leaves[2], stride=s), h, w)
                side = oc.center_crop(F.conv_transpose2d(leaves[1], leaves[3], stride=s), h, w)
                dF, dp, dV, dA = torch.autograd.grad((fused * g4).sum() + (side * gk).sum(), leaves)
                pair.append((dF, dp[:, 0], dV[:, 0].permute(1, 2, 0).reshape(taps, 16), dA.flatten()))
            out.append(pair)
        return out

    def check(self, family, got, gmaps, gmags, e, fast):
        """dF, the zero channels and every column of red[k] against reference(gmaps, gmags) with map error e."""
        his, los, reds, _ = got
        for k, ((dF, dp, H, gA), (mF, mp, mH, mA)) in enumerate(self.reference(gmaps, gmags)):
            s = self.scales[k][2]
            taps = 4 * s * s
            sw = self.sws[k].double().view(1, 16, 1, 1)
            fk = self.feats[k].double().permute(0, 3, 1, 2)
            dFt = dF + dp.unsqueeze(1) * sw
            mdF = mF + mp.unsqueeze(1) * sw.abs()
            dp_steps = taps // 16 + 4 + e
            bF = (taps + 1 + e) * U * mF + (dp_steps + 1) * U * mp.unsqueeze(1) * sw.abs()
            hi = his[k].permute(0, 3, 1, 2)
            val = hi[:, :16].double() + (0.0 if fast else los[k].permute(0, 3, 1, 2)[:, :16].double())
            check_bound(f"{family} dF", val, dFt, bF, f"dF of scale {k}", slack=_store_rounding(val, fast))
            assert bool((_bits(hi[:, 16:]) == 0).all()), f"dF hi channels 16..63 of scale {k} are not +0"
            if not fast:
                assert bool((_bits(los[k][..., 16:]) == 0).all()), f"dF lo channels 16..63 of scale {k} are not +0"
            row = reds[k]
            depth = tdr.reduce_rows_depth(self.plan.nrows[k])
            check_bound(f"{family} H gA", row[:16 * taps].view(taps, 16), H, (16 + depth + e) * U * mH, f"H {k}")
            check_bound(f"{family} H gA", row[16 * taps:17 * taps], gA, (16 + depth + e) * U * mA, f"gA {k}")
            sums = row[17 * taps:]
            st = 16 + depth + dp_steps
            want = torch.cat([(dp.unsqueeze(1) * fk).sum((0, 2, 3)), dp.sum().view(1), dFt.sum((0, 2, 3))])
            bound = torch.cat([st * U * (mp.unsqueeze(1) * fk.abs()).sum((0, 2, 3)), st * U * mp.sum().view(1),
                               (16 + depth) * U * mdF.sum((0, 2, 3)) + bF.sum((0, 2, 3))])
            check_bound(f"{family} sums", sums, want, bound, f"sum dp F, sum dp, sum dF of scale {k}")


def _expected(loss):
    return {("tail_general_bwd_kernel", (loss,)): 1, ("reduce_rows_segments_kernel", ()): 4,
            ("reduce_rows_final_kernel", ()): 4}


def _labels(kind, shape, g):
    n, h, w = shape
    if kind == "all_pos":
        return torch.ones(n, 1, h, w)
    if kind == "all_neg":
        return torch.zeros(n, 1, h, w)
    y = torch.randint(0, 3, (n, 1, h, w), generator=g).float() * 0.5          # 0, 0.5 (positive) and 1
    y.view(-1)[:2] = torch.tensor([1.0, 0.0])[:y.numel()]
    return y


def _loss_weights(kind, i):
    if kind == "online":
        return (0.0, 0.0, 0.0, 0.0, 1.0)
    if kind == "parent":
        return (0.3, 0.45, 0.6, 0.75, 1.0)
    return tuple(0.7 if k == i % 4 else 0.0 for k in range(5))              # one side map, its scale by shape


@pytest.mark.parametrize("target", BWD_TARGETS, ids=[_bwd_id(*t) for t in BWD_TARGETS])
def test_tail_general_bwd(dev, target):
    i, loss, fast = target
    shape = SHAPES[i]
    n, h, w = shape
    case = _Case(shape, 600 + 7 * i, dev)
    prec = "fast" if fast else "exact"
    g = _gen(800 + 7 * i + 2 * loss + fast)
    if not loss:
        family = f"general tail bwd maps {prec}"
        full = [torch.randn(n, 1, h, w, generator=g).to(dev) for _ in range(5)]
        for kind in MAP_SETS:
            keep = {"all": range(5), "sides": range(4), "fused": (4,), "single": (i % 4,)}[kind]
            maps = [full[k] if k in keep else None for k in range(5)]
            got = ran_into(lambda: case.outputs(fast, False), lambda o: case.launch(fast, maps=maps, out=o),
                           _expected(False))
            assert _same_bits(sum(got[:3], []), sum(case.launch(fast, maps=maps)[:3], [])), "two calls differ"
            zero = torch.zeros(n, 1, h, w, dtype=torch.float64, device=dev)
            gm = [zero if t is None else t.double() for t in maps]
            case.check(family, got, gm, [t.abs() for t in gm], 0, fast)
        return
    family = f"general tail bwd loss {prec}"
    logits = (torch.randn(5, n, 1, h, w, generator=g) * 8.0).clamp(-20.0, 20.0)
    d_logits = logits.to(dev)
    up32 = _f32(UPSTREAM)
    e = 8 + 1.2 * logits.abs().max().item() + 7
    for j, (wkind, lkind) in enumerate((a, b) for a in LOSS_WEIGHTS for b in LABELS):
        weights = tuple(_f32(x) for x in _loss_weights(wkind, i))
        with_up = (i + j) % 2 == 1
        label = _labels(lkind, shape, g)
        pos = label >= 0.5
        P, N = float(pos.sum()), float(n * h * w)
        sums = torch.zeros(tdr.TAIL_SUMS, dtype=torch.float64)
        sums[10], sums[11], sums[12], sums[13] = P, N, 37.25, -11.5
        d_label, d_sums = label.to(dev), sums.to(dev)
        upstream = torch.tensor([UPSTREAM], device=dev) if with_up else None
        unread = torch.tensor([wt == 0.0 for wt in weights]).view(5, 1, 1, 1, 1).to(dev)
        nan_logits = torch.where(unread, torch.full_like(d_logits, NAN), d_logits)

        got = ran_into(lambda: case.outputs(fast, True),
                       lambda o: case.launch(fast, objective=(nan_logits, d_label, d_sums, weights, upstream), out=o),
                       _expected(True))
        again = case.launch(fast, objective=(d_logits, d_label, d_sums, weights, upstream))
        flat = sum(got[:3], []) + [got[3]]
        assert all(bool(torch.isfinite(t.float()).all()) for t in flat if t is not None), "non-finite output"
        assert _same_bits(flat, sum(again[:3], []) + [again[3]]), \
            "the maps of zero-weight losses were read, or two calls differ"

        xd = logits.double().to(dev)
        sg = torch.sigmoid(xd)
        yv = pos.double().to(dev)
        cls = (N - P) / N * yv + P / N * (1.0 - yv)
        up = up32 if with_up else 1.0
        cs = [wt * up / _f32(DIVISOR) for wt in weights]
        gm = [c * cls * (sg[k] - yv) for k, c in enumerate(cs)]
        gg = [abs(c) * cls * (sg[k] + 1.0) for k, c in enumerate(cs)]
        case.check(family, got, gm, gg, e, fast)
        wp, wn = (N - P) / N, P / N
        fb_ref = cs[4] * (wp * 37.25 + wn * -11.5)
        fb_mag = abs(cs[4]) * (wp * 37.25 + wn * 11.5)
        check_bound("general tail bwd fuse bias", got[3], torch.tensor([fb_ref]), torch.tensor([6 * U * fb_mag]),
                    f"fuse_bias_grad {wkind} {lkind}")


# ------------------------------------------------------------------------------------------------ upsampling finish
FINISH_OUTPUTS = ("d_upscale", "d_upscale1", "d_fuse_w", "d_score_w", "d_score_b", "d_side_b")


def _finish_shapes(k):
    t = 4 << k
    return {"d_upscale": (16, 16, t, t), "d_upscale1": (1, 1, t, t), "d_score_w": (16,), "d_score_b": (1,),
            "d_side_b": (16,)}


@pytest.mark.parametrize("null", (None,) + FINISH_OUTPUTS, ids=["all"] + [f"no-{o}" for o in FINISH_OUTPUTS])
@pytest.mark.parametrize("acc", [False, True], ids=["overwrite", "accumulate"])
def test_upsampling_grads_finish(dev, acc, null):
    """Random reduced rows (the finish reads nothing else of the backward), random U and fuse.weight.  Outputs start
    as NaN (overwrite) or as random values (accumulate); the NULL output's buffer stays as it was."""
    from osvos_pytorch_b200 import ops
    up, _, fw = _gen_weights(950 + acc, dev)
    g = _gen(960 + acc + 2 * len(null or ""))
    reds = [(torch.randn(tdr.gen_row_len((4 << k) ** 2), generator=g) * 3.0).to(dev) for k in range(4)]

    def base(shape):
        return (torch.randn(shape, generator=g) if acc else torch.full(shape, NAN)).to(dev)
    bases = {o: [base(_finish_shapes(k)[o]) for k in range(4)] for o in FINISH_OUTPUTS if o != "d_fuse_w"}
    bases["d_fuse_w"] = base((64,))

    def fresh():
        return {o: ([b.clone() for b in v] if o != "d_fuse_w" else v.clone()) for o, v in bases.items()}

    def launch(outs):
        ops.upsampling_grads_finish(reds, up, fw, accumulate=acc,
                                    **{o: (None if o == null else v) for o, v in outs.items()})
        return outs
    outs = ran_into(fresh, launch, {("upsampling_grads_finish_kernel", ()): 1})
    family = f"upsampling grads finish {'accumulate' if acc else 'overwrite'}"
    f = fw.double()
    for k in range(4):
        taps = (4 << k) ** 2
        row = reds[k]
        H = row[:16 * taps].view(taps, 16)
        u = up[k].flatten(2)                                                       # [ci][co][t]
        if null != "d_upscale":
            got, old = outs["d_upscale"][k], bases["d_upscale"][k]
            fH = (f[16 * k:16 * k + 16].view(1, 16, 1) * H.double().t().reshape(16, 1, taps)).view_as(got)
            if acc:
                check_bound(family, got, old.double() + fH, 2 * U * (old.double().abs() + fH.abs()), f"d_upscale {k}")
            else:
                want = fw[16 * k:16 * k + 16].view(1, 16, 1) * H.t().reshape(16, 1, taps)
                assert torch.equal(_bits(got.view(16, 16, taps)), _bits(want)), f"d_upscale {k} is not f H in fp32"
        copies = {"d_upscale1": row[16 * taps:17 * taps], "d_score_w": row[17 * taps:17 * taps + 16],
                  "d_score_b": row[17 * taps + 16:17 * taps + 17], "d_side_b": row[17 * taps + 17:]}
        for o, v in copies.items():
            if o == null:
                continue
            got, old = outs[o][k].flatten(), bases[o][k].flatten()
            want = old + v if acc else v
            assert torch.equal(_bits(got), _bits(want)), f"{o} {k}: not a copy of its red[k] columns"
        dfw = torch.einsum("iot,ti->o", u.double(), H.double())
        mag = torch.einsum("iot,ti->o", u.double().abs(), H.double().abs())
        if null != "d_fuse_w":
            got, old = outs["d_fuse_w"][16 * k:16 * k + 16], bases["d_fuse_w"][16 * k:16 * k + 16]
            want, mag = (old.double() + dfw, mag + old.double().abs()) if acc else (dfw, mag)
            steps = -(-16 * taps // 256) + 8 + acc
            check_bound(family, got, want, steps * U * mag, f"d_fuse_w {k}")
    if null is not None:
        kept = bases[null] if null == "d_fuse_w" else torch.cat([b.flatten() for b in bases[null]])
        now = outs[null] if null == "d_fuse_w" else torch.cat([b.flatten() for b in outs[null]])
        assert torch.equal(_bits(now), _bits(kept)), f"the NULL output {null}'s buffer changed"


# ------------------------------------------------------------------------------------------------ side finish
SIDE_TABLES = [(128, 256, 512, 512), (512, 512, 256, 128), (64,), (300, 64), (1024,), (64, 1024, 1000)]
SIDE_NULLS = (None, "side_b", "d_score_w", "d_score_b", "d_fuse_w")


@pytest.mark.parametrize("acc", [False, True], ids=["overwrite", "accumulate"])
@pytest.mark.parametrize("cs", SIDE_TABLES, ids=["c" + "-".join(map(str, t)) for t in SIDE_TABLES])
def test_side_grads_finish(dev, cs, acc):
    """One launch over the table; in each variant the named input / output is NULL for the entries 0, 2 (the others
    keep it).  G, S, side_w, side_b and proj random; outputs start as NaN (overwrite) or random (accumulate)."""
    from osvos_pytorch_b200 import ops
    plan = gtr.side_finish_plan(cs)
    assert plan.opt_in == (max(cs) == 1024)
    g = _gen(1100 + sum(cs) + acc)
    ins = []
    for c in cs:
        ins.append({"g": (torch.randn(18 * c + 2, generator=g) * 2.0).to(dev),
                    "side_w": (torch.randn(16, c, 3, 3, generator=g) * 0.05).to(dev),
                    "side_b": (torch.randn(16, generator=g) * 0.1).to(dev),
                    "proj_w": torch.randn(32, generator=g).to(dev), "c": c})
    outs = {"d_side_w": lambda c: (16, c, 3, 3), "d_side_b": lambda c: (16,), "d_score_w": lambda c: (16,),
            "d_score_b": lambda c: (1,), "d_fuse_w": lambda c: (16,)}
    family = f"side grads finish {'accumulate' if acc else 'overwrite'}"
    for null in SIDE_NULLS:
        bases = [{o: (torch.randn(shape(c), generator=g) if acc else torch.full(shape(c), NAN)).to(dev)
                  for o, shape in outs.items()} for c in cs]

        def fresh():
            return [{o: t.clone() for o, t in b.items()} for b in bases]

        def launch(res):
            entries = [dict(ins[k], **res[k]) for k in range(len(cs))]
            for k in range(0, len(cs), 2):
                if null is not None:
                    entries[k][null] = None
            ops.side_grads_finish(entries, accumulate=acc)
            return res
        res = ran_into(fresh, launch, {("side_grads_finish_kernel", ()): 1})
        for k, c in enumerate(cs):
            nulled = null if k % 2 == 0 else None
            gk = ins[k]["g"].double()
            G, S = gk[:18 * c].view(9, 2, c), gk[18 * c:]
            proj = ins[k]["proj_w"].double()
            ps, pf = proj[:16], proj[16:]
            sw = ins[k]["side_w"].double().view(16, c, 9)
            sb = torch.zeros(16, dtype=torch.float64, device=dev) if nulled == "side_b" else ins[k]["side_b"].double()
            old = {o: t.double() for o, t in bases[k].items()}

            def check(o, want, mag, steps):
                got = res[k][o]
                if nulled == o:
                    assert torch.equal(_bits(got), _bits(bases[k][o])), f"the NULL output {o}'s buffer changed"
                    return
                if acc:
                    want, mag, steps = want + old[o], mag + old[o].abs(), steps + 1
                check_bound(family, got, want, steps * U * mag, f"{o} of entry {k} (c = {c}), NULL {nulled}")
            a0, a1 = ps.view(16, 1, 1) * G[:, 0].t().unsqueeze(0), pf.view(16, 1, 1) * G[:, 1].t().unsqueeze(0)
            check("d_side_w", (a0 + a1).view(16, c, 3, 3), (a0.abs() + a1.abs()).view(16, c, 3, 3), 2)
            check("d_side_b", ps * S[0] + pf * S[1], (ps * S[0]).abs() + (pf * S[1]).abs(), 2)
            dots = -(-9 * c // 1024) + 5 + 32 + 1
            for o, r in (("d_score_w", 0), ("d_fuse_w", 1)):
                want = torch.einsum("fct,tc->f", sw, G[:, r]) + sb * S[r]
                mag = torch.einsum("fct,tc->f", sw.abs(), G[:, r].abs()) + (sb * S[r]).abs()
                check(o, want, mag, dots)
            if nulled == "d_score_b":
                assert torch.equal(_bits(res[k]["d_score_b"]), _bits(bases[k]["d_score_b"]))
            else:
                want = bases[k]["d_score_b"] + ins[k]["g"][18 * c:18 * c + 1] if acc else ins[k]["g"][18 * c:18 * c + 1]
                assert torch.equal(_bits(res[k]["d_score_b"]), _bits(want)), f"d_score_b of entry {k} is not S0"

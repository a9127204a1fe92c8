"""Tensor-level wrappers over the C ABI: they allocate outputs with torch (device
memory + stream plumbing only) and enqueue the native kernels on the current
torch stream.  No arithmetic happens in Python / PyTorch here."""
import dataclasses
from ctypes import byref, c_void_p

import torch

from . import _native as nat


MEANVAL = (104.00699, 116.66877, 122.67892)      # dataloaders/davis_2016.py:19 of the reference (BGR)

# number of native kernels enqueued since import (bench.py reports the per-step delta)
KERNEL_LAUNCHES = [0]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _count(n=1):
    KERNEL_LAUNCHES[0] += n


class Act:
    """Split-bf16 NHWC activation tensor: value ~= hi + lo (lo is None in fast mode)."""
    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo):
        self.hi = hi
        self.lo = lo

    @property
    def shape(self):
        return tuple(self.hi.shape)

    @staticmethod
    def empty(n, h, w, c, device, fast=False):
        hi = torch.empty((n, h, w, c), dtype=torch.bfloat16, device=device)
        lo = None if fast else torch.empty((n, h, w, c), dtype=torch.bfloat16, device=device)
        return Act(hi, lo)


class no_uninitialized_fill:
    """Under torch.use_deterministic_algorithms torch fills every torch.empty with NaN
    (torch.utils.deterministic.fill_uninitialized_memory).  The package's workspaces and outputs are written in full
    by its kernels before they are read, so that fill is pure memory traffic (~0.5 ms per 480x854 backward for the
    weight-gradient slices alone); this context turns it off around the package's own allocations."""
    def __enter__(self):
        import torch.utils.deterministic as d
        self.prev = d.fill_uninitialized_memory
        d.fill_uninitialized_memory = False

    def __exit__(self, *exc):
        import torch.utils.deterministic as d
        d.fill_uninitialized_memory = self.prev


def _require_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"osvos_pytorch_b200: {name} must be a CUDA tensor; the OSVOS hot path has no CPU fallback "
                           "(the CPU restatement under oracle/ is test infrastructure only)")


def pack_conv3x3_weights(weight, transpose_flip=False, col_pad=64):
    """nn.Conv2d weight (OIHW fp32) -> packed split-bf16 GEMM operand (see include/osvos_b200.h)."""
    _require_cuda(weight, "weight")
    lib = nat.load()
    w = weight.detach().contiguous().float()
    cout, cin = int(w.shape[0]), int(w.shape[1])
    rows, cols = (cin, cout) if transpose_flip else (cout, cin)
    colp = (cols + col_pad - 1) // col_pad * col_pad
    nbytes = lib.osvos_packed_weight_bytes(rows, colp)
    packed = torch.empty(nbytes // 2, dtype=torch.bfloat16, device=w.device)
    _count()
    nat.check(lib.osvos_pack_conv3x3_weights(w.data_ptr(), packed.data_ptr(), cout, cin, int(transpose_flip), col_pad,
                                             _stream()), "osvos_pack_conv3x3_weights")
    return packed


def nchw_to_act(x, fast=False):
    _require_cuda(x, "x")
    lib = nat.load()
    x = x.contiguous().float()
    n, c, h, w = (int(v) for v in x.shape)
    a = Act.empty(n, h, w, c, x.device, fast)
    _count()
    nat.check(lib.osvos_nchw_to_act(x.data_ptr(), a.hi.data_ptr(), nat.ptr(a.lo), n, c, h, w, _stream()),
              "osvos_nchw_to_act")
    return a


def act_to_nchw(a):
    lib = nat.load()
    n, h, w, c = a.shape
    y = torch.empty((n, c, h, w), dtype=torch.float32, device=a.hi.device)
    _count()
    nat.check(lib.osvos_act_to_nchw(a.hi.data_ptr(), nat.ptr(a.lo), y.data_ptr(), n, c, h, w, _stream()),
              "osvos_act_to_nchw")
    return y


def conv_first(x, weight, bias, relu=True, fast=False):
    """conv1_1 (+ReLU) straight from the NCHW fp32 frame."""
    _require_cuda(x, "x")
    lib = nat.load()
    n, c, h, w = (int(v) for v in x.shape)
    assert c == 3 and tuple(weight.shape) == (64, 3, 3, 3)
    y = Act.empty(n, h, w, 64, x.device, fast)
    flags = (nat.FLAG_RELU if relu else 0) | (nat.FLAG_FAST if fast else 0)
    _count()
    nat.check(lib.osvos_conv_first_fwd(x.data_ptr(), weight.data_ptr(), nat.ptr(bias), y.hi.data_ptr(), nat.ptr(y.lo),
                                       n, h, w, flags, _stream()), "osvos_conv_first_fwd")
    return y


def fold_side_weights_multi(entries, want_f32=True):
    """All side scales folded in ONE launch.  entries: [(side_w, side_b, proj_w [32], proj_b)] ->
    [(packed, bias2, folded_f32 [9, 2, cin] | None)]; see include/osvos_b200.h (osvos_fold_side_weights_multi)."""
    lib = nat.load()
    items = (nat.FoldItem * len(entries))()
    outs, keep = [], []
    for k, (side_w, side_b, proj_w, proj_b) in enumerate(entries):
        side_w = side_w.detach().contiguous().float()
        cin = int(side_w.shape[1])
        dev = side_w.device
        packed = torch.empty(lib.osvos_packed_weight_bytes(2, cin) // 2, dtype=torch.bfloat16, device=dev)
        bias2 = torch.empty(2, dtype=torch.float32, device=dev)
        f32 = torch.empty((9, 2, cin), dtype=torch.float32, device=dev) if want_f32 else None
        it = items[k]
        it.side_w, it.side_b = side_w.data_ptr(), nat.ptr(side_b)
        it.proj_w, it.proj_b = proj_w.data_ptr(), nat.ptr(proj_b)
        it.packed, it.bias2, it.folded_f32, it.cin = packed.data_ptr(), bias2.data_ptr(), nat.ptr(f32), cin
        keep.append(side_w)
        outs.append((packed, bias2, f32))
    _count()
    nat.check(lib.osvos_fold_side_weights_multi(items, len(entries), _stream()), "osvos_fold_side_weights_multi")
    return outs


def stage1_fused(x, w1, b1, w2_packed, b2, pool=True, out_act=False):
    """conv1_1 + ReLU + conv1_2 + ReLU (+ fused 2x2 ceil-mode max pool) of an fp32 NCHW frame in ONE kernel (exact
    mode, inference): -> (full-resolution Act | None, pooled Act | None).  See include/osvos_b200.h."""
    _require_cuda(x, "x")
    lib = nat.load()
    x = x.contiguous().float()
    n, _, h, w = (int(v) for v in x.shape)
    dev = x.device
    y = Act.empty(n, h, w, 64, dev) if out_act else None
    yp = Act.empty(n, (h + 1) // 2, (w + 1) // 2, 64, dev) if pool else None
    a = nat.Stage1Args()
    a.x, a.w1, a.b1 = x.data_ptr(), w1.data_ptr(), nat.ptr(b1)
    a.w2_packed, a.b2 = w2_packed.data_ptr(), nat.ptr(b2)
    a.y_hi, a.y_lo = (y.hi.data_ptr(), y.lo.data_ptr()) if y is not None else (None, None)
    a.pool_hi, a.pool_lo = (yp.hi.data_ptr(), yp.lo.data_ptr()) if yp is not None else (None, None)
    a.n, a.h, a.w = n, h, w
    _count()
    nat.check(lib.osvos_stage1_fused(byref(a), _stream()), "osvos_stage1_fused")
    return y, yp


def side_folded(x, packed, bias2, fast=False):
    """pq [n,h,w,2] of the folded side branch (cout == 2 call of osvos_conv3x3)."""
    lib = nat.load()
    n, h, w, cin = x.shape
    dev = x.hi.device
    pq = torch.empty((n, h, w, 2), dtype=torch.float32, device=dev)
    a = nat.Conv3x3Args()
    a.x_hi, a.x_lo = x.hi.data_ptr(), nat.ptr(x.lo)
    a.w_packed, a.bias, a.pq = packed.data_ptr(), bias2.data_ptr(), pq.data_ptr()
    a.n, a.h, a.w, a.cin, a.cout = n, h, w, cin, 2
    a.flags = nat.FLAG_FAST if fast else 0
    _count()
    nat.check(lib.osvos_conv3x3(byref(a), _stream()), "osvos_conv3x3 (folded side branch)")
    return pq


def side_folded_multi(xs, folded, fast=False):
    """The folded side branches of several scales in ONE launch: xs = stage outputs (Acts), folded = [(packed, bias2, ...)]
    per scale -> list of pq [n,h,w,2] in the same order (osvos_side_folded_multi)."""
    lib = nat.load()
    arr = (nat.Conv3x3Args * len(xs))()
    pqs = []
    for k, (x, f) in enumerate(zip(xs, folded)):
        n, h, w, cin = x.shape
        pq = torch.empty((n, h, w, 2), dtype=torch.float32, device=x.hi.device)
        a = arr[k]
        a.x_hi, a.x_lo = x.hi.data_ptr(), nat.ptr(x.lo)
        a.w_packed, a.bias, a.pq = f[0].data_ptr(), f[1].data_ptr(), pq.data_ptr()
        a.n, a.h, a.w, a.cin, a.cout = n, h, w, cin, 2
        a.flags = nat.FLAG_FAST if fast else 0
        pqs.append(pq)
    _count()
    nat.check(lib.osvos_side_folded_multi(arr, len(xs), _stream()), "osvos_side_folded_multi")
    return pqs


def conv3x3(x, w_packed, bias, cout, relu=False, fast=False, out_act=True, out_f32=False, mask=None,
            proj_w=None, proj_b=None, simt=False, pool=False, colsum=None, deterministic=False):
    """3x3 / pad 1 conv of an Act through the wgmma kernel.  Returns (Act|None, f32|None, pq|None), or
    (Act, pooled Act) when pool=True (fused MaxPool2d(2,2,ceil_mode)).  `colsum` ([cout] fp32, pre-zeroed)
    receives the per-channel sum of the output (fused bias gradient); ``deterministic``: added in a fixed order
    (per-tile partial rows + osvos_reduce_rows) instead of with atomics."""
    lib = nat.load()
    n, h, w, cin = x.shape
    dev = x.hi.device
    y = Act.empty(n, h, w, cout, dev, fast) if out_act else None
    yf = torch.empty((n, h, w, cout), dtype=torch.float32, device=dev) if out_f32 else None
    pq = torch.empty((n, h, w, 2), dtype=torch.float32, device=dev) if proj_w is not None else None
    a = nat.Conv3x3Args()
    a.x_hi, a.x_lo = x.hi.data_ptr(), nat.ptr(x.lo)
    a.w_packed, a.bias = w_packed.data_ptr(), nat.ptr(bias)
    a.y_hi = nat.ptr(y.hi) if y is not None else None
    a.y_lo = nat.ptr(y.lo) if y is not None else None
    a.y_f32 = nat.ptr(yf)
    a.mask_hi = nat.ptr(mask)
    a.proj_w, a.proj_b, a.pq = nat.ptr(proj_w), nat.ptr(proj_b), nat.ptr(pq)
    yp = Act.empty(n, (h + 1) // 2, (w + 1) // 2, cout, dev, fast) if pool else None
    a.pool_hi = nat.ptr(yp.hi) if pool else None
    a.pool_lo = nat.ptr(yp.lo) if pool else None
    rows = None
    if deterministic and colsum is not None:
        nrows = lib.osvos_conv3x3_colsum_rows(n, h, w)
        rows = torch.empty((nrows, cout), dtype=torch.float32, device=dev)
    a.colsum = nat.ptr(rows if rows is not None else colsum)
    a.n, a.h, a.w, a.cin, a.cout = n, h, w, cin, cout
    a.flags = (nat.FLAG_RELU if relu else 0) | (nat.FLAG_FAST if fast else 0) | \
              (nat.FLAG_RELU_MASK if mask is not None else 0) | (nat.FLAG_DETERMINISTIC if rows is not None else 0)
    fn = lib.osvos_conv3x3_simt if simt else lib.osvos_conv3x3
    _count()
    nat.check(fn(byref(a), _stream()), "osvos_conv3x3")
    if rows is not None:
        reduce_rows(rows, colsum, accumulate=True)
    if pool:
        return y, yp
    return y, yf, pq


def maxpool2x2(x):
    lib = nat.load()
    n, h, w, c = x.shape
    y = Act.empty(n, (h + 1) // 2, (w + 1) // 2, c, x.hi.device, x.lo is None)
    _count()
    nat.check(lib.osvos_maxpool2x2_fwd(x.hi.data_ptr(), nat.ptr(x.lo), y.hi.data_ptr(), nat.ptr(y.lo), n, h, w, c,
                                       _stream()), "osvos_maxpool2x2_fwd")
    return y


def side_project(feat, proj_w, proj_b):
    lib = nat.load()
    n, h, w, c = (int(v) for v in feat.shape)
    assert c == 16
    pq = torch.empty((n, h, w, 2), dtype=torch.float32, device=feat.device)
    _count()
    nat.check(lib.osvos_side_project(feat.data_ptr(), proj_w.data_ptr(), nat.ptr(proj_b), pq.data_ptr(), n, h, w,
                                     _stream()), "osvos_side_project")
    return pq


def _tail_maps(n, h, w, dev):
    """The five output maps of a tail forward, [5,n,1,h,w] fp32, each starting on a 16-byte boundary so that the kernel
    can use 128-bit stores."""
    per = (n * h * w + 3) // 4 * 4
    return torch.empty((5, per), dtype=torch.float32, device=dev)[:, :n * h * w].view(5, n, 1, h, w)


def _tail_losses(a, name, label, loss_weights, divisor, dev):
    """With `loss_weights`, points the forward args `a` at a new losses [6] tensor and sets the weights and divisor;
    returns that tensor, or None without `loss_weights`."""
    if loss_weights is None:
        return None
    if label is None or divisor is None:
        raise ValueError(f"{name}: loss_weights needs label and divisor")
    losses = torch.empty(6, dtype=torch.float32, device=dev)
    a.losses = losses.data_ptr()
    for k in range(5):
        a.loss_weights[k] = float(loss_weights[k])
    a.divisor = float(divisor)
    return losses


def _tail_dpq(a, n, h, w, dev):
    """The four side-map gradients [n,hk,wk,2] of a tail backward, pointed to by the args `a`."""
    dpq, hk, wk = [], h, w
    for k in range(4):
        hk, wk = (hk + 1) // 2, (wk + 1) // 2
        t = torch.empty((n, hk, wk, 2), dtype=torch.float32, device=dev)
        dpq.append(t)
        a.dpq[k] = t.data_ptr()
    return dpq


def tail_fwd(pqs, fuse_bias, n, h, w, label=None, out=None, loss_weights=None, divisor=None, deterministic=False,
             void=False):
    """Upsample + crop + fuse (+ loss sums, + the five class-balanced BCE losses and their weighted total).
    Returns (out [5,n,1,h,w] fp32, sums [TAIL_SUMS] f64 | None) and, with `loss_weights` (5 floats) and `divisor`,
    additionally losses [6] fp32 = the five per-map losses and sum_k loss_weights[k] * loss_k.  ``void``: label < 0
    marks void pixels, left out of the loss (OSVOS_FLAG_VOID_LABELS)."""
    lib = nat.load()
    dev = pqs[0].device
    if out is None:
        out = _tail_maps(n, h, w, dev)
    if void and label is None:
        raise ValueError("tail_fwd: void needs a label")
    flags = (nat.FLAG_DETERMINISTIC if deterministic else 0) | (nat.FLAG_VOID_LABELS if void else 0)
    nsums = lib.osvos_tail_fwd_sums(n, h, w, flags)
    sums = torch.empty(nsums, dtype=torch.float64, device=dev) if label is not None else None
    a = nat.TailFwdArgs()
    a.flags = flags
    for k in range(4):
        a.pq[k] = pqs[k].data_ptr()
    for k in range(5):
        a.out[k] = out[k].data_ptr()
    a.fuse_bias = nat.ptr(fuse_bias)
    a.label = nat.ptr(label)
    a.sums = nat.ptr(sums)
    losses = _tail_losses(a, "tail_fwd", label, loss_weights, divisor, dev)
    a.n, a.h, a.w = n, h, w
    _count()
    nat.check(lib.osvos_tail_fwd(byref(a), _stream()), "osvos_tail_fwd")
    if losses is not None:
        return out, sums, losses
    return out, sums


def tail_loss_bwd(out, label, sums, loss_weights, divisor, upstream, n, h, w, want_fuse_bias=True, deterministic=False,
                  void=False):
    """Backward of tail + the weighted class-balanced BCE objective in one launch (see include/osvos_b200.h):
    -> (list of 4 dpq tensors [n,hk,wk,2], fuse.bias gradient [1] | None).  ``void`` as passed to tail_fwd."""
    lib = nat.load()
    dev = out.device
    a = nat.TailLossBwdArgs()
    a.flags = (nat.FLAG_DETERMINISTIC if deterministic else 0) | (nat.FLAG_VOID_LABELS if void else 0)
    for k in range(5):
        a.logits[k] = out[k].data_ptr()
        a.loss_weights[k] = float(loss_weights[k])
    a.label, a.sums, a.upstream = label.data_ptr(), sums.data_ptr(), nat.ptr(upstream)
    a.divisor = float(divisor)
    dpq = _tail_dpq(a, n, h, w, dev)
    fb = torch.empty(1, dtype=torch.float32, device=dev) if want_fuse_bias else None
    a.fuse_bias_grad = nat.ptr(fb)
    a.n, a.h, a.w = n, h, w
    _count(1)
    nat.check(lib.osvos_tail_loss_bwd(byref(a), _stream()), "osvos_tail_loss_bwd")
    return dpq, fb


def upsampling_fold(upscale_ws, upscale1_ws, fuse_w):
    """The eight deconvolution weights and fuse.weight -> one fp32 table [17 * UPSAMPLING_TAPS]: V [taps][16] (each
    upscale[k] folded with its slice of fuse), then A [taps] (the upscale_[k] taps); osvos_upsampling_fold."""
    lib = nat.load()
    ws = [w.detach().contiguous().float() for w in list(upscale_ws) + list(upscale1_ws) + [fuse_w]]
    for k in range(4):
        t = 4 << k
        if tuple(ws[k].shape) != (16, 16, t, t) or tuple(ws[4 + k].shape) != (1, 1, t, t):
            raise ValueError(f"upscale[{k}] / upscale_[{k}] must be [16,16,{t},{t}] / [1,1,{t},{t}], got "
                             f"{tuple(ws[k].shape)} / {tuple(ws[4 + k].shape)}")
    taps = nat.UPSAMPLING_TAPS
    tab = torch.empty(17 * taps, dtype=torch.float32, device=fuse_w.device)
    a = nat.UpsamplingFoldArgs()
    for k in range(4):
        a.upscale_w[k], a.upscale1_w[k] = ws[k].data_ptr(), ws[4 + k].data_ptr()
    a.fuse_w, a.vtab, a.atab = ws[8].data_ptr(), tab.data_ptr(), tab[16 * taps:].data_ptr()
    _count()
    nat.check(lib.osvos_upsampling_fold(byref(a), _stream()), "osvos_upsampling_fold")
    return tab


def tail_general_fwd(feats, pqs, table, fuse_bias, n, h, w, label=None, loss_weights=None, divisor=None):
    """tail_fwd with general deconvolution weights: the four 16-channel side features, their pq (p in channel 0) and
    the upsampling_fold table -> (out [5,n,1,h,w], sums | None[, losses [6]]) with tail_fwd's contract."""
    lib = nat.load()
    dev = feats[0].device
    out = _tail_maps(n, h, w, dev)
    sums = torch.empty(lib.osvos_tail_general_fwd_sums(n, h, w), dtype=torch.float64, device=dev) \
        if label is not None else None
    a = nat.TailGeneralFwdArgs()
    for k in range(4):
        a.feat[k], a.pq[k] = feats[k].data_ptr(), pqs[k].data_ptr()
    for k in range(5):
        a.out[k] = out[k].data_ptr()
    taps = nat.UPSAMPLING_TAPS
    a.vtab, a.atab = table.data_ptr(), table[16 * taps:].data_ptr()
    a.fuse_bias, a.label, a.sums = nat.ptr(fuse_bias), nat.ptr(label), nat.ptr(sums)
    losses = _tail_losses(a, "tail_general_fwd", label, loss_weights, divisor, dev)
    a.n, a.h, a.w = n, h, w
    _count(2 if label is not None else 1)
    nat.check(lib.osvos_tail_general_fwd(byref(a), _stream()), "osvos_tail_general_fwd")
    if losses is not None:
        return out, sums, losses
    return out, sums


def tail_general_bwd(feats, pqs, score_ws, table, n, h, w, fast=False, grads=None, objective=None,
                     want_fuse_bias=False):
    """Backward of tail_general_fwd (osvos_tail_general_bwd): from the five gradient maps `grads` (None entries are
    zero), or with `objective` = (logits [5,n,1,h,w], label, sums, loss_weights, divisor, upstream) from dL/dlogit
    formed on the fly -> (dF acts [n,hk,wk,64] per scale, reduced rows per scale, fuse.bias gradient [1] | None)."""
    lib = nat.load()
    dev = feats[0].device
    a = nat.TailGeneralBwdArgs()
    taps = nat.UPSAMPLING_TAPS
    a.vtab, a.atab = table.data_ptr(), table[16 * taps:].data_ptr()
    keep, dfs, reds = [], [], []
    for k in range(4):
        a.feat[k], a.pq[k] = feats[k].data_ptr(), pqs[k].data_ptr()
        sw = score_ws[k].detach().contiguous().float()
        keep.append(sw)
        a.score_w[k] = sw.data_ptr()
        _, hk, wk, _ = feats[k].shape
        df = Act.empty(n, hk, wk, 64, dev, fast)
        dfs.append(df)
        a.df_hi[k], a.df_lo[k] = df.hi.data_ptr(), nat.ptr(df.lo)
        t = (4 << k) ** 2
        red = torch.empty(17 * t + 33, dtype=torch.float32, device=dev)
        reds.append(red)
        a.red[k] = red.data_ptr()
    fb = None
    if objective is not None:
        logits, label, sums, weights, divisor, upstream = objective
        for k in range(5):
            a.src[k] = logits[k].data_ptr()
            a.loss_weights[k] = float(weights[k])
        a.label, a.sums, a.upstream = label.data_ptr(), sums.data_ptr(), nat.ptr(upstream)
        a.divisor = float(divisor)
        if want_fuse_bias:
            fb = torch.empty(1, dtype=torch.float32, device=dev)
            a.fuse_bias_grad = fb.data_ptr()
    else:
        for k in range(5):
            g = grads[k]
            if g is not None:
                g = g.contiguous().float()
                keep.append(g)
            a.src[k] = nat.ptr(g)
    ws = torch.empty((lib.osvos_tail_general_bwd_workspace_bytes(n, h, w) + 3) // 4, dtype=torch.float32, device=dev)
    a.workspace = ws.data_ptr()
    a.n, a.h, a.w = n, h, w
    _count(9)
    nat.check(lib.osvos_tail_general_bwd(byref(a), _stream()), "osvos_tail_general_bwd")
    return dfs, reds, fb


def upsampling_grads_finish(reds, upscale_ws, fuse_w, d_upscale=None, d_upscale1=None, d_fuse_w=None, d_score_w=None,
                            d_score_b=None, d_side_b=None, accumulate=False):
    """Every tail parameter gradient from the reduced rows of tail_general_bwd, one launch
    (osvos_upsampling_grads_finish).  The d_* arguments are lists of four tensors / None (d_fuse_w: one [64] tensor)."""
    lib = nat.load()
    a = nat.UpsamplingGradsArgs()
    none4 = [None] * 4
    keep = [u.detach().contiguous().float() for u in upscale_ws] + [fuse_w.detach().contiguous().float()]
    for k in range(4):
        a.red[k], a.upscale_w[k] = reds[k].data_ptr(), keep[k].data_ptr()
        a.d_upscale_w[k] = nat.ptr((d_upscale or none4)[k])
        a.d_upscale1_w[k] = nat.ptr((d_upscale1 or none4)[k])
        a.d_score_w[k] = nat.ptr((d_score_w or none4)[k])
        a.d_score_b[k] = nat.ptr((d_score_b or none4)[k])
        a.d_side_b[k] = nat.ptr((d_side_b or none4)[k])
    a.fuse_w, a.d_fuse_w = keep[4].data_ptr(), nat.ptr(d_fuse_w)
    a.accumulate = 1 if accumulate else 0
    _count()
    nat.check(lib.osvos_upsampling_grads_finish(byref(a), _stream()), "osvos_upsampling_grads_finish")


def unpool_mask(dpool, x, dside=None, dpq=None, wfold=None, colsum=None, deterministic=False):
    """dz = ReLU'(x) * (unpool(dpool) + side-branch gradient) (osvos_unpool_mask).  The side-branch gradient is the
    fp32 map `dside` [n,h,w,c], the folded form of `dpq` [n,h,w,2] and `wfold` [9,2,c], or none; dpool None: the
    deepest stage (no pooling consumer).  `colsum` [c] accumulates the per-channel sums of dz (the bias gradient);
    ``deterministic``: they go to per-block rows that are added in order."""
    lib = nat.load()
    n, h, w, c = x.shape
    dz = Act.empty(n, h, w, c, x.hi.device, x.lo is None)
    flags = nat.FLAG_DETERMINISTIC if deterministic else 0
    rows = None
    if deterministic and colsum is not None:
        nrows = lib.osvos_unpool_colsum_rows(n, h, w, c, int(dpool is not None), int(dpq is not None))
        rows = torch.empty((nrows, c), dtype=torch.float32, device=x.hi.device)
    _count()
    nat.check(lib.osvos_unpool_mask(dpool.hi.data_ptr() if dpool is not None else None,
                                    nat.ptr(dpool.lo) if dpool is not None else None, x.hi.data_ptr(), nat.ptr(x.lo),
                                    nat.ptr(dside), nat.ptr(dpq), nat.ptr(wfold), dz.hi.data_ptr(), nat.ptr(dz.lo),
                                    nat.ptr(rows if rows is not None else colsum), n, h, w, c, flags, _stream()),
              "osvos_unpool_mask")
    if rows is not None:
        reduce_rows(rows, colsum, accumulate=True)
    return dz


# ------------------------------------------------------------------ backward ops
def wgrad_workspace_floats(dz_channels, cin, shape, deterministic=False):
    """Workspace of one weight gradient over an input of ``shape`` = (n, h, w) (osvos_wgrad_workspace_bytes);
    ``deterministic``: one slice per pixel-range split."""
    flags = nat.FLAG_DETERMINISTIC if deterministic else 0
    return nat.load().osvos_wgrad_workspace_bytes(*shape, cin, dz_channels, flags) // 4


def conv3x3_wgrad(x, dz, cout, fast=False, deferred_ws=None, deterministic=False):
    """dW [cout, cin, 3, 3] of a 3x3 conv from its input act `x` and output-gradient act `dz`.
    With `deferred_ws` (a ZEROED fp32 workspace of wgrad_workspace_floats(dz.channels, cin, shape)) only the tensor-core
    accumulation is enqueued and a finish item for ops.wgrad_finish is returned instead of dW.  ``deterministic``:
    per-split workspace slices summed in order (the workspace is then wgrad_workspace_floats(..., deterministic=True)
    floats and needs no zeroing)."""
    lib = nat.load()
    n, h, w, cin = x.shape
    dzc = dz.shape[3]
    dev = x.hi.device
    a = nat.WgradArgs()
    a.x_hi, a.x_lo, a.dz_hi, a.dz_lo = x.hi.data_ptr(), nat.ptr(x.lo), dz.hi.data_ptr(), nat.ptr(dz.lo)
    a.n, a.h, a.w, a.cin, a.cout, a.dz_channels = n, h, w, cin, cout, dzc
    a.flags = (nat.FLAG_FAST if fast else 0) | (nat.FLAG_DETERMINISTIC if deterministic else 0)
    if deferred_ws is not None:
        a.dw, a.workspace = None, deferred_ws.data_ptr()
        a.flags |= nat.FLAG_DEFER_FINISH
        _count(1)
        nat.check(lib.osvos_conv3x3_wgrad(byref(a), _stream()), "osvos_conv3x3_wgrad")
        item = {"ws": deferred_ws, "cout": cout, "cin": cin, "dz_channels": dzc}
        if deterministic:
            item["splits"] = lib.osvos_wgrad_deterministic_splits(n, h, w, cin, dzc)
        return item
    dw = torch.empty((cout, cin, 3, 3), dtype=torch.float32, device=dev)
    ws = torch.empty(wgrad_workspace_floats(dzc, cin, (n, h, w), deterministic), dtype=torch.float32, device=dev)
    a.dw, a.workspace = dw.data_ptr(), ws.data_ptr()
    _count(3)
    nat.check(lib.osvos_conv3x3_wgrad(byref(a), _stream()), "osvos_conv3x3_wgrad")
    return dw


def wgrad_finish(items):
    """One launch for the workspace -> OIHW step of many layers.  items: dicts from conv3x3_wgrad(deferred_ws=...)
    extended with 'dw' (destination tensor) and 'accumulate' (add into it, e.g. the parameter's .grad)."""
    lib = nat.load()
    for lo in range(0, len(items), nat.WGRAD_FINISH_MAX):
        part = items[lo:lo + nat.WGRAD_FINISH_MAX]
        arr = (nat.WgradFinishItem * len(part))()
        for f, it in zip(arr, part):
            f.workspace, f.dw = it["ws"].data_ptr(), it["dw"].data_ptr()
            f.cout, f.cin, f.dz_channels = it["cout"], it["cin"], it["dz_channels"]
            f.accumulate, f.scale = int(bool(it.get("accumulate"))), 1.0
        det = any("splits" in it for it in part)         # deterministic workspaces: their split slices in order
        splits = (nat.c_int * len(part))(*(int(it.get("splits", 1)) for it in part)) if det else None
        _count(1)
        nat.check(lib.osvos_wgrad_finish(arr, splits, len(part), nat.FLAG_DETERMINISTIC if det else 0, _stream()),
                  "osvos_wgrad_finish")


def tail_bwd(grads, n, h, w, deterministic=False):
    """grads: list of 5 tensors [n,1,h,w] or None -> list of 4 dpq tensors [n,hk,wk,2]."""
    lib = nat.load()
    dev = next(g for g in grads if g is not None).device
    a = nat.TailBwdArgs()
    a.flags = nat.FLAG_DETERMINISTIC if deterministic else 0
    keep = []
    for k in range(5):
        g = grads[k]
        if g is not None:
            g = g.contiguous().float()
            keep.append(g)
        a.grad_out[k] = nat.ptr(g)
    dpq = _tail_dpq(a, n, h, w, dev)
    a.n, a.h, a.w = n, h, w
    _count(1)
    nat.check(lib.osvos_tail_bwd(byref(a), _stream()), "osvos_tail_bwd")
    return dpq


def reduce_rows(rows, out, accumulate=False):
    """out[c] = (accumulate ? out[c] : 0) + sum_r rows[r][c] in a fixed order (osvos_reduce_rows); rows [R, C] fp32."""
    lib = nat.load()
    nrows, ncols = int(rows.shape[0]), int(rows.shape[1])
    scratch = torch.empty(lib.osvos_reduce_rows_scratch_floats(nrows, ncols), dtype=torch.float32, device=rows.device)
    _count(2)
    nat.check(lib.osvos_reduce_rows(rows.data_ptr(), nrows, ncols, scratch.data_ptr(), out.data_ptr(), int(accumulate),
                                    _stream()), "osvos_reduce_rows")
    return out


def sum_f32(x, deterministic=False):
    """sum(x) as a [1] fp32 tensor (osvos_sum_f32); ``deterministic``: fixed grid of contiguous ranges, totals added in
    order."""
    lib = nat.load()
    x = x.contiguous().float()
    flags = nat.FLAG_DETERMINISTIC if deterministic else 0
    scratch = torch.empty(lib.osvos_sum_f32_scratch_bytes(flags), dtype=torch.uint8, device=x.device)
    out = torch.empty(1, dtype=torch.float32, device=x.device)
    _count(1)
    nat.check(lib.osvos_sum_f32(x.data_ptr(), x.numel(), scratch.data_ptr(), out.data_ptr(), flags, _stream()),
              "osvos_sum_f32")
    return out


def side_folded_wgrad_floats(c):
    return int(nat.load().osvos_side_folded_wgrad_floats(c))


def side_folded_wgrad_multi(xs, dpqs, gs, deterministic=False):
    """gs[k] ([18 c + 2] fp32, PRE-ZEROED) += folded weight gradient of the side branch of scale k, all scales in ONE
    launch (osvos_side_folded_wgrad_multi); ``deterministic``: the blocks' partial rows are added in order."""
    lib = nat.load()
    arr = (nat.SideWgradItem * len(xs))()
    for it, x, dpq, g in zip(arr, xs, dpqs, gs):
        n, h, w, c = x.shape
        it.x_hi, it.x_lo, it.dpq, it.g = x.hi.data_ptr(), nat.ptr(x.lo), dpq.data_ptr(), g.data_ptr()
        it.n, it.h, it.w, it.c = n, h, w, c
    flags = nat.FLAG_DETERMINISTIC if deterministic else 0
    nbytes = lib.osvos_side_folded_wgrad_workspace_bytes(arr, len(xs), flags)
    ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=gs[0].device) if nbytes else None
    _count(1 + 2 * len(xs) if deterministic else 1)
    nat.check(lib.osvos_side_folded_wgrad_multi(arr, len(xs), nat.ptr(ws), flags, _stream()),
              "osvos_side_folded_wgrad_multi")


def side_grads_finish(entries, accumulate):
    """entries: dicts with g, side_w, side_b, proj_w, d_side_w, d_side_b, d_score_w, d_score_b, d_fuse_w (tensors or
    None), c.  One launch for all scales."""
    lib = nat.load()
    items = (nat.SideGradsItem * len(entries))()
    for k, e in enumerate(entries):
        it = items[k]
        it.g, it.side_w, it.side_b, it.proj_w = e["g"].data_ptr(), e["side_w"].data_ptr(), nat.ptr(e["side_b"]), \
            e["proj_w"].data_ptr()
        it.d_side_w, it.d_side_b = e["d_side_w"].data_ptr(), e["d_side_b"].data_ptr()
        it.d_score_w, it.d_score_b, it.d_fuse_w = nat.ptr(e.get("d_score_w")), nat.ptr(e.get("d_score_b")), \
            nat.ptr(e.get("d_fuse_w"))
        it.c, it.accumulate = int(e["c"]), 1 if accumulate else 0
    _count()
    nat.check(lib.osvos_side_grads_finish(items, len(entries), _stream()), "osvos_side_grads_finish")


def conv_first_bwd(x, dz, weight, need_dx, deterministic=False):
    lib = nat.load()
    n, _, h, w = (int(v) for v in x.shape)
    dw = torch.empty((64, 3, 3, 3), dtype=torch.float32, device=x.device)
    dx = torch.empty_like(x) if need_dx else None
    flags = nat.FLAG_DETERMINISTIC if deterministic else 0   # deterministic: one partial slot per block, added in order
    ws = torch.empty(lib.osvos_conv_first_bwd_workspace_bytes(n, h, w, flags), dtype=torch.uint8, device=x.device)
    _count(2 if need_dx else 1)
    nat.check(lib.osvos_conv_first_bwd(x.data_ptr(), dz.hi.data_ptr(), nat.ptr(dz.lo), weight.data_ptr(),
                                       dw.data_ptr(), nat.ptr(dx), ws.data_ptr(), n, h, w, flags, _stream()),
              "osvos_conv_first_bwd")
    return dw, dx


_U8_MODES = {"prob": nat.U8_PROB, "bytescale": nat.U8_BYTESCALE, "mask": nat.U8_MASK}


def logits_to_u8(logits, mode="bytescale", out=None):
    """Test-time output path on the device (reference train_online.py:181-187): fused logits [N,1,H,W] fp32 ->
    uint8 [N,1,H,W].  mode 'bytescale' is the PNG payload the reference's sigmoid + scipy.misc.imsave writes,
    'prob' is round(255*sigmoid), 'mask' is 255*(logit > 0)."""
    lib = nat.load()
    _require_cuda(logits, "logits")
    x = logits.detach().contiguous().float()
    frames = int(x.shape[0])
    per = x.numel() // frames
    if out is None:
        out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    ws = torch.empty(2 * frames, dtype=torch.int32, device=x.device) if mode == "bytescale" else None
    _count(3 if mode == "bytescale" else 1)
    nat.check(lib.osvos_logits_to_u8(x.data_ptr(), out.data_ptr(), nat.ptr(ws), frames, per, _U8_MODES[mode], _stream()),
              "osvos_logits_to_u8")
    return out


def _require_u8(t, name, dims):
    _require_cuda(t, name)
    if t.dtype != torch.uint8 or t.dim() != dims:
        raise ValueError(f"{name} must be a uint8 tensor with {dims} dimensions, got {t.dtype} {tuple(t.shape)}")
    return t.contiguous()


def image_from_bgr8(frames, meanval=MEANVAL, out=None):
    """Decoded frames uint8 [N,H,W,3] (BGR, as cv2.imread returns them) -> fp32 [N,3,H,W] = float(v) - meanval[c], the
    reference's make_img_gt_pair + ToTensor (dataloaders/davis_2016.py:101-102), bit for bit."""
    lib = nat.load()
    x = _require_u8(frames, "frames", 4)
    n, h, w, c = (int(v) for v in x.shape)
    if c != 3:
        raise ValueError("frames must be [N,H,W,3]")
    if out is None:
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=x.device)
    _count()
    nat.check(lib.osvos_image_from_bgr8(x.data_ptr(), out.data_ptr(), n, h, w, *(float(m) for m in meanval), _stream()),
              "osvos_image_from_bgr8")
    return out


def label_stats_u8(masks):
    """uint8 masks [N,H,W] -> int32 [N,2] on the device: {max byte, 1 if every byte is 0 or the max}."""
    lib = nat.load()
    x = _require_u8(masks, "masks", 3)
    n, h, w = (int(v) for v in x.shape)
    stats = torch.empty((n, 2), dtype=torch.int32, device=x.device)
    _count(3)
    nat.check(lib.osvos_label_stats_u8(x.data_ptr(), stats.data_ptr(), n, h, w, _stream()), "osvos_label_stats_u8")
    return stats


def label_from_u8(masks, stats=None, out=None):
    """uint8 masks [N,H,W] -> fp32 [N,1,H,W] = v / max(frame max, 1e-8), the reference's gt normalisation
    (dataloaders/davis_2016.py:104-106) rounded to fp32, bit for bit.  ``stats``: label_stats_u8 of the same masks."""
    lib = nat.load()
    x = _require_u8(masks, "masks", 3)
    n, h, w = (int(v) for v in x.shape)
    stats = label_stats_u8(x) if stats is None else stats
    if out is None:
        out = torch.empty((n, 1, h, w), dtype=torch.float32, device=x.device)
    _count()
    nat.check(lib.osvos_label_from_u8(x.data_ptr(), stats.data_ptr(), out.data_ptr(), n, h, w, _stream()),
              "osvos_label_from_u8")
    return out


def _id_object(obj):
    """The native `object` argument of the id-map ingest: 0 for every object (None / "all"), else k in 1..254."""
    if obj is None or obj == "all":
        return 0
    if isinstance(obj, bool) or not isinstance(obj, int) or not 1 <= obj <= 254:
        raise ValueError(f"object must be None, 'all' or an object id in 1..254, got {obj!r}")
    return obj


def labels_from_ids(ids, object=None, out=None):
    """DAVIS-2017 object-id maps uint8 [N,H,W] (0 background, 1..K objects, 255 void) -> fp32 labels [N,1,H,W]:
    -1 for void, 1 for an object (any of 1..254 with ``object`` None / "all", only id ``object`` otherwise), else 0
    (osvos_labels_from_ids).  The labels of the class-balanced loss's void form (OSVOS_FLAG_VOID_LABELS)."""
    lib = nat.load()
    x = _require_u8(ids, "ids", 3)
    k = _id_object(object)
    n, h, w = (int(v) for v in x.shape)
    if out is None:
        out = torch.empty((n, 1, h, w), dtype=torch.float32, device=x.device)
    _count()
    nat.check(lib.osvos_labels_from_ids(x.data_ptr(), out.data_ptr(), n, h, w, k, _stream()), "osvos_labels_from_ids")
    return out


_RESIZE_MODES = {"bilinear": nat.RESIZE_BILINEAR, "nearest": nat.RESIZE_NEAREST}


def resize_u8(x, size, mode="bilinear", out=None):
    """uint8 [N,H,W,C] (C = 3, e.g. BGR frames) or [N,H,W] (C = 1, masks) -> the same layout at ``size`` = (h', w'),
    bit-identical to scipy 1.0's imresize of each frame (Pillow's Image.resize with ``mode`` 'bilinear' or 'nearest';
    csrc/resize.cu, DESIGN.md §17).  Equal sizes are a copy.  No host synchronisation."""
    lib = nat.load()
    _require_cuda(x, "x")
    if x.dtype != torch.uint8 or x.dim() not in (3, 4) or (x.dim() == 4 and int(x.shape[3]) not in (1, 3)):
        raise ValueError(f"x must be uint8 [N,H,W,3], [N,H,W,1] or [N,H,W], got {x.dtype} {tuple(x.shape)}")
    if mode not in _RESIZE_MODES:
        raise ValueError("mode must be 'bilinear' or 'nearest'")
    oh, ow = (int(v) for v in size)
    x = x.contiguous()
    n, h, w = (int(v) for v in x.shape[:3])
    c = int(x.shape[3]) if x.dim() == 4 else 1
    shape = (n, oh, ow) + tuple(x.shape[3:])
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=x.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != shape or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape {shape}")
    nbytes = lib.osvos_resize_u8_workspace_bytes(n, h, w, c, oh, ow, _RESIZE_MODES[mode])
    if nbytes == 0 and (oh, ow) != (h, w):
        raise ValueError(f"cannot resize [{n},{h},{w},{c}] to ({oh}, {ow}): sizes must lie in [1, 32767] and N < 65536")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device) if nbytes else None
    if (oh, ow) == (h, w):
        _count()
    else:
        _count(2 if mode == "nearest" else 1 + int(h != oh) + int(w != ow))
    nat.check(lib.osvos_resize_u8(x.data_ptr(), out.data_ptr(), nat.ptr(ws), n, h, w, c, oh, ow, _RESIZE_MODES[mode],
                                  _stream()), "osvos_resize_u8")
    return out


def resize_f32(x, size, out=None):
    """fp32 maps [N,H,W] or [N,1,H,W] (e.g. fused logits) -> the same layout at ``size`` = (h', w'), bit-identical to
    scipy 1.0's imresize(map, size, interp='bilinear', mode='F') of each map (Pillow's BILINEAR resize of an 'F' image;
    csrc/resize.cu, DESIGN.md §18).  Equal sizes are a copy.  No host synchronisation."""
    lib = nat.load()
    _require_cuda(x, "x")
    if x.dtype != torch.float32 or x.dim() not in (3, 4) or (x.dim() == 4 and int(x.shape[1]) != 1):
        raise ValueError(f"x must be fp32 [N,H,W] or [N,1,H,W], got {x.dtype} {tuple(x.shape)}")
    oh, ow = (int(v) for v in size)
    x = x.detach().contiguous()
    n, h, w = int(x.shape[0]), int(x.shape[-2]), int(x.shape[-1])
    if not (0 < n < 65536 and all(0 < v < 32768 for v in (h, w, oh, ow))):
        raise ValueError(f"cannot resize [{n},{h},{w}] to ({oh}, {ow}): sizes must lie in [1, 32767] and N < 65536")
    shape = tuple(x.shape[:-2]) + (oh, ow)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    elif out.dtype != torch.float32 or tuple(out.shape) != shape or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous fp32 tensor of shape {shape}")
    nbytes = lib.osvos_resize_f32_workspace_bytes(n, h, w, oh, ow)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device) if nbytes else None
    _count(1 if (oh, ow) == (h, w) else 1 + int(h != oh) + int(w != ow))
    nat.check(lib.osvos_resize_f32(x.data_ptr(), out.data_ptr(), nat.ptr(ws), n, h, w, oh, ow, _stream()),
              "osvos_resize_f32")
    return out


def _palette_bytes(palette):
    pal = bytes(palette)
    if not pal or len(pal) % 3 or len(pal) > 768:
        raise ValueError(f"palette must be 3 * n bytes with 1 <= n <= 256 (the PLTE chunk's RGB triples), got {len(pal)}")
    return pal


def png_max_bytes(h, w, palette=None):
    """Capacity of one encoded frame (osvos_png_max_bytes): the size with every segment stored.  With ``palette`` (the
    PLTE bytes of encode_png) the PLTE chunk is added (osvos_png_max_bytes_palette)."""
    if palette is None:
        return int(nat.load().osvos_png_max_bytes(int(h), int(w)))
    return int(nat.load().osvos_png_max_bytes_palette(int(h), int(w), len(_palette_bytes(palette)) // 3))


def encode_png(maps, out=None, lengths=None, palette=None):
    """uint8 maps [N,H,W] or [N,1,H,W] -> (out uint8 [N, png_max_bytes(H, W)], lengths int64 [N]): frame i's 8-bit
    grayscale PNG file is out[i, :lengths[i]], what the reference's sm.imsave (train_online.py:187) or
    Image.fromarray(map, "L").save writes, with other (deterministic) deflate bytes (csrc/png.cu, DESIGN.md §21).
    ``palette`` (3 * n bytes of RGB triples, 1 <= n <= 256, e.g. png.palette_of a DAVIS-2017 annotation): palette
    files instead, the bytes as indices (IHDR colour type 3 and a PLTE chunk; the rest of the file is the grayscale
    one's; out is then [N, png_max_bytes(H, W, palette)], DESIGN.md §24).  No host synchronisation."""
    lib = nat.load()
    _require_cuda(maps, "maps")
    if maps.dtype != torch.uint8 or maps.dim() not in (3, 4) or (maps.dim() == 4 and int(maps.shape[1]) != 1):
        raise ValueError(f"maps must be uint8 [N,H,W] or [N,1,H,W], got {maps.dtype} {tuple(maps.shape)}")
    pal = None if palette is None else _palette_bytes(palette)
    x = maps.contiguous()
    n, h, w = int(x.shape[0]), int(x.shape[-2]), int(x.shape[-1])
    cap = lib.osvos_png_max_bytes(h, w) if pal is None else lib.osvos_png_max_bytes_palette(h, w, len(pal) // 3)
    nbytes = lib.osvos_png_encode_workspace_bytes(n, h, w)
    if cap == 0 or nbytes == 0:
        raise ValueError(f"cannot encode [{n},{h},{w}]: sizes must lie in [1, 32767] and 0 < N < 65536")
    if out is None:
        out = torch.empty((n, cap), dtype=torch.uint8, device=x.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (n, cap) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape ({n}, {cap})")
    if lengths is None:
        lengths = torch.empty(n, dtype=torch.int64, device=x.device)
    elif lengths.dtype != torch.int64 or tuple(lengths.shape) != (n,) or not lengths.is_contiguous():
        raise ValueError(f"lengths must be a contiguous int64 tensor of shape ({n},)")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    _count(3)
    if pal is None:
        nat.check(lib.osvos_png_encode(x.data_ptr(), out.data_ptr(), lengths.data_ptr(), ws.data_ptr(), n, h, w,
                                       _stream()), "osvos_png_encode")
    else:
        nat.check(lib.osvos_png_encode_palette(x.data_ptr(), pal, len(pal) // 3, out.data_ptr(), lengths.data_ptr(),
                                               ws.data_ptr(), n, h, w, _stream()), "osvos_png_encode_palette")
    return out, lengths


def davis_measures(logits, gt_u8, r=None, out=None):
    """DAVIS-2016 J and F counts on the device (csrc/measures.cu, DESIGN.md §14): fused logits fp32 [N,1,H,W] or
    [N,H,W] and annotations uint8 [N,H,W] -> int32 [N,6] = {|P∧G|, |P∨G|, |B(P)|, |B(G)|, fg_match, gt_match} with
    P = logit > 0 and G = byte != 0.  ``r``: boundary tolerance in pixels, default evaluation.bound_pix(H, W).
    evaluation.j_and_f turns the counts into J and F.  No host synchronisation."""
    from .evaluation import bound_pix
    lib = nat.load()
    _require_cuda(logits, "logits")
    g = _require_u8(gt_u8, "gt_u8", 3)
    n, h, w = (int(v) for v in g.shape)
    if logits.dtype != torch.float32 or logits.numel() != n * h * w or tuple(logits.shape[-2:]) != (h, w):
        raise ValueError(f"logits must be fp32 [N,1,H,W] or [N,H,W] matching gt_u8 {tuple(g.shape)}, got "
                         f"{logits.dtype} {tuple(logits.shape)}")
    x = logits.detach().contiguous()
    r = bound_pix(h, w) if r is None else int(r)
    if out is None:
        out = torch.empty((n, 6), dtype=torch.int32, device=g.device)
    ws = torch.empty(lib.osvos_davis_measures_workspace_bytes(n, h, w), dtype=torch.uint8, device=g.device)
    _count(4)
    nat.check(lib.osvos_davis_measures(x.data_ptr(), g.data_ptr(), out.data_ptr(), ws.data_ptr(), n, h, w, r, _stream()),
              "osvos_davis_measures")
    return out


def _object_maps(maps, name):
    """The K contiguous fp32 maps of merge_objects / upsample_merge_objects: a list of K tensors of one shape
    [N,1,H,W] or [N,H,W] on one CUDA device, or one tensor [K,N,1,H,W] / [K,N,H,W]; 1 <= K <= 254."""
    items = list(maps.unbind(0)) if torch.is_tensor(maps) else list(maps)
    if not 1 <= len(items) <= nat.DAVIS_MAX_OBJECTS:
        raise ValueError(f"{name} takes 1 .. {nat.DAVIS_MAX_OBJECTS} maps, got {len(items)}")
    shape = tuple(items[0].shape)
    if len(shape) not in (3, 4) or (len(shape) == 4 and shape[1] != 1):
        raise ValueError(f"maps must be fp32 [N,1,H,W] or [N,H,W], got {shape}")
    keep = []
    for t in items:
        _require_cuda(t, "maps")
        if t.dtype != torch.float32 or tuple(t.shape) != shape or t.device != items[0].device:
            raise ValueError(f"every map must be fp32 {shape} on one device, got {t.dtype} {tuple(t.shape)}")
        keep.append(t.detach().contiguous())
    return keep


def merge_objects(maps, out=None):
    """Per-object fused logit maps -> uint8 label map [N,H,W] (csrc/measures.cu, DESIGN.md §24): label = 1 + argmax_k
    logit_k where that maximum is > 0, else 0; ties go to the lowest k, NaN never wins and ±0 is background.  ``maps``:
    a list of K fp32 tensors of one shape [N,1,H,W] or [N,H,W], or one fp32 tensor [K,N,1,H,W] / [K,N,H,W];
    1 <= K <= 254.  ``out`` may be any contiguous uint8 [N,H,W] tensor (e.g. a view of a [N,1,H,W] buffer), at any
    alignment.  No host synchronisation."""
    lib = nat.load()
    keep = _object_maps(maps, "merge_objects")
    n, h, w = int(keep[0].shape[0]), int(keep[0].shape[-2]), int(keep[0].shape[-1])
    if out is None:
        out = torch.empty((n, h, w), dtype=torch.uint8, device=keep[0].device)
    elif out.dtype != torch.uint8 or out.numel() != n * h * w or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of {n * h * w} elements, e.g. [{n},{h},{w}]")
    ptrs = (c_void_p * len(keep))(*(t.data_ptr() for t in keep))
    _count()
    nat.check(lib.osvos_merge_objects(ptrs, len(keep), out.data_ptr(), n * h * w, _stream()), "osvos_merge_objects")
    return out


def upsample_merge_objects(maps, size, out=None):
    """Per-object fused logit maps at the network resolution -> uint8 label map [N, h', w'] at ``size`` = (h', w')
    (csrc/resize.cu, DESIGN.md §27): bit-identical to merge_objects([resize_f32(m, size) for m in maps]), in two
    launches whatever K (one for equal sizes) and without the K resized maps.  ``maps`` as merge_objects';
    ``out`` may be any contiguous uint8 tensor of N * h' * w' elements, at any alignment.  A vertical downscale by more
    than about 22 is refused.  No host synchronisation."""
    lib = nat.load()
    keep = _object_maps(maps, "upsample_merge_objects")
    n, h, w = int(keep[0].shape[0]), int(keep[0].shape[-2]), int(keep[0].shape[-1])
    oh, ow = (int(v) for v in size)
    if not (0 < n < 65536 and all(0 < v < 32768 for v in (h, w, oh, ow))):
        raise ValueError(f"cannot resize [{n},{h},{w}] to ({oh}, {ow}): sizes must lie in [1, 32767] and N < 65536")
    nbytes = lib.osvos_upsample_merge_objects_workspace_bytes(n, len(keep), h, w, oh, ow)
    if nbytes == 0 and (oh, ow) != (h, w):
        raise ValueError(f"cannot resize [{n},{h},{w}] to ({oh}, {ow}) in upsample_merge_objects: a vertical downscale "
                         "by more than about 22 is not supported")
    if out is None:
        out = torch.empty((n, oh, ow), dtype=torch.uint8, device=keep[0].device)
    elif out.dtype != torch.uint8 or out.numel() != n * oh * ow or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of {n * oh * ow} elements, e.g. [{n},{oh},{ow}]")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=keep[0].device) if nbytes else None
    ptrs = (c_void_p * len(keep))(*(t.data_ptr() for t in keep))
    _count(1 if (oh, ow) == (h, w) else 2)
    nat.check(lib.osvos_upsample_merge_objects(ptrs, len(keep), out.data_ptr(), nat.ptr(ws), n, h, w, oh, ow, _stream()),
              "osvos_upsample_merge_objects")
    return out


def davis_measures_objects(labels, gt, n_objects, r=None, out=None):
    """DAVIS-2017 per-object J and F counts on the device (csrc/measures.cu, DESIGN.md §24): label maps uint8 [N,H,W]
    (or [N,1,H,W]) and index annotations uint8 [N,H,W] -> int32 [N,K,6], K = ``n_objects``; row (i, k-1) holds the six
    counts of davis_measures with P = label == k and G = gt == k, both cleared where gt == 255 (void).  ``r``:
    boundary tolerance, default evaluation.bound_pix(H, W).  No host synchronisation."""
    from .evaluation import bound_pix
    lib = nat.load()
    g = _require_u8(gt, "gt", 3)
    n, h, w = (int(v) for v in g.shape)
    _require_cuda(labels, "labels")
    if labels.dtype != torch.uint8 or labels.numel() != n * h * w or tuple(labels.shape[-2:]) != (h, w):
        raise ValueError(f"labels must be uint8 [N,H,W] or [N,1,H,W] matching gt {tuple(g.shape)}, got "
                         f"{labels.dtype} {tuple(labels.shape)}")
    k = int(n_objects)
    if not 1 <= k <= nat.DAVIS_MAX_OBJECTS or n * k >= 65536:
        raise ValueError(f"n_objects must lie in 1 .. {nat.DAVIS_MAX_OBJECTS} with N * K < 65536, got K = {k}, N = {n}")
    lab = labels.contiguous()
    r = bound_pix(h, w) if r is None else int(r)
    if out is None:
        out = torch.empty((n, k, 6), dtype=torch.int32, device=g.device)
    ws = torch.empty(lib.osvos_davis_measures_objects_workspace_bytes(n, k, h, w), dtype=torch.uint8, device=g.device)
    _count(4)
    nat.check(lib.osvos_davis_measures_objects(lab.data_ptr(), g.data_ptr(), out.data_ptr(), ws.data_ptr(), n, k, h, w,
                                               r, _stream()), "osvos_davis_measures_objects")
    return out


def _non_negative_int(v, name):
    if isinstance(v, bool) or not isinstance(v, int) or v < 0:
        raise ValueError(f"{name} must be a non-negative integer, got {v!r}")
    return v


def adaptation_threshold(alpha):
    """The logit threshold of the positives for a probability ``alpha`` (0 < alpha < 1): float32(ln(alpha / (1 - alpha))),
    computed in float64."""
    import math
    if isinstance(alpha, bool) or not isinstance(alpha, (int, float)) or not 0.0 < float(alpha) < 1.0:
        raise ValueError(f"alpha must lie strictly between 0 and 1, got {alpha!r}")
    a = float(alpha)
    return float(torch.tensor(math.log(a / (1.0 - a)), dtype=torch.float64).float())


def adaptation_labels(logits, last_mask, alpha, erosion, distance, out=None):
    """Online adaptation targets (csrc/adapt.cu, DESIGN.md §28): fused logits fp32 [N,1,H,W] and the last masks uint8
    [N,H,W] (any alignment) -> (labels fp32 [N,1,H,W], counts int32 [N,3]).  Per frame, M = last_mask != 0, E = M eroded
    by the disk of radius ``erosion`` (pixels outside the frame are not background), D = the exact squared distance to
    E.  A pixel is negative (0) when E is non-empty and D > distance², positive (1) when it is not negative and its logit
    exceeds adaptation_threshold(alpha), and void (-1) otherwise; counts = {|E|, #positive, #negative}.  ``out``: a
    contiguous fp32 [N,1,H,W] tensor to write the labels into (e.g. a graphed training step's static label buffer).
    Everything is checked before the launch.  No host synchronisation."""
    lib = nat.load()
    _require_cuda(logits, "logits")
    _require_cuda(last_mask, "last_mask")
    if last_mask.dtype != torch.uint8 or last_mask.dim() != 3:
        raise ValueError(f"last_mask must be uint8 [N,H,W], got {last_mask.dtype} {tuple(last_mask.shape)}")
    n, h, w = (int(v) for v in last_mask.shape)
    if logits.dtype != torch.float32 or tuple(logits.shape) != (n, 1, h, w):
        raise ValueError(f"logits must be fp32 [N,1,H,W] = {(n, 1, h, w)} matching last_mask, got {logits.dtype} "
                         f"{tuple(logits.shape)}")
    if logits.device != last_mask.device:
        raise ValueError("logits and last_mask must be on one device")
    if not (0 < n < 65536 and 0 < h < 32768 and 0 < w < 32768):
        raise ValueError(f"cannot label [{n},{h},{w}]: sizes must lie in [1, 32767] and 0 < N < 65536")
    threshold = adaptation_threshold(alpha)
    e = _non_negative_int(erosion, "erosion")
    d = _non_negative_int(distance, "distance")
    if out is None:
        out = torch.empty((n, 1, h, w), dtype=torch.float32, device=logits.device)
    elif (out.dtype != torch.float32 or tuple(out.shape) != (n, 1, h, w) or not out.is_contiguous()
          or out.device != logits.device):
        raise ValueError(f"out must be a contiguous fp32 tensor of shape {(n, 1, h, w)} on the logits' device")
    x = logits.detach().contiguous()
    m = last_mask.contiguous()
    counts = torch.empty((n, 3), dtype=torch.int32, device=logits.device)
    ws = torch.empty(lib.osvos_adaptation_workspace_bytes(n, h, w), dtype=torch.uint8, device=logits.device)
    _count(4)
    # distances beyond the frame's diagonal all mean "no negative"; clamp so the radius fits the C int
    cap = 1 << 16
    nat.check(lib.osvos_adaptation_labels(x.data_ptr(), m.data_ptr(), out.data_ptr(), counts.data_ptr(), ws.data_ptr(),
                                          n, h, w, threshold, min(e, cap), min(d, cap), _stream()),
              "osvos_adaptation_labels")
    return out, counts


@dataclasses.dataclass(frozen=True)
class CRF:
    """Parameters of dense_crf (DESIGN.md §29): ``iterations`` mean-field updates, the bilateral message's weight and
    its position / colour scales in pixels and intensity levels, and the Gaussian message's weight and scale.  The
    defaults are pydensecrf's example values; nobody has tuned them for OSVOS, and their effect on J and F is not
    measured."""
    iterations: int = 5
    bilateral_weight: float = 10.0
    bilateral_xy: float = 80.0
    bilateral_rgb: float = 13.0
    gaussian_weight: float = 3.0
    gaussian_xy: float = 3.0

    def __post_init__(self):
        import math
        if isinstance(self.iterations, bool) or not isinstance(self.iterations, int) or self.iterations < 0:
            raise ValueError(f"iterations must be a non-negative integer, got {self.iterations!r}")
        for name in ("bilateral_weight", "gaussian_weight", "bilateral_xy", "bilateral_rgb", "gaussian_xy"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
                raise ValueError(f"{name} must be a finite number, got {v!r}")
            if v < 0 or (name.endswith(("_xy", "_rgb")) and v == 0):
                raise ValueError(f"{name} must be {'> 0' if name.endswith(('_xy', '_rgb')) else '>= 0'}, got {v!r}")


def dense_crf(frames, maps, crf=CRF(), out=None, vertices=None):
    """Refine K fused logit maps with a fully connected CRF (csrc/crf.cu, DESIGN.md §29): ``frames`` the bytes the
    network saw, uint8 [N,H,W,3] BGR at any alignment; ``maps`` the forms merge_objects takes (K maps of [N,1,H,W] or
    [N,H,W], 1 <= K <= 254) -> fp32 [K,N,1,H,W], map k the refined logit a_k - a_0 of labels 0 (background) and 1..K
    after ``crf.iterations`` Potts mean-field updates, which merge_objects / upsample_merge_objects take as they are.
    ``out``: a contiguous fp32 tensor of K*N*H*W elements.  ``vertices``: an int32 [N] tensor that receives each
    frame's lattice vertex count (with iterations > 0).  Everything is checked before the launch.  No host
    synchronisation."""
    lib = nat.load()
    if not isinstance(crf, CRF):
        raise ValueError(f"crf must be an ops.CRF, got {type(crf).__name__}")
    x = _require_u8(frames, "frames", 4)
    n, h, w, c = (int(v) for v in x.shape)
    if c != 3:
        raise ValueError("frames must be [N,H,W,3]")
    keep = _object_maps(maps, "dense_crf")
    k = len(keep)
    if int(keep[0].shape[0]) != n or tuple(keep[0].shape[-2:]) != (h, w) or keep[0].device != x.device:
        raise ValueError(f"maps must be [N,1,H,W] or [N,H,W] matching frames {tuple(x.shape)} on their device, got "
                         f"{tuple(keep[0].shape)}")
    nbytes = lib.osvos_dense_crf_workspace_bytes(n, k, h, w)
    if nbytes == 0:
        raise ValueError(f"cannot refine [{n},{h},{w}] with {k} maps: sizes must lie in [1, 32767], N in [1, 2048] and "
                         "6*N*H*W below 2^31")
    if out is None:
        out = torch.empty((k, n, 1, h, w), dtype=torch.float32, device=x.device)
    elif (out.dtype != torch.float32 or out.numel() != k * n * h * w or not out.is_contiguous()
          or out.device != x.device or out.data_ptr() % 4):
        raise ValueError(f"out must be a contiguous fp32 tensor of {k * n * h * w} elements on the frames' device")
    if vertices is not None and (vertices.dtype != torch.int32 or vertices.numel() != n or vertices.device != x.device):
        raise ValueError(f"vertices must be an int32 tensor of {n} elements on the frames' device")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    ptrs = (c_void_p * k)(*(t.data_ptr() for t in keep))
    # the library refuses, before any launch, frame sizes and scales whose lattice coordinates overflow the packed keys
    nat.check(lib.osvos_dense_crf(x.data_ptr(), ptrs, out.data_ptr(), ws.data_ptr(), n, k, h, w, crf.iterations,
                                  crf.bilateral_weight, crf.bilateral_xy, crf.bilateral_rgb, crf.gaussian_weight,
                                  crf.gaussian_xy, _stream()), "osvos_dense_crf")
    _count(CRF_LAUNCHES_BUILD + CRF_LAUNCHES_PER_ITERATION * crf.iterations if crf.iterations else 0)
    if vertices is not None and crf.iterations:
        vertices.copy_(ws[:4 * n].view(torch.int32).view(vertices.shape))
    return out


# launches of one dense_crf call: elevate, sort (counted once), mark, scan (once), compact, neighbours, the F(1)
# filter (splat, 6 blurs, slice), taps, the initial softmax; then per iteration the filter, the Gaussian rows, the update.
# With 0 iterations the maps are only copied.
CRF_LAUNCHES_BUILD = 16
CRF_LAUNCHES_PER_ITERATION = 10


def _connectivity(c):
    if isinstance(c, bool) or c not in (4, 8):
        raise ValueError(f"connectivity must be 4 or 8, got {c!r}")
    return c


def _component_sizes_ok(n, k, h, w):
    if not (0 < h < 32768 and 0 < w < 32768) or n * k * h * w >= 1 << 31:
        raise ValueError(f"cannot label {k} x [{n},{h},{w}]: H and W must lie in [1, 32767] and N*K*H*W below 2^31")


def connected_components(masks, connectivity=8):
    """Connected components of uint8 masks [N,H,W] (nonzero = foreground, any alignment; csrc/components.cu, DESIGN.md
    §30) -> (labels int32 [N,H,W], counts int32 [N]): per frame scipy.ndimage.label(mask != 0, structure), the cross
    structure for ``connectivity`` 4 and the 3x3 square for 8: 0 background, components 1..counts[f] numbered in the
    raster order of their first pixels.  Frames are independent.  Checked before the launch; no host synchronisation."""
    lib = nat.load()
    x = _require_u8(masks, "masks", 3)
    c = _connectivity(connectivity)
    n, h, w = (int(v) for v in x.shape)
    if n == 0:
        raise ValueError("masks must hold at least one frame")
    _component_sizes_ok(n, 1, h, w)
    labels = torch.empty((n, h, w), dtype=torch.int32, device=x.device)
    counts = torch.empty(n, dtype=torch.int32, device=x.device)
    ws = torch.empty(lib.osvos_connected_components_workspace_bytes(n, h, w), dtype=torch.uint8, device=x.device)
    _count(5)                                       # local, border, compress, scan (counted once), numbering
    nat.check(lib.osvos_connected_components(x.data_ptr(), labels.data_ptr(), counts.data_ptr(), ws.data_ptr(), n, h, w,
                                             c, _stream()), "osvos_connected_components")
    return labels, counts


@dataclasses.dataclass(frozen=True)
class Components:
    """Parameters of filter_components (DESIGN.md §30): ``mode`` "largest" keeps each object's largest connected
    component; "near" keeps every component within ``radius`` pixels (exact Euclidean distance) of the prior mask, or
    the largest when the prior is empty or none is that near.  ``connectivity`` 4 or 8.  The defaults are this project's
    choices, not tuned; their effect on J and F is not measured."""
    mode: str
    radius: int = 32
    connectivity: int = 8

    def __post_init__(self):
        if self.mode not in ("largest", "near"):
            raise ValueError(f"mode must be 'largest' or 'near', got {self.mode!r}")
        if isinstance(self.radius, bool) or not isinstance(self.radius, int) or self.radius < 0:
            raise ValueError(f"radius must be a non-negative integer, got {self.radius!r}")
        _connectivity(self.connectivity)


_COMPONENT_MODES = {"largest": nat.COMPONENTS_LARGEST, "near": nat.COMPONENTS_NEAR}


def filter_components(maps, params, prior=None, out=None):
    """Drop stray components from K fused logit maps (csrc/components.cu, DESIGN.md §30).  ``maps``: the forms
    merge_objects takes (K maps of [N,1,H,W] or [N,H,W], 1 <= K <= 254); ``params`` an ops.Components; ``prior``: uint8
    [K,H,W] (nonzero = object), the mask "near" measures frame 0 against, or None (frame 0 keeps its largest component).
    Frame j > 0 is measured against frame j - 1's kept mask.  Per object and frame, F = z > 0 (NaN and ±0 are not
    foreground); the pixels of dropped components get -z, every other pixel keeps z, so every later stage sees them as
    background.  Returns (out fp32 [K,N,1,H,W], kept uint8 [K,N,H,W] 0/1, stats int32 [K,N,4] = {components, components
    kept, |F|, pixels removed}).  ``out``: a contiguous fp32 tensor of K*N*H*W elements.  Everything is checked before
    the launch.  No host synchronisation."""
    lib = nat.load()
    if not isinstance(params, Components):
        raise ValueError(f"params must be an ops.Components, got {type(params).__name__}")
    keep = _object_maps(maps, "filter_components")
    k = len(keep)
    n, h, w = int(keep[0].shape[0]), int(keep[0].shape[-2]), int(keep[0].shape[-1])
    dev = keep[0].device
    if n == 0:
        raise ValueError("maps must hold at least one frame")
    _component_sizes_ok(n, k, h, w)
    if prior is not None:
        _require_cuda(prior, "prior")
        if prior.dtype != torch.uint8 or tuple(prior.shape) != (k, h, w) or prior.device != dev:
            raise ValueError(f"prior must be uint8 [K,H,W] = {(k, h, w)} on the maps' device, got {prior.dtype} "
                             f"{tuple(prior.shape)}")
        prior = prior.contiguous()
    if out is None:
        out = torch.empty((k, n, 1, h, w), dtype=torch.float32, device=dev)
    elif (out.dtype != torch.float32 or out.numel() != k * n * h * w or not out.is_contiguous() or out.device != dev
          or out.data_ptr() % 4):
        raise ValueError(f"out must be a contiguous fp32 tensor of {k * n * h * w} elements on the maps' device")
    mode = _COMPONENT_MODES[params.mode]
    kept = torch.empty((k, n, h, w), dtype=torch.uint8, device=dev)
    stats = torch.empty((k, n, 4), dtype=torch.int32, device=dev)
    ws = torch.empty(lib.osvos_filter_components_workspace_bytes(n, k, h, w, mode), dtype=torch.uint8, device=dev)
    ptrs = (c_void_p * k)(*(t.data_ptr() for t in keep))
    radius = min(params.radius, 1 << 16)            # past the frame's diagonal every radius means the same
    if params.mode == "largest":
        _count(COMPONENTS_LAUNCHES_LABEL + COMPONENTS_LAUNCHES_PER_DECISION)
    else:
        _count(COMPONENTS_LAUNCHES_LABEL + COMPONENTS_LAUNCHES_PER_DECISION * n
               + COMPONENTS_LAUNCHES_PER_DISTANCE * (n - 1 + (prior is not None)))
    nat.check(lib.osvos_filter_components(ptrs, nat.ptr(prior), out.data_ptr(), kept.data_ptr(), stats.data_ptr(),
                                          ws.data_ptr(), n, k, h, w, mode, radius, params.connectivity, _stream()),
              "osvos_filter_components")
    return out.view(k, n, 1, h, w), kept, stats


# launches of one filter_components call: the labelling of every plane (local, border, compress); per decision (all
# frames at once for "largest", each frame for "near") the decision and the write; per distance transform ("near", each
# frame with a prior) the column and row passes.
COMPONENTS_LAUNCHES_LABEL = 3
COMPONENTS_LAUNCHES_PER_DECISION = 2
COMPONENTS_LAUNCHES_PER_DISTANCE = 2


def decode_jpeg(blob, n, h, w, out=None, status=None, nseg=None, chunk_bits=0):
    """A batch of n JPEGs of size h x w packed by jpeg.pack (``blob``: uint8 device tensor) -> (out uint8 [n,h,w,3] BGR,
    bit-identical to cv2.imread; status int32 [n]: 1 bad Huffman code, 2 zig-zag index past 63, 4 data ended before the
    last MCU, 8 header inconsistent with (n, h, w)).  ``out`` may be any uint8 [n,h,w,3] view with contiguous rows of
    pixels, e.g. a slot range of a collated buffer.  ``chunk_bits``: the Huffman decoder's chunk size (0: default).
    No host synchronisation (csrc/jpeg.cu, DESIGN.md §19).  ``nseg`` (required): the blob's segment count,
    jpeg.segment_count of the host blob.  It sizes the launch, and reading it from the device blob would make the call
    wait for the device."""
    if nseg is None:
        raise ValueError("nseg: pass jpeg.segment_count(host_blob); the device copy is not read back")
    lib = nat.load()
    _require_cuda(blob, "blob")
    if blob.dtype != torch.uint8 or blob.dim() != 1 or not blob.is_contiguous():
        raise ValueError("blob must be a contiguous 1-D uint8 device tensor from jpeg.pack")
    if blob.data_ptr() % 16:
        raise ValueError("blob must be 16-byte aligned")
    shape = (n, h, w, 3)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=blob.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != shape or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape {shape}")
    if status is None:
        status = torch.empty(n, dtype=torch.int32, device=blob.device)
    elif status.dtype != torch.int32 or tuple(status.shape) != (n,) or not status.is_contiguous():
        raise ValueError(f"status must be a contiguous int32 tensor of shape ({n},)")
    nbytes = lib.osvos_jpeg_decode_workspace_bytes(n, h, w, nseg, blob.numel(), chunk_bits)
    if nbytes == 0:
        raise ValueError(f"cannot decode [{n},{h},{w}] with {nseg} segments, {blob.numel()} blob bytes, chunk_bits "
                         f"{chunk_bits}")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=blob.device)
    a = nat.JpegArgs(blob.data_ptr(), blob.numel(), out.data_ptr(), status.data_ptr(), ws.data_ptr(), n, h, w, nseg,
                     chunk_bits, 0)
    nat.check(lib.osvos_jpeg_decode(byref(a), _stream()), "osvos_jpeg_decode")
    _count(6)
    return out, status


def decode_png(blob, n, h, w, nseg, out=None, status=None, path=None):
    """A batch of n grayscale PNGs of size h x w packed by png.pack (``blob``: uint8 device tensor) -> (out uint8
    [n,h,w], what cv2.imread(path, 0) gives, 1-bit files as 0 / 255; palette files parsed with palette="index" as
    their raw indices, what np.array(PIL.Image.open(f)) gives (DESIGN.md §24); status int32 [n]: 1 invalid block type, code
    lengths or code, 2 distance beyond the bytes written, 4 stream ended early or wrong output size, 8 Adler-32
    mismatch, 16 filter type above 4, 32 header inconsistent with (n, h, w)).  ``out`` may be any contiguous uint8
    [n,h,w] tensor, at any alignment.  ``nseg`` (required): the blob's segment count, png.segment_count of the host
    blob; it sizes the launch, and reading it from the device blob would make the call wait for the device.
    ``path``: optional int32 [n] that receives which pass wrote each file (1 the per-segment passes over proven cuts,
    2 the in-order pass).  No host synchronisation (csrc/png_decode.cu, DESIGN.md §22)."""
    if nseg is None:
        raise ValueError("nseg: pass png.segment_count(host_blob); the device copy is not read back")
    lib = nat.load()
    _require_cuda(blob, "blob")
    if blob.dtype != torch.uint8 or blob.dim() != 1 or not blob.is_contiguous():
        raise ValueError("blob must be a contiguous 1-D uint8 device tensor from png.pack")
    if blob.data_ptr() % 16:
        raise ValueError("blob must be 16-byte aligned")
    shape = (n, h, w)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=blob.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != shape or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape {shape}")
    if status is None:
        status = torch.empty(n, dtype=torch.int32, device=blob.device)
    elif status.dtype != torch.int32 or tuple(status.shape) != (n,) or not status.is_contiguous():
        raise ValueError(f"status must be a contiguous int32 tensor of shape ({n},)")
    if path is not None and (path.dtype != torch.int32 or tuple(path.shape) != (n,) or not path.is_contiguous()):
        raise ValueError(f"path must be a contiguous int32 tensor of shape ({n},)")
    nbytes = lib.osvos_png_decode_workspace_bytes(n, h, w, nseg, blob.numel())
    if nbytes == 0:
        raise ValueError(f"cannot decode [{n},{h},{w}] with {nseg} segments, {blob.numel()} blob bytes")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=blob.device)
    a = nat.PngDecodeArgs(blob.data_ptr(), blob.numel(), out.data_ptr(), status.data_ptr(), ws.data_ptr(), nat.ptr(path),
                          n, h, w, nseg)
    nat.check(lib.osvos_png_decode(byref(a), _stream()), "osvos_png_decode")
    _count(5 if nseg == n else 7)
    return out, status


def overlay_mask(frames, logits, color=(0, 0, 255), out=None):
    """The mask drawn over the frame (the reference's helpers.overlay_mask, shown by train_online.py's vis_res):
    frames uint8 [N,H,W,3] BGR and fused logits fp32 [N,1,H,W] or [N,H,W] -> uint8 [N,H,W,3].  fg = logit > 0 (+-0
    and NaN are background); fg pixels with a 4-neighbour in the background or outside the frame (the contour
    cv2.drawContours draws) are black, the rest of fg is (v + c + 1) >> 1 per channel with ``color`` in BGR order, the
    background keeps its bytes.  ``out`` may be ``frames`` itself.  No host synchronisation (DESIGN.md §23)."""
    lib = nat.load()
    x = _require_u8(frames, "frames", 4)
    n, h, w, c = (int(v) for v in x.shape)
    if c != 3:
        raise ValueError("frames must be [N,H,W,3]")
    _require_cuda(logits, "logits")
    if logits.dtype != torch.float32 or logits.numel() != n * h * w or tuple(logits.shape[-2:]) != (h, w):
        raise ValueError(f"logits must be fp32 [N,1,H,W] or [N,H,W] matching frames {tuple(x.shape)}, got "
                         f"{logits.dtype} {tuple(logits.shape)}")
    col = tuple(int(v) for v in color)
    if len(col) != 3 or not all(0 <= v <= 255 for v in col):
        raise ValueError(f"color must be three values in 0..255, got {color}")
    lg = logits.detach().contiguous()
    if out is None:
        out = torch.empty_like(x)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (n, h, w, 3) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape {(n, h, w, 3)}")
    _count()
    nat.check(lib.osvos_overlay_mask(x.data_ptr(), lg.data_ptr(), out.data_ptr(), n, h, w, *col, _stream()),
              "osvos_overlay_mask")
    return out


def overlay_labels(frames, labels, palette=None, out=None):
    """A label map drawn over the frame, each object in its palette colour (DESIGN.md §25): frames uint8 [N,H,W,3] BGR
    and labels uint8 [N,H,W] or [N,1,H,W] of object ids -> uint8 [N,H,W,3].  Id 0 keeps the frame's bytes; a pixel of
    id k != 0 with a 4-neighbour of another id or outside the frame (object k's contour as cv2.drawContours draws it)
    is black, the rest of object k is (v + c_k + 1) >> 1 per channel.  ``palette``: the colours as RGB triples, the
    PLTE chunk's bytes as png.palette_of returns them (1 .. 256 entries); ids past its end are drawn with (0, 0, 0).
    None is the DAVIS palette (png.davis_palette).  With labels = logit > 0 and entry 1 = (255, 0, 0) RGB this is
    overlay_mask.  ``out`` may be ``frames`` itself.  No host synchronisation."""
    from .png import davis_palette
    lib = nat.load()
    x = _require_u8(frames, "frames", 4)
    n, h, w, c = (int(v) for v in x.shape)
    if c != 3:
        raise ValueError("frames must be [N,H,W,3]")
    _require_cuda(labels, "labels")
    if (labels.dtype != torch.uint8 or labels.dim() not in (3, 4) or labels.numel() != n * h * w
            or tuple(labels.shape[-2:]) != (h, w) or (labels.dim() == 4 and int(labels.shape[1]) != 1)):
        raise ValueError(f"labels must be uint8 [N,H,W] or [N,1,H,W] matching frames {tuple(x.shape)}, got "
                         f"{labels.dtype} {tuple(labels.shape)}")
    pal = _palette_bytes(davis_palette() if palette is None else palette)
    colors = nat.OverlayColors()
    for k in range(len(pal) // 3):                           # RGB -> the frame's BGR order
        colors.bgr[3 * k:3 * k + 3] = [pal[3 * k + 2], pal[3 * k + 1], pal[3 * k]]
    lab = labels.contiguous()
    if out is None:
        out = torch.empty_like(x)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (n, h, w, 3) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape {(n, h, w, 3)}")
    _count()
    nat.check(lib.osvos_overlay_labels(x.data_ptr(), lab.data_ptr(), out.data_ptr(), n, h, w, byref(colors),
                                       len(pal) // 3, _stream()), "osvos_overlay_labels")
    return out


def jpeg_max_bytes(h, w):
    """Capacity of one encoded frame (osvos_jpeg_max_bytes): header and EOI plus twice the largest possible scan."""
    return int(nat.load().osvos_jpeg_max_bytes(int(h), int(w)))


def encode_jpeg(frames, quality=95, out=None, lengths=None):
    """uint8 BGR frames [N,H,W,3] -> (out uint8 [N, jpeg_max_bytes(H, W)], lengths int64 [N]): frame i's JPEG file is
    out[i, :lengths[i]], byte for byte what cv2.imencode('.jpg', frame, [cv2.IMWRITE_JPEG_QUALITY, quality]) writes
    (quality 95 is cv2.imwrite's default; csrc/jpeg_encode.cu, DESIGN.md §23).  No host synchronisation."""
    lib = nat.load()
    x = _require_u8(frames, "frames", 4)
    n, h, w, c = (int(v) for v in x.shape)
    if c != 3:
        raise ValueError("frames must be [N,H,W,3]")
    q = int(quality)
    if not 1 <= q <= 100:
        raise ValueError(f"quality must lie in 1..100, got {quality}")
    cap = lib.osvos_jpeg_max_bytes(h, w)
    nbytes = lib.osvos_jpeg_encode_workspace_bytes(n, h, w)
    if cap == 0 or nbytes == 0:
        raise ValueError(f"cannot encode [{n},{h},{w},3]: sizes must lie in [1, 65500] and 0 < N < 65536")
    if out is None:
        out = torch.empty((n, cap), dtype=torch.uint8, device=x.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != (n, cap) or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 tensor of shape ({n}, {cap})")
    if lengths is None:
        lengths = torch.empty(n, dtype=torch.int64, device=x.device)
    elif lengths.dtype != torch.int64 or tuple(lengths.shape) != (n,) or not lengths.is_contiguous():
        raise ValueError(f"lengths must be a contiguous int64 tensor of shape ({n},)")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    _count(7)
    nat.check(lib.osvos_jpeg_encode(x.data_ptr(), out.data_ptr(), lengths.data_ptr(), ws.data_ptr(), n, h, w, q,
                                    _stream()), "osvos_jpeg_encode")
    return out, lengths

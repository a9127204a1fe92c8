"""Training path: one torch.autograd.Function spanning the whole network, so that autograd sees
a single node whose forward/backward are sequences of native kernels (no PyTorch op does
arithmetic).  Replaces the autograd graph of reference networks/vgg_osvos.py:59-74 built at
train_online.py:124 / train_parent.py:140 and walked at :141 / :164.

Gradient bookkeeping mirrors the reference: parameters that do not influence the objective get
``None`` (e.g. score_dsn.* under the fuse-only online loss, SURVEY.md 8c item 9); the eight
deconvolution weights (lr = 0 in both scripts) receive a gradient only when the module's
``learn_upsampling`` is set (the general tail, DESIGN.md §20).

Determinism: the forward reads ``torch.are_deterministic_algorithms_enabled()`` once and keeps it on ``ctx``; the loss
sums of the fused objective and every float reduction of the backward then take their fixed-order forms
(OSVOS_FLAG_DETERMINISTIC, DESIGN.md §16), so two runs on one device give bit-identical losses and gradients.
"""
import torch

from . import ops


class _OSVOSFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, x, objective, *params):
        with ops.no_uninitialized_fill():             # every buffer below is written in full by a kernel
            return _OSVOSFunction._forward(ctx, engine, x, objective, *params)

    @staticmethod
    def backward(ctx, *grads):
        with ops.no_uninitialized_fill():
            return _OSVOSFunction._backward(ctx, *grads)

    @staticmethod
    def _forward(ctx, engine, x, objective, *params):
        """objective: None (plain forward: the five maps, each differentiable) or (label, loss_weights[5], divisor, void):
        the package's own objective fused into the tail - outputs are then (5 maps, total, losses[5]) with only
        `total = sum_k w_k * class_balanced_cross_entropy_loss(map_k, label)` differentiable."""
        m = engine.m
        fast = m.precision == "fast"
        general = engine.uses_general_tail()
        ctx.params = params
        ctx.set_materialize_grads(False)
        det = torch.are_deterministic_algorithms_enabled()      # the backward uses the mode this forward saw
        ctx.det = det
        xin = x.detach().contiguous().float()
        n, _, h, w = (int(v) for v in xin.shape)
        acts, pooled = engine._trunk(xin, fast, keep=True)      # acts[i][j] = output act of conv j of stage i
        # side_prep has no ReLU: folded, its backward needs neither the 16 features nor their gradient
        # (csrc/side_bwd_folded.cu); with general deconvolution weights the features feed the tail (csrc/tail_general.cu)
        feats, pqs = engine._side_outputs([s[-1] for s in acts[1:]], fast)
        if general:
            table = engine._upsampling_table()
            ctx.general = (feats, pqs, table)

            def tail(**kw):
                return ops.tail_general_fwd(feats, pqs, table, m.fuse.bias.detach(), n, h, w, **kw)
        else:
            ctx.general = None

            def tail(**kw):
                return ops.tail_fwd(pqs, m.fuse.bias.detach(), n, h, w, **kw)
        ctx.engine = engine
        ctx.dims = (n, h, w)
        ctx.fast = fast
        if getattr(engine, "debug_capture", None) is not None:      # tests: the saved activations of this pass
            engine.debug_capture.update(acts=acts, pooled=pooled)
        if objective is None:
            out, _ = tail()
            ctx.objective = None
            ctx.saved = (xin, acts, pooled)
            return tuple(out[k] for k in range(5))
        label, weights, divisor, void = objective
        if void and general:
            raise ValueError("void labels are not supported by the general tail (learn_upsampling)")
        label = label.detach().to(xin.device).contiguous().float()
        if label.numel() != n * h * w:
            raise ValueError("objective label must be [N,1,H,W] like the output maps")
        weights = tuple(float(v) for v in weights)
        if general:
            out, sums, losses = tail(label=label, loss_weights=weights, divisor=divisor)
        else:
            out, sums, losses = tail(label=label, loss_weights=weights, divisor=divisor, deterministic=det, void=void)
        ctx.objective = (out, label, sums, weights, float(divisor))
        ctx.void = void
        ctx.saved = (xin, acts, pooled)
        maps = tuple(out[k] for k in range(5))
        total = losses[5:6].reshape(())          # 0-dim view of the weighted total
        per_map = losses[0:5]
        ctx.mark_non_differentiable(*maps, per_map)
        return maps + (total, per_map)

    @staticmethod
    def _backward(ctx, *grads):
        engine = ctx.engine
        m = engine.m
        fast = ctx.fast
        det = ctx.det
        xin, acts, pooled = ctx.saved
        n, h, w = ctx.dims
        convs = m.trunk_convs()
        pg = {}                                   # parameter -> gradient tensor
        obj = ctx.objective
        if obj is not None:
            g_total = grads[5]
            weights = obj[3]
            grads = tuple((True if weights[k] != 0.0 else None) for k in range(5)) if g_total is not None else (None,) * 5
        if all(g is None for g in grads):
            return (None, None, None) + tuple(None for _ in ctx.params)
        # ---- weight-gradient plumbing: ONE zeroed arena for all tensor-core wgrad workspaces, ONE finish launch at
        # the end.  In direct mode (engine.accumulate_param_grads_in_place, set by the package's training loops) the
        # finish adds straight into an existing p.grad and the bias column sums are accumulated into p.grad by the
        # dgrad epilogues - what autograd's AccumulateGrad would otherwise do with one add kernel per parameter.
        direct = bool(getattr(engine, "accumulate_param_grads_in_place", False))

        def grad_target(p):
            g = p.grad
            if direct and p.requires_grad and g is not None and g.is_cuda and g.dtype == torch.float32 \
                    and g.is_contiguous() and g.device == xin.device:
                return g
            return None
        # the saved activation each tensor-core conv reads: the operand of its weight gradient
        inputs = {c: acts[i][j - 1] if j else pooled[i]
                  for i, stage in enumerate(convs) for j, c in enumerate(stage) if i or j}
        general = ctx.general
        if general is not None:                        # side_prep's weight gradient from the 64-channel dF operand
            inputs.update((sp, acts[i + 1][-1]) for i, sp in enumerate(m.side_prep))
        wconvs = list(inputs)
        ws_sizes = [(ops.wgrad_workspace_floats(64 if c in m.side_prep else c.out_channels, c.in_channels,
                                                inputs[c].shape[:3], det) + 3) // 4 * 4
                    for c in wconvs]
        # folded side branch: G [18 C + 2] per scale (rounded up to 16 bytes) behind the wgrad workspaces
        g_sizes = [] if general is not None else [(ops.side_folded_wgrad_floats(sp.in_channels) + 3) // 4 * 4
                                                  for sp in m.side_prep]
        if det:
            # the per-split slices are written in full: only G needs zeroing
            arena = torch.empty(sum(ws_sizes) + sum(g_sizes), dtype=torch.float32, device=xin.device)
            arena[sum(ws_sizes):].zero_()
        else:
            arena = torch.zeros(sum(ws_sizes) + sum(g_sizes), dtype=torch.float32, device=xin.device)
        ws_of, off = {}, 0
        for c, sz in zip(wconvs, ws_sizes):
            ws_of[c] = arena[off:off + sz]
            off += sz
        g_of = []
        for sz in g_sizes:
            g_of.append(arena[off:off + sz])
            off += sz
        fresh = [c for c in wconvs if c in m.side_prep or grad_target(c.weight) is None]
        fresh_buf = torch.empty(sum(c.weight.numel() * (4 if c in m.side_prep else 1) for c in fresh),
                                dtype=torch.float32, device=xin.device)
        finish_items, off = [], 0

        def wgrad(conv, inp, dz_act):
            nonlocal off
            if conv in m.side_prep:     # dW [64, C, 3, 3] of the zero-padded dF operand: its first 16 rows are side_prep's
                it = ops.conv3x3_wgrad(inp, dz_act, 64, fast=fast, deferred_ws=ws_of[conv], deterministic=det)
                nel = 4 * conv.weight.numel()
                it["dw"], it["accumulate"] = fresh_buf[off:off + nel].view(64, *conv.weight.shape[1:]), False
                off += nel
                pg[conv.weight] = it["dw"][:16]
                finish_items.append(it)
                return
            it = ops.conv3x3_wgrad(inp, dz_act, conv.out_channels, fast=fast, deferred_ws=ws_of[conv], deterministic=det)
            tgt = grad_target(conv.weight)
            if tgt is not None:
                it["dw"], it["accumulate"] = tgt, True
                pg[conv.weight] = None
            else:
                nel = conv.weight.numel()
                it["dw"], it["accumulate"] = fresh_buf[off:off + nel].view(conv.weight.shape), False
                off += nel
                pg[conv.weight] = it["dw"]
            finish_items.append(it)

        if general is not None:
            feats, pqs, table = general
            score_ws = [sd.weight for sd in m.score_dsn]
            if obj is not None:
                out, label, sums, weights, divisor = obj
                dfs, reds, fb = ops.tail_general_bwd(
                    feats, pqs, score_ws, table, n, h, w, fast,
                    objective=(out, label, sums, weights, divisor, g_total.detach().contiguous().float()),
                    want_fuse_bias=grads[4] is not None)
                if fb is not None:
                    pg[m.fuse.bias] = fb.reshape(m.fuse.bias.shape)
            else:
                dfs, reds, _ = ops.tail_general_bwd(feats, pqs, score_ws, table, n, h, w, fast, grads=list(grads))
                if grads[4] is not None:
                    pg[m.fuse.bias] = ops.sum_f32(grads[4], deterministic=det).reshape(m.fuse.bias.shape)
        elif obj is not None:
            # tail + loss backward in ONE launch: dL/dlogit is formed on the fly (never written), d fuse.bias comes from
            # the forward's sums
            out, label, sums, weights, divisor = obj
            dpq, fb = ops.tail_loss_bwd(out, label, sums, weights, divisor, g_total.detach().contiguous().float(),
                                        n, h, w, want_fuse_bias=grads[4] is not None, deterministic=det, void=ctx.void)
            if fb is not None:
                pg[m.fuse.bias] = fb.reshape(m.fuse.bias.shape)
        else:
            dpq = ops.tail_bwd(list(grads), n, h, w, deterministic=det)
            if grads[4] is not None:
                pg[m.fuse.bias] = ops.sum_f32(grads[4], deterministic=det).reshape(m.fuse.bias.shape)
        # one zeroed buffer for all 13 trunk bias gradients; the dgrad / unpool epilogues accumulate into its slices
        flat_convs = [c for stage in convs for c in stage]
        bias_buf = torch.zeros(sum(c.out_channels for c in flat_convs), dtype=torch.float32, device=xin.device)
        bias_slices, bias_direct, boff = {}, set(), 0
        for c in flat_convs:
            tgt = grad_target(c.bias)
            if tgt is not None:
                bias_direct.add(c)
            bias_slices[c] = tgt if tgt is not None else bias_buf[boff:boff + c.out_channels]
            boff += c.out_channels

        def bias_grad(c):                              # None: already accumulated into c.bias.grad
            return None if c in bias_direct else bias_slices[c]
        if general is not None:
            # every parameter gradient of the tail from H, gA and the source sums (one launch); side_prep's weight
            # gradient comes from the tensor-core wgrad below, its data gradient from a dgrad conv 16 -> C
            learn = bool(getattr(m, "learn_upsampling", False))
            small = torch.zeros(64 + 4 * 33, dtype=torch.float32, device=xin.device)
            d_up = [torch.empty_like(l.weight) for l in m.upscale] if learn else None
            d_up1 = [torch.empty_like(l.weight) for l in m.upscale_] if learn else None
            d_score_w = [small[64 + 33 * i:80 + 33 * i] if grads[i] is not None else None for i in range(4)]
            d_score_b = [small[80 + 33 * i:81 + 33 * i] if grads[i] is not None else None for i in range(4)]
            d_side_b = [small[81 + 33 * i:97 + 33 * i] for i in range(4)]
            ops.upsampling_grads_finish(reds, [l.weight for l in m.upscale], m.fuse.weight, d_up, d_up1,
                                        small[:64] if grads[4] is not None else None, d_score_w, d_score_b, d_side_b)
            if grads[4] is not None:
                pg[m.fuse.weight] = small[:64].view(m.fuse.weight.shape)
            for i in range(4):
                pg[m.side_prep[i].bias] = d_side_b[i]
                if grads[i] is not None:
                    pg[m.score_dsn[i].weight] = d_score_w[i].view(m.score_dsn[i].weight.shape)
                    pg[m.score_dsn[i].bias] = d_score_b[i].view(m.score_dsn[i].bias.shape)
                if learn and grads[4] is not None:
                    pg[m.upscale[i].weight] = d_up[i]
                if learn and grads[i] is not None:
                    pg[m.upscale_[i].weight] = d_up1[i]
                wgrad(m.side_prep[i], acts[i + 1][-1], dfs[i])
        else:
            # every parameter gradient of the side branch from G[t][o][c] = sum_px dpq[px - t][o] x[px][c] (one pass over
            # the stage output per scale) and one finish launch for the four scales
            fold = engine._folded_side_all()
            side_params = [m.fuse.weight] if grads[4] is not None else []
            for i in range(4):
                side_params += [m.side_prep[i].weight, m.side_prep[i].bias]
                if grads[i] is not None:
                    side_params += [m.score_dsn[i].weight, m.score_dsn[i].bias]
            in_place = all(grad_target(p) is not None for p in side_params)
            if not in_place:
                fresh_small = torch.zeros(4 * 34 + 64, dtype=torch.float32, device=xin.device)
                fresh_side = torch.empty(sum(sp.weight.numel() for sp in m.side_prep), dtype=torch.float32,
                                         device=xin.device)
            ops.side_folded_wgrad_multi([acts[i + 1][-1] for i in range(4)], dpq, g_of, deterministic=det)   # G, one launch
            entries, off_side = [], 0
            for i in range(4):
                sp, sd = m.side_prep[i], m.score_dsn[i]
                e = {"g": g_of[i], "side_w": sp.weight.detach(), "side_b": sp.bias.detach(), "proj_w": engine._proj(i),
                     "c": sp.in_channels}
                if in_place:
                    e["d_side_w"], e["d_side_b"] = sp.weight.grad, sp.bias.grad
                    pg[sp.weight] = pg[sp.bias] = None
                    if grads[i] is not None:
                        e["d_score_w"], e["d_score_b"] = sd.weight.grad, sd.bias.grad
                        pg[sd.weight] = pg[sd.bias] = None
                    if grads[4] is not None:
                        e["d_fuse_w"] = m.fuse.weight.grad.view(-1)[16 * i:16 * i + 16]
                        pg[m.fuse.weight] = None
                else:
                    nel = sp.weight.numel()
                    e["d_side_w"] = fresh_side[off_side:off_side + nel].view(sp.weight.shape)
                    off_side += nel
                    small = fresh_small[34 * i:34 * i + 34]
                    e["d_side_b"] = small[0:16]
                    pg[sp.weight], pg[sp.bias] = e["d_side_w"], e["d_side_b"]
                    if grads[i] is not None:
                        e["d_score_w"], e["d_score_b"] = small[16:32], small[32:33]
                        pg[sd.weight] = e["d_score_w"].view(sd.weight.shape)
                        pg[sd.bias] = e["d_score_b"].view(sd.bias.shape)
                    if grads[4] is not None:
                        e["d_fuse_w"] = fresh_small[136 + 16 * i:136 + 16 * i + 16]
                entries.append(e)
            if not in_place and grads[4] is not None:
                pg[m.fuse.weight] = fresh_small[136:200].view(m.fuse.weight.shape)
            ops.side_grads_finish(entries, accumulate=in_place)
        dpool = None
        for i in range(4, -1, -1):
            # ReLU'(x) * (unpool(dpool) + side gradient); deepest stage: dpool None, the side branch is the only consumer;
            # stage 0 has no side branch.  Folded, the side gradient is formed on the fly from dpq and the fp32 folded
            # weights (18 FMAs per element)
            dside = dpq_i = wfold = None
            if i and general is not None:
                sp = m.side_prep[i - 1]
                _, dside, _ = ops.conv3x3(dfs[i - 1], engine._packed(sp, transpose_flip=True), None, sp.in_channels,
                                          fast=fast, out_act=False, out_f32=True)
            elif i:
                dpq_i, wfold = dpq[i - 1], fold[i - 1][2]
            dz = ops.unpool_mask(dpool, acts[i][-1], dside=dside, dpq=dpq_i, wfold=wfold,
                                 colsum=bias_slices[convs[i][-1]], deterministic=det)
            for j in range(len(convs[i]) - 1, -1, -1):
                conv = convs[i][j]
                pg[conv.bias] = bias_grad(conv)
                if i == j == 0:                        # conv1_1: weight and input gradient from the fp32 frame
                    pg[conv.weight], dx = ops.conv_first_bwd(xin, dz, conv.weight.detach(), ctx.needs_input_grad[1],
                                                             deterministic=det)
                    break
                inp = inputs[conv]
                wgrad(conv, inp, dz)
                wt = engine._packed(conv, transpose_flip=True)
                if j > 0:
                    dz, _, _ = ops.conv3x3(dz, wt, None, conv.in_channels, fast=fast, mask=inp.hi,
                                           colsum=bias_slices[convs[i][j - 1]], deterministic=det)
                else:
                    dpool, _, _ = ops.conv3x3(dz, wt, None, conv.in_channels, fast=fast)
        ops.wgrad_finish(finish_items)
        ctx.saved = None
        ctx.objective = None
        params = ctx.params
        ctx.params = None
        ctx.general = None
        return (None, dx, None) + tuple(pg.get(p) for p in params)


def osvos_apply(engine, x):
    params = engine._param_list()
    outs = _OSVOSFunction.apply(engine, x, None, *params)
    return list(outs)


def osvos_apply_objective(engine, x, label, loss_weights, divisor, void=False):
    """Forward + the weighted class-balanced BCE objective as one autograd node (``void``: label < 0 is left out).
    -> (maps: list of 5 [N,1,H,W] logit tensors (detached), total: 0-dim differentiable loss, per_map: [5] losses)."""
    params = engine._param_list()
    res = _OSVOSFunction.apply(engine, x, (label, loss_weights, divisor, bool(void)), *params)
    return list(res[:5]), res[5], res[6]

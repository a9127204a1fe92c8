"""Execution engine behind ``OSVOS.forward``: walks the module's parameter
containers and enqueues the native kernels (include/osvos_b200.h).  Python here
is plumbing - packing caches keyed on parameter versions, buffer allocation,
stream handling; all arithmetic is in csrc/.

Call graph replaced: reference networks/vgg_osvos.py:59-74 (forward) and, in
training, the autograd graph PyTorch builds for it.
"""
import contextlib
import gc
import os

import torch

from . import ops
from .layers.osvos_layers import bilinear_deconv_weight


@contextlib.contextmanager
def no_collection_during_capture():
    """Wrap a CUDA graph capture: collect the garbage first, then keep the cyclic collector off until it ends.  A dead
    reference cycle that still holds a captured graph (an unreferenced network and its engine) would otherwise be
    collected at a random moment, possibly inside the capture, and destroying a graph is not permitted while a stream
    captures: it invalidates the capture.  torch.cuda.graph no longer collects before capturing."""
    gc.collect()
    enabled = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if enabled:
            gc.enable()


class OSVOSEngine:
    def __init__(self, module):
        # no reference cycle through nn.Module registration: keep a plain attribute
        object.__setattr__(self, "m", module)
        self._packed_layouts = {}        # (conv, transpose_flip) -> (weight version, packed layout)
        self._derived = {}               # folded side weights, projections, upsampling table
        self._deconv_checked = {}
        # CUDA-graph cache for the inference path: (shape, device, precision, parameter versions) -> captured step.
        # One frame is ~22 kernel launches; replaying a graph removes the Python / launch overhead (OSVOS_CUDA_GRAPH=0
        # disables it).
        self._graphs = {}
        self._buffers_seen = {}          # (graph key, input address) -> calls seen (engine._forward_graphed)
        self._graphs_pver = None         # parameter versions the captured graphs belong to
        # graphs bound to input buffers: at most this many (each pins its activation pool); once reached, further
        # buffers go through the generic entry (one input copy) - no eviction, hence no capture / evict churn
        self.max_direct_graphs = 12
        self.use_cuda_graph = os.environ.get("OSVOS_CUDA_GRAPH", "1") != "0"
        # training loops of this package set this: backward adds weight / trunk-bias gradients straight into an
        # existing p.grad (and hands autograd None for them) instead of returning tensors for AccumulateGrad
        self.accumulate_param_grads_in_place = False

    def direct_grad_accumulation(self):
        """Context manager enabling in-place gradient accumulation for the backward passes run inside it."""
        eng = self

        class _Ctx:
            def __enter__(self):
                self.prev = eng.accumulate_param_grads_in_place
                eng.accumulate_param_grads_in_place = True

            def __exit__(self, *exc):
                eng.accumulate_param_grads_in_place = self.prev
                return False
        return _Ctx()

    # ------------------------------------------------------------ weight caches
    def _cached(self, key, params, make, cache=None):
        """make(), cached in `cache` (default: the derived-tensor cache) on the address and version of every tensor in
        `params`."""
        cache = self._derived if cache is None else cache
        ver = tuple((p.data_ptr(), p._version) for p in params)
        hit = cache.get(key)
        if hit is not None and hit[0] == ver:
            return hit[1]
        val = make()
        cache[key] = (ver, val)
        return val

    def _packed(self, conv, transpose_flip=False):
        """conv's packed tensor-core layout (transposed and flipped for the data gradient)."""
        return self._cached((conv, transpose_flip), [conv.weight],
                            lambda: ops.pack_conv3x3_weights(conv.weight, transpose_flip), self._packed_layouts)

    def _tensor_core_convs(self):
        """Every 3x3 conv that runs on the packed tensor-core path: the trunk convs (conv1_1 takes its OIHW weights
        directly) and, when the general tail runs (uses_general_tail), the four side_prep convs, whose forward and
        data-gradient convolutions then read packed layouts too.  On the folded path side_prep is folded with its 1x1
        projections instead (engine._folded_side_all) and has no packed layout."""
        convs = [c for stage in self.m.trunk_convs() for c in stage][1:]
        return convs + list(self.m.side_prep) if self.uses_general_tail() else convs

    def packed_weight_table(self):
        """[(weight Parameter, forward layout, transposed+flipped layout)] of the tensor-core convs, packed now if
        stale.  optim.FusedSGD rewrites these buffers in place from the updated weights."""
        return [(conv.weight, self._packed(conv), self._packed(conv, transpose_flip=True))
                for conv in self._tensor_core_convs()]

    def restamp_packed(self):
        """Declare the cached layouts of the tensor-core convs current for the present parameter versions (called by
        optim.FusedSGD after it has updated the weights AND those layouts in one kernel).  Other cached layouts, such
        as side_prep's on the folded path, were not rewritten and keep their stamps."""
        for conv in self._tensor_core_convs():
            for flip in (False, True):
                hit = self._packed_layouts.get((conv, flip))
                if hit is not None:
                    self._packed_layouts[(conv, flip)] = (((conv.weight.data_ptr(), conv.weight._version),), hit[1])

    def drop_derived_caches(self, keep_packed=False):
        """Forget cached derived tensors; with keep_packed the packed conv layouts (static buffers a captured graph
        may point at) are kept."""
        self._derived.clear()
        if not keep_packed:
            self._packed_layouts.clear()

    def _param_list(self):
        """Parameters the native path differentiates: everything, the eight deconvolution weights only when the module
        learns its upsampling (otherwise they are fixed taps and their .grad stays None)."""
        m = self.m
        extra = ([l.weight for l in m.upscale] + [l.weight for l in m.upscale_]
                 if getattr(m, "learn_upsampling", False) else [])
        return ([p for p in m.stages.parameters()] + [p for p in m.side_prep.parameters()]
                + [p for p in m.score_dsn.parameters()] + [m.fuse.weight, m.fuse.bias] + extra)

    def _proj(self, i):
        m = self.m
        sd, fu = m.score_dsn[i], m.fuse
        return self._cached(("proj", i), [sd.weight, fu.weight],
                            lambda: torch.cat([sd.weight.detach().reshape(16),
                                               fu.weight.detach().reshape(64)[16 * i:16 * i + 16]]).float().contiguous())

    def _folded_side_all(self):
        """[(packed operand, bias2, fp32 W' [9,2,C])] of the four side scales, folded by ONE launch and cached on the
        versions of every parameter that enters (training re-folds after each optimizer step)."""
        m = self.m
        deps = [m.fuse.weight]
        for i in range(4):
            deps += [m.side_prep[i].weight, m.side_prep[i].bias, m.score_dsn[i].weight, m.score_dsn[i].bias]
        return self._cached(("fold_all",), deps, lambda: ops.fold_side_weights_multi(
            [(m.side_prep[i].weight, m.side_prep[i].bias.detach(), self._proj(i), m.score_dsn[i].bias.detach())
             for i in range(4)]))

    def _deconvs_bilinear(self):
        """True when the eight deconvolution weights are the fixed bilinear taps interp_surgery writes (reference
        layers/osvos_layers.py:72-85), the only weights the folded tail implements.  Checked once per weight version
        (a host sync), never inside a graph capture: the eager warm-up before each capture fills the cache."""
        m = self.m
        for name, lst in (("upscale", m.upscale), ("upscale_", m.upscale_)):
            for i, lay in enumerate(lst):
                w = lay.weight
                key = (name, i)
                ver = (w.data_ptr(), w._version)
                hit = self._deconv_checked.get(key)
                if hit is None or hit[0] != ver:
                    ref = bilinear_deconv_weight(w.shape[0], w.shape[1], w.shape[2]).to(w.device)
                    ok = tuple(w.shape[2:]) == (2 ** (i + 2),) * 2 and torch.equal(w.detach().float(), ref)
                    hit = self._deconv_checked[key] = (ver, ok)
                if not hit[1]:
                    return False
        return True

    def uses_general_tail(self):
        """Which tail runs: the general one (csrc/tail_general.cu, DESIGN.md §20) when the module learns its upsampling
        or its deconvolution weights are not the bilinear taps, else the folded one (tail.cu).  With learn_upsampling the
        weight check is skipped, so a training step does not wait for the host."""
        return bool(getattr(self.m, "learn_upsampling", False)) or not self._deconvs_bilinear()

    def _upsampling_table(self):
        """V (upscale[k] folded with its slice of fuse.weight) and the upscale_[k] taps in one table, cached on the
        versions of the nine weights that enter (an optimizer step re-folds)."""
        m = self.m
        deps = [m.fuse.weight] + [l.weight for l in m.upscale] + [l.weight for l in m.upscale_]
        return self._cached(("upsampling",), deps, lambda: ops.upsampling_fold(
            [l.weight for l in m.upscale], [l.weight for l in m.upscale_], m.fuse.weight))

    def _side_features(self, stage_outs, fast, simt=False):
        """(feats, pqs) of the four scales: side_prep's 16 fp32 features and their projections (simt: the SIMT conv and
        a separate projection)."""
        m = self.m
        feats, pqs = [], []
        for i, full in enumerate(stage_outs):
            sp = m.side_prep[i]
            if simt:
                _, feat, _ = ops.conv3x3(full, self._packed(sp), sp.bias.detach(), 16, relu=False, fast=fast,
                                         out_act=False, out_f32=True, simt=True)
                pq = ops.side_project(feat, self._proj(i), m.score_dsn[i].bias.detach())
            else:
                _, feat, pq = ops.conv3x3(full, self._packed(sp), sp.bias.detach(), 16, relu=False, fast=fast,
                                          out_act=False, out_f32=True, proj_w=self._proj(i),
                                          proj_b=m.score_dsn[i].bias.detach())
            feats.append(feat)
            pqs.append(pq)
        return feats, pqs

    def _side_outputs(self, stage_outs, fast, want_feats=False, simt=False):
        """(feats | None, pqs) of the four side scales from the stage outputs of stages 1-4.  When the folded tail runs
        and no side features are wanted, side_prep o (score_dsn, fuse slice) is folded into one 3x3 conv C -> 2
        (include/osvos_b200.h) and the four scales run in ONE launch; the features themselves are then never formed."""
        if want_feats or simt or self.uses_general_tail():
            return self._side_features(stage_outs, fast, simt)
        return None, ops.side_folded_multi(stage_outs, self._folded_side_all(), fast=fast)

    def _trunk(self, x, fast, keep, simt=False, fuse_stage1=False):
        """The 13 trunk convs over the fp32 NCHW frame x -> (acts, pooled).  With `keep`, acts[i] lists the outputs of
        stage i's convs and pooled[i] is stage i's input (the backward reads them all); without it acts[i] holds only
        the stage's output and pooled stays [None], so each inner activation is freed once the next conv has read it.
        The last conv of stages 0-3 has the 2x2 max pool fused into its epilogue (simt: SIMT convs and a separate pool
        after stages 1-3); conv1_2's full-resolution output is only written when kept.  fuse_stage1: conv1_1 and
        conv1_2 in one kernel (exact-mode inference)."""
        convs = self.m.trunk_convs()
        c11, c12 = convs[0]
        acts, pooled = [[]], [None]
        if fuse_stage1:
            full, a = ops.stage1_fused(x, c11.weight.detach().contiguous().float(), c11.bias.detach(),
                                       self._packed(c12), c12.bias.detach(), pool=True, out_act=keep)
        else:
            a = ops.conv_first(x, c11.weight.detach(), c11.bias.detach(), relu=True, fast=fast)
            if keep:
                acts[0].append(a)
            full, a = ops.conv3x3(a, self._packed(c12), c12.bias.detach(), c12.out_channels, relu=True, fast=fast,
                                  pool=True, out_act=keep)
        acts[0].append(full)
        for i in range(1, 5):
            if keep:
                pooled.append(a)
            acts.append([])
            for j, conv in enumerate(convs[i]):
                if j == len(convs[i]) - 1 and i < 4 and not simt:
                    full, a = ops.conv3x3(a, self._packed(conv), conv.bias.detach(), conv.out_channels, relu=True,
                                          fast=fast, pool=True)
                else:
                    a, _, _ = ops.conv3x3(a, self._packed(conv), conv.bias.detach(), conv.out_channels, relu=True,
                                          fast=fast, simt=simt)
                    full = a
                if keep or j == len(convs[i]) - 1:
                    acts[i].append(full)
            if simt and i < 4:
                a = ops.maxpool2x2(full)
        return acts, pooled

    # ----------------------------------------------------------------- forward
    def forward(self, x, fresh_outputs=True):
        if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.size(1) != 3:
            raise ValueError("OSVOS.forward expects a [N, 3, H, W] tensor")
        if not x.is_cuda:
            raise RuntimeError("osvos_pytorch_b200.OSVOS runs on CUDA (sm_90a) only: move the module and the input "
                               "to the GPU.  There is no CPU fallback for the hot path.")
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.m.parameters()))
        if x.device != torch.device("cuda", torch.cuda.current_device()):
            with torch.cuda.device(x.device):       # kernels are enqueued on the current stream of x's device
                return self.forward(x, fresh_outputs)
        if needs_grad:
            from .autograd import osvos_apply
            return osvos_apply(self, x)
        if self.use_cuda_graph and not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(x, fresh_outputs)
        return self.forward_inference(x)

    def forward_objective(self, x, gts, loss_weights, size_average=False, batch_average=True, void=False):
        """See OSVOS.forward_objective."""
        if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.size(1) != 3:
            raise ValueError("OSVOS.forward_objective expects a [N, 3, H, W] tensor")
        if not x.is_cuda:
            raise RuntimeError("osvos_pytorch_b200.OSVOS runs on CUDA (sm_90a) only; there is no CPU fallback")
        if len(loss_weights) != 5:
            raise ValueError("loss_weights: one weight per output map (5)")
        if void and size_average:
            raise ValueError("void labels with size_average are not supported: the divisor would be the non-void count")
        if void and self.uses_general_tail():
            raise ValueError("void labels are not supported with learn_upsampling or non-bilinear deconvolution "
                             "weights (the general tail)")
        if size_average:
            divisor = float(gts.numel())
        elif batch_average:
            divisor = float(gts.size(0))
        else:
            divisor = 1.0
        if x.device != torch.device("cuda", torch.cuda.current_device()):
            with torch.cuda.device(x.device):
                return self.forward_objective(x, gts, loss_weights, size_average, batch_average, void)
        from .autograd import osvos_apply_objective
        return osvos_apply_objective(self, x, gts, loss_weights, divisor, void)

    def _forward_graphed(self, x, fresh_outputs=True):
        """Inference through a captured CUDA graph.  Two kinds of entry:
        * generic: the frame is copied into the graph's static input, the graph replayed (any input tensor);
        * direct: an input BUFFER that comes back (same address, shape, contiguous fp32 - the second call on) gets a graph
          captured on that buffer itself: no input copy.  A video pipeline feeds a small ring of device buffers
          (inference.SequenceSegmenter does), so in steady state every replay is direct.  At most `max_direct_graphs`
          of them; all graphs are dropped when a parameter changes.
        The five maps are handed back as fresh tensors (one device copy) unless `fresh_outputs` is False: then they are
        views of the entry's static output, valid until the SAME entry is replayed again (the sequence pipeline reads them
        straight into its pinned host buffers).  Re-captured when shapes or parameters change."""
        m = self.m
        pver = tuple((p.data_ptr(), p._version) for p in m.parameters())
        if pver != self._graphs_pver:                            # parameters changed: every captured graph is stale
            self._graphs.clear()
            self._buffers_seen.clear()
            self._graphs_pver = pver
        pkey = (tuple(x.shape), x.device.index, (m.precision, self.uses_general_tail()))
        direct_ok = x.dtype == torch.float32 and x.is_contiguous() and not x.requires_grad
        entry = None
        if direct_ok:
            dkey = pkey + (x.data_ptr(),)
            entry = self._graphs.get(dkey)
            if entry is None and sum(1 for k in self._graphs if len(k) == 4) < self.max_direct_graphs:
                seen = self._buffers_seen.get(dkey, 0) + 1
                if len(self._buffers_seen) > 64:
                    self._buffers_seen.clear()
                self._buffers_seen[dkey] = seen
                if seen >= 2:                                    # the buffer came back: give it its own graph
                    entry = self._capture(dkey, x, direct=True)
        if entry is None:
            entry = self._graphs.get(pkey)
            if entry is None:
                generic = [k for k in self._graphs if len(k) == 3]
                if len(generic) >= 4:                            # bounded: each entry pins its activation pool
                    self._graphs.pop(generic[0])
                entry = self._capture(pkey, x, direct=False)
        graph, static_x, outs, base = entry
        if static_x is not None:
            static_x.copy_(x, non_blocking=True)
        graph.replay()
        if not fresh_outputs:
            return list(outs)
        if base is not None:
            fresh = base.clone()
            n, _, h, w = (int(v) for v in x.shape)
            return [fresh[k, :n * h * w].view(n, 1, h, w) for k in range(5)]
        return [o.clone() for o in outs]

    def _capture(self, key, x, direct):
        """Capture the inference pass for `key`; direct: on the caller's buffer itself (no static input)."""
        self.forward_inference(x)                                # eager warm-up: packs weights, sets kernel attributes
        static_x = None if direct else x.detach().contiguous().float().clone()
        torch.cuda.synchronize(x.device)
        graph = torch.cuda.CUDAGraph()
        with no_collection_during_capture(), torch.cuda.graph(graph):
            outs = self.forward_inference(x if direct else static_x)
        base = outs[0]._base if outs[0]._base is not None else None
        entry = (graph, static_x, outs, base)
        self._graphs[key] = entry
        return entry

    @torch.no_grad()
    def forward_inference(self, x, simt=False, return_intermediates=False):
        """The inference pass (eager, or while a CUDA graph captures it).  Programmatic dependent launch is switched on
        for its kernels (every one of them waits before touching its predecessor's data, so only prologues overlap)."""
        from . import _native as nat
        lib = nat.load()
        prev = lib.osvos_set_pdl(1)
        try:
            return self._forward_inference(x, simt, return_intermediates)
        finally:
            lib.osvos_set_pdl(prev)

    def _forward_inference(self, x, simt=False, return_intermediates=False):
        m = self.m
        fast = m.precision == "fast"
        general = self.uses_general_tail()
        x = x.detach().contiguous().float()
        n, _, h, w = (int(v) for v in x.shape)
        # stage 1 as one kernel (opt-in): conv1_1 is computed inside conv1_2's kernel on its halo patch (no 105 MB round
        # trip).  Its fp32 conv1_1 builder warps take about as long as the tile's tensor work, and on an H100 it measured
        # slower than the two kernels (553 vs 584 frames/s at 480x854, 700 W card), so it is not the default.
        fuse_stage1 = not fast and not simt and os.environ.get("OSVOS_FUSE_STAGE1", "0") == "1"
        acts, _ = self._trunk(x, fast, keep=return_intermediates, simt=simt, fuse_stage1=fuse_stage1)
        feats, pqs = self._side_outputs([s[-1] for s in acts[1:]], fast, want_feats=return_intermediates, simt=simt)
        if general:
            out, _ = ops.tail_general_fwd(feats, pqs, self._upsampling_table(), m.fuse.bias.detach(), n, h, w)
        else:
            out, _ = ops.tail_fwd(pqs, m.fuse.bias.detach(), n, h, w)
        outs = [out[k] for k in range(5)]
        if not return_intermediates:
            return outs
        inter = {f"stage{i}": s[-1] for i, s in enumerate(acts)}
        for i in range(4):
            inter[f"side{i + 1}"], inter[f"pq{i + 1}"] = feats[i], pqs[i]
        return outs, inter

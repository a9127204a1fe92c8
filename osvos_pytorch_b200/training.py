"""Loop bodies of the two entry points, factored so that train_online.py / train_parent.py stay thin:
optimizer construction with the reference's per-group learning rates, synthetic DAVIS-shaped data,
the online fine-tune loop (train_online.py:112-149 of the reference) and the parent loop with the new
data-parallel exchange step (train_parent.py:129-176 + parallel.py)."""
import torch

from .engine import no_collection_during_capture
from .layers.osvos_layers import class_balanced_cross_entropy_loss
from .ops import MEANVAL  # noqa: F401  (dataloaders/davis_2016.py:19 of the reference)
ONLINE_WEIGHTS = (0.0, 0.0, 0.0, 0.0, 1.0)       # train_online.py:127: only the fused map is supervised


def _named(module, key):
    return [p for n, p in module.named_parameters() if key in n]


def make_optimizer(net, mode, lr=1e-8, wd=0.0002, momentum=0.9, fused=False, upsampling_lr=0.0):
    """SGD with the reference's parameter groups (``fused``: optim.FusedSGD - one launch per step, packed conv
    layouts re-emitted in the same pass - instead of torch.optim.SGD).
    online (train_online.py:77-88): stages / side_prep weights (wd) and biases (2 lr), deconvs lr 0,
    fuse at lr/100; score_dsn is NOT optimised.  parent (train_parent.py:85-103): additionally score_dsn at lr/10.
    ``upsampling_lr``: the lr of the two deconvolution groups (the reference's 0 by default; weight decay stays 0).  It
    only moves the weights when the net has ``learn_upsampling`` set, which makes backward write their gradients; a
    nonzero value on a net without it is refused rather than ignored."""
    if upsampling_lr != 0.0 and not getattr(net, "learn_upsampling", False):
        raise ValueError("upsampling_lr != 0 needs net.learn_upsampling = True: without it backward writes no gradient "
                         "for upscale / upscale_ and the optimizer would leave them unchanged")
    groups = [
        {"params": _named(net.stages, "weight"), "weight_decay": wd, "initial_lr": lr},
        {"params": _named(net.stages, "bias"), "lr": 2 * lr, "initial_lr": 2 * lr},
        {"params": _named(net.side_prep, "weight"), "weight_decay": wd, "initial_lr": lr},
        {"params": _named(net.side_prep, "bias"), "lr": 2 * lr, "initial_lr": 2 * lr},
    ]
    if mode == "parent":
        groups += [
            {"params": _named(net.score_dsn, "weight"), "lr": lr / 10, "weight_decay": wd, "initial_lr": lr / 10},
            {"params": _named(net.score_dsn, "bias"), "lr": 2 * lr / 10, "initial_lr": 2 * lr / 10},
        ]
    groups += [
        {"params": _named(net.upscale, "weight"), "lr": upsampling_lr, "initial_lr": upsampling_lr},
        {"params": _named(net.upscale_, "weight"), "lr": upsampling_lr, "initial_lr": upsampling_lr},
        {"params": [net.fuse.weight], "lr": lr / 100, "initial_lr": lr / 100, "weight_decay": wd},
        {"params": [net.fuse.bias], "lr": 2 * lr / 100, "initial_lr": 2 * lr / 100},
    ]
    if fused:
        from .optim import FusedSGD
        return FusedSGD(groups, lr=lr, momentum=momentum, engine=net._engine)
    return torch.optim.SGD(groups, lr=lr, momentum=momentum)


def synthetic_batch(n, h, w, seed, device):
    """DAVIS-shaped synthetic sample: BGR 0..255 mean-subtracted image, ~30 % positive mask."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(n, 3, h, w, generator=g) * 255.0 - torch.tensor(MEANVAL).view(1, 3, 1, 1)
    gt = (torch.rand(n, 1, h, w, generator=g) > 0.7).float()
    return {"image": img.to(device), "gt": gt.to(device)}


class GraphedTrainStep:
    """Forward + objective + backward of one fixed-shape micro-batch captured in a CUDA graph (SURVEY.md 8f item 1:
    at > 250 fwd+bwd/s the ~120 kernel launches and the Python around them cost as much as the kernels).

    Gradients ACCUMULATE into the static ``p.grad`` buffers exactly like repeated ``loss.backward()`` calls
    (train_online.py:140-149): call ``zero_grads()`` after ``optimizer.step()`` (``optimizer.zero_grad()`` with
    set_to_none would detach the graph from its buffers).  The weight-packing kernels are part of the graph, so
    parameter updates between replays are picked up - unless ``external_pack`` is set: then the packed conv
    layouts are static buffers outside the graph that ``optim.FusedSGD`` rewrites in its update kernel (no
    packing work per micro-batch; only valid with that optimizer).  ``objective(outputs, gts) -> scalar tensor``, or a
    tuple of five loss weights = the package's fused objective (``OSVOS.forward_objective``).

    The graph keeps the kernels of the mode ``torch.are_deterministic_algorithms_enabled()`` had at capture; a replay
    under the other mode raises instead of silently running those.

    ``void``: gt < 0 marks void pixels, left out of the fused objective (``OSVOS.forward_objective(void=True)``); only
    with loss weights as the objective.
    """

    def __init__(self, net, objective, sample, grad_scale=1.0, external_pack=False, void=False):
        if void and callable(objective):
            raise ValueError("GraphedTrainStep(void=True) needs the fused objective (a tuple of five loss weights)")
        self.net, self.objective, self.grad_scale, self.void = net, objective, float(grad_scale), bool(void)
        self.deterministic = torch.are_deterministic_algorithms_enabled()
        self.x = sample["image"].detach().clone()
        self.gt = sample["gt"].detach().clone()
        from .parallel import trainable_parameters
        self.params = trainable_parameters(net)
        for p in self.params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        keep = [p.grad.clone() for p in self.params]
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(2):                              # warm-up: lazy kernel attributes, allocator, autograd
                self._body()
        cur.wait_stream(side)
        for p, g in zip(self.params, keep):                 # undo the warm-up accumulation
            p.grad.copy_(g)
        if external_pack:
            net._engine.packed_weight_table()               # packed now, outside the graph
        # everything else derived from parameters is recomputed inside the graph
        net._engine.drop_derived_caches(keep_packed=external_pack)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        try:
            with no_collection_during_capture(), torch.cuda.graph(self.graph):
                self.loss = self._body()
        finally:
            # graph-private buffers must not serve eager calls (also after a failed capture: the cached packed layouts
            # would point into the aborted capture's memory pool)
            net._engine.drop_derived_caches(keep_packed=external_pack)

    def _body(self):
        if not callable(self.objective):
            # loss weights of the package's fused objective (tail + five losses = one kernel each way); grad_scale is
            # folded into the weights, so no scaling kernel runs either
            w = [float(v) * self.grad_scale for v in self.objective]
            _, total, per_map = self.net.forward_objective(self.x, self.gt, w, void=self.void)
            with self.net._engine.direct_grad_accumulation():
                total.backward()
            self.per_map = per_map
            nz = [k for k, v in enumerate(self.objective) if float(v) != 0.0]
            if len(nz) == 1 and float(self.objective[nz[0]]) == 1.0:
                return per_map[nz[0]]                       # the unscaled objective IS that map's loss: no extra kernel
            return total.detach() if self.grad_scale == 1.0 else total.detach() / self.grad_scale
        outputs = self.net(self.x)
        loss = self.objective(outputs, self.gt)
        with self.net._engine.direct_grad_accumulation():   # p.grad buffers are static: add into them in the kernels
            (loss * self.grad_scale).backward()
        return loss.detach()

    def __call__(self, sample=None):
        if torch.are_deterministic_algorithms_enabled() != self.deterministic:
            raise RuntimeError(
                "GraphedTrainStep was captured with torch.use_deterministic_algorithms(%s) but is replayed with %s; "
                "capture a new step after changing the setting" % (self.deterministic, not self.deterministic))
        if sample is not None:
            self.x.copy_(sample["image"], non_blocking=True)
            self.gt.copy_(sample["gt"], non_blocking=True)
        self.graph.replay()
        return self.loss

    def zero_grads(self, skip=()):
        """Zero the accumulated gradients (``skip``: parameters already cleared, e.g. by FusedSGD.step(zero_grad=True))."""
        skip = {id(p) for p in skip}
        for p in self.params:
            if id(p) not in skip:
                p.grad.zero_()


def online_finetune(net, sample_fn, iters, n_ave_grad=5, lr=1e-8, wd=0.0002, log_every=0, log=print, use_graph=True,
                    fused_optimizer=True, upsampling_lr=0.0, void=False):
    """`iters` forward/backward passes on the annotated frame, SGD step every `n_ave_grad` (reference
    train_online.py:112-149).  Losses are kept on the device; one host read per `log_every` iterations
    instead of the reference's per-iteration .item() sync.  With `use_graph` the fwd+loss+bwd of a micro-batch
    is a replayed CUDA graph (shapes must not change between iterations); with `fused_optimizer` the SGD step,
    the gradient zeroing and the repack of the conv weights are one kernel (optim.FusedSGD).  ``void``: gt < 0 marks
    void pixels, left out of the loss.  Returns the list of logged losses."""
    net.train()
    opt = make_optimizer(net, "online", lr, wd, fused=fused_optimizer, upsampling_lr=upsampling_lr)
    opt.zero_grad()
    opt_params = [p for g in opt.param_groups for p in g["params"]]
    history, running = [], None
    step = None
    for it in range(iters):
        sample = sample_fn(it)
        inputs, gts = sample["image"], sample["gt"]
        if use_graph:
            if step is None:
                step = GraphedTrainStep(net, ONLINE_WEIGHTS, sample, grad_scale=1.0 / n_ave_grad,
                                        external_pack=fused_optimizer, void=void)
            loss_val = step(sample)
            running = loss_val.clone() if running is None else running + loss_val
            if (it + 1) % n_ave_grad == 0:
                if fused_optimizer:
                    opt.step(zero_grad=True)
                    step.zero_grads(skip=opt_params)
                else:
                    opt.step()
                    step.zero_grads()
        else:
            # fuse-map loss only (train_online.py:127), 1/nAveGrad folded into the weight (train_online.py:140)
            _, loss, per_map = net.forward_objective(inputs, gts, [v / n_ave_grad for v in ONLINE_WEIGHTS], void=void)
            running = per_map[4].clone() if running is None else running + per_map[4]
            with net._engine.direct_grad_accumulation():
                loss.backward()
            if (it + 1) % n_ave_grad == 0:
                if fused_optimizer:
                    opt.step(zero_grad=True)
                else:
                    opt.step()
                    opt.zero_grad()
        if log_every and (it + 1) % log_every == 0:
            val = float(running) / log_every
            history.append(val)
            running = None
            log(f"[iter {it + 1:6d}] loss {val:.6f}")
    return history


class OnlineAdaptation:
    """Online adaptation of a fine-tuned network while a DAVIS-2016 sequence is segmented (OnAVOS, Voigtlaender & Leibe,
    BMVC 2017; DESIGN.md §28), for ``inference.SequenceSegmenter(adapt=...)``.  Before frame t >= 1 is segmented:
    one forward with the current weights, ops.adaptation_labels of its fused map against the last mask (the annotation
    ``first_mask`` for frame 1, then each segmented frame's mask) -> the frame's labels; then, unless the eroded last mask
    is empty (the object is lost: the frame is skipped), ``steps`` SGD steps of one micro-batch each.  Step s trains on
    the current frame when s = floor(i * steps / current_steps) for some i < current_steps, with loss weights
    (0, 0, 0, 0, ``weight``) on its labels (void pixels left out), and on a fresh sample of ``sample_fn`` (the
    fine-tuning's augmented first-frame sampler, called with a running count) with ONLINE_WEIGHTS otherwise.

    ``first_mask``: the annotation, uint8 [1,H,W] on the device at the network resolution.  ``alpha``, ``distance`` and
    ``erosion``: the targets' parameters (ops.adaptation_labels).  The optimizer is make_optimizer(net, "online", lr, wd,
    fused=True), with fresh momentum; the two micro-batches are GraphedTrainSteps over the packed layouts FusedSGD
    rewrites, each captured when it first runs, so a run that takes no step of a kind captures no graph for it.
    ``counts`` lists each adapted frame's int32 [3] counts {|E|, #positive, #negative}; ``skipped`` the
    number of frames with |E| = 0."""

    def __init__(self, net, sample_fn, first_mask, lr, wd, steps=15, current_steps=3, weight=0.05, alpha=0.97,
                 distance=220, erosion=15):
        from . import ops
        if isinstance(steps, bool) or not isinstance(steps, int) or steps < 0:
            raise ValueError(f"steps must be a non-negative integer, got {steps!r}")
        if isinstance(current_steps, bool) or not isinstance(current_steps, int) or not 0 <= current_steps <= steps:
            raise ValueError(f"current_steps must be an integer in 0 .. steps ({steps}), got {current_steps!r}")
        ops.adaptation_threshold(alpha)                     # the checks of ops.adaptation_labels, before anything runs
        ops._non_negative_int(distance, "distance")
        ops._non_negative_int(erosion, "erosion")
        if not torch.is_tensor(first_mask) or first_mask.dtype != torch.uint8 or first_mask.dim() != 3 \
                or int(first_mask.shape[0]) != 1 or not first_mask.is_cuda:
            raise ValueError("first_mask must be a uint8 CUDA tensor [1,H,W] at the network resolution")
        if net._engine.uses_general_tail():
            raise ValueError("online adaptation trains with void labels, which the general tail (learn_upsampling or "
                             "non-bilinear deconvolution weights) does not support")
        self.net, self.sample_fn = net, sample_fn
        self.steps, self.current_steps = steps, current_steps
        self.weight, self.alpha, self.distance, self.erosion = float(weight), float(alpha), distance, erosion
        self.current_at = {i * steps // current_steps for i in range(current_steps)}
        self.last_mask = first_mask.detach().clone()
        self.opt = make_optimizer(net, "online", lr, wd, fused=True)
        self.opt.zero_grad()
        in_opt = {id(p) for g in self.opt.param_groups for p in g["params"]}
        from .parallel import trainable_parameters
        self._not_in_opt = [p for p in trainable_parameters(net) if id(p) not in in_opt]
        self._first = self._current = None
        self.samples = 0
        self.counts = []
        self.skipped = 0
        self._events = []

    @torch.enable_grad()
    def adapt(self, x):
        """The adaptation before the frame in ``x`` (fp32 [1,3,H,W] at the network resolution) is segmented.  Reads the
        frame's counts back (one host synchronisation).  Runs with autograd enabled, also inside torch.no_grad() (the
        segmenter's forwards): a training step captured here at its first use records its backward."""
        from . import ops
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fused = self.net._engine.forward_inference(x)[-1]
        cur = self._current                                # once captured, its static buffers take the frame directly
        labels, counts = ops.adaptation_labels(fused, self.last_mask, self.alpha, self.erosion, self.distance,
                                               out=None if cur is None else cur.gt)
        if cur is not None:
            cur.x.copy_(x)
        counts = counts[0].cpu()
        self.counts.append(counts)
        if int(counts[0]) == 0:                            # the object is lost: no step
            self.skipped += 1
        else:
            for s in range(self.steps):
                if s in self.current_at:
                    if self._current is None:              # captured on this frame's image and labels
                        self._current = GraphedTrainStep(self.net, (0.0, 0.0, 0.0, 0.0, self.weight),
                                                         {"image": x, "gt": labels}, external_pack=True, void=True)
                    self._current()
                else:
                    sample = self.sample_fn(self.samples)
                    self.samples += 1
                    if self._first is None:
                        self._first = GraphedTrainStep(self.net, ONLINE_WEIGHTS, sample, external_pack=True)
                    self._first(sample)
                self.opt.step(zero_grad=True)
                for p in self._not_in_opt:                 # score_dsn: gradients written, not trained online
                    p.grad.zero_()
        t1.record()
        self._events.append((t0, t1))

    def segmented(self, fused):
        """Record the frame's fused map (fp32 [1,1,H,W] at the network resolution) as the next frame's last mask."""
        from . import ops
        ops.logits_to_u8(fused, "mask", out=self.last_mask.view(fused.shape))

    def seconds(self):
        """Device time spent in adapt() so far (one synchronisation)."""
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self._events) / 1000.0


def parent_epoch(net, opt, bucket, batches, epoch, n_epochs, n_ave_grad=1, group=None, state=None, void=False):
    """One epoch of the parent objective on this rank's shard: deep-supervision loss
    (1 - epoch/nEpochs) * sum_{k<4} L_k + L_fuse (train_parent.py:143-147), gradient accumulation over
    `n_ave_grad` local micro-batches, then ONE allreduce(mean) and one SGD step.
    Returns the mean of the five losses over the micro-batches as a device tensor (the reference reads `.item()` of
    every loss in every iteration, train_parent.py:146: a host sync per step that exposes launch latency and, in data
    parallel, lets rank skew accumulate; here the host only waits when it logs).
    `state`: a dict the caller keeps across epochs; it carries the accumulation counter, which the reference does NOT
    reset at epoch boundaries (`aveGrad`, train_parent.py:125,165-172) - leftover micro-batches of an epoch whose length
    is not a multiple of nAveGrad complete their group in the next epoch instead of inflating its first step.
    ``void``: gt < 0 marks void pixels (DAVIS-2017's 255), left out of the five losses."""
    net.train()
    if state is None:
        state = {}
    state.setdefault("ave_grad", 0)
    side_w = 1.0 - epoch / n_epochs
    totals = torch.zeros(5, device=bucket.flat.device)
    count = 0
    for it, sample in enumerate(batches):
        # (1 - epoch/nEpochs) * sum(side losses) + fuse loss, / nAveGrad (train_parent.py:143-147,163), as the fused
        # objective: tail + five losses are one kernel forward and one backward
        w = [side_w / n_ave_grad] * 4 + [1.0 / n_ave_grad]
        _, loss, per_map = net.forward_objective(sample["image"], sample["gt"], w, void=void)
        totals += per_map
        count += 1
        with net._engine.direct_grad_accumulation():
            loss.backward()
        state["ave_grad"] += 1
        if state["ave_grad"] % n_ave_grad == 0:
            state["ave_grad"] = 0
            bucket.allreduce_mean(group)
            if hasattr(opt, "_engine"):                     # optim.FusedSGD: update + zeroing + repack in one kernel
                opt.step(zero_grad=True)
            else:
                opt.step()
                bucket.zero_()
    return totals / max(count, 1)          # DEVICE tensor [5]: no host sync per call; callers read it when they log


def timed_parent_steps(net, opt, bucket, make_batch, steps, warmup, epoch=0, n_epochs=240, group=None):
    """Benchmark helper: `steps` optimizer steps (1 micro-batch each); device time via CUDA events."""
    def one(i):
        parent_epoch(net, opt, bucket, [make_batch(i)], epoch, n_epochs, 1, group)
    for i in range(warmup):
        one(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        one(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps

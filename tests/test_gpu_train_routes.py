"""Every route the trainers take through the autograd node, held to the gated fp64 reference of the same step
(tests/train_routes_ref.py, DESIGN.md §11), and every buffer the node allocates checked to be written before it is read
(DESIGN.md §16).

(a) Gated matrix.  Each case builds a fresh seeded network, takes the ReLU masks and pool argmax of one eager training
    forward (engine.debug_capture) and evaluates the reference in fp64 on that linear piece.  The routes: the plain
    `net(x)` + the reference-style loss + `.backward()`; `forward_objective` + a direct backward (the kernels add into
    `p.grad`), with and without void labels; and GraphedTrainStep over K = 3 samples with grad_scale 1/3.  Each runs
    with atomic and with deterministic kernels, on the folded and the general tail, under the online, parent and mixed
    loss weights, onto no prior `.grad`, seeded non-zero ones, partial ones, or the views of a GradientBucket.  Some
    cases take an optimizer step and check a second window at the parameters read back after it, so that a stale folded
    table, general-tail table or packed layout shows.  Required: every parameter's ||got - ref|| / ||ref|| < GATED_TOL
    (SUM_TOL for the pixel-sum biases fuse.bias and side_prep.i.bias, whose terms cancel: tests/train_routes_ref.py),
    the set of parameters with a gradient equal to the reference's, the losses within 1e-4, and the input gradient.
(b) Written before read.  Under torch.use_deterministic_algorithms(True) torch fills every torch.empty with NaN (integers
    with their maximum); the node turns that fill off for its own buffers (ops.no_uninitialized_fill) on the grounds that
    its kernels write them in full.  Each deterministic case, the online fine-tuning loop and parent_epoch run once with
    the fill forced on and once without, each on a fresh network: the results must be bit-identical and free of NaN.
(c) The checker of (a) fails on a 1 % error in any one parameter and on a missing one."""
import contextlib
import dataclasses
import time

import pytest
import torch

from oracle import osvos_oracle as oc
from train_routes_ref import GATED_TOL, SUM_TOL, WEIGHTS, check_gradients, gates_of, reference_step, relnorm
from upsampling_ref import deconv_weights

pytestmark = pytest.mark.gpu
LOSS_TOL = 1e-4
WORST = {}                        # route -> (worst gated error, parameter, case)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    for route, (err, name, case) in sorted(WORST.items()):
        print(f"\n{route}: worst gated gradient error {err:.2e} ({name}; {case})")
    print(f"\ntest_gpu_train_routes.py: {time.time() - t0:.1f} s")


@dataclasses.dataclass(frozen=True)
class Case:
    route: str                    # "plain" | "objective" | "graphed"
    det: bool                     # deterministic kernels (torch.use_deterministic_algorithms)
    general: bool                 # general tail with learn_upsampling (dense deconvolution weights), else folded
    weights: str                  # key of WEIGHTS
    prior: str                    # .grad before the step: none | all | trunk | weights | bucket
    shape: tuple
    void: bool = False            # void labels (forward_objective(void=True) / GraphedTrainStep(void=True))
    opt: str = ""                 # then an optimizer step and a second window: fused | fused_ext | torch
    seed: int = 0

    def __str__(self):
        return "-".join([self.label, "det" if self.det else "atomic", "general" if self.general else "folded",
                         self.weights, self.prior, "x".join(map(str, self.shape))] + ([self.opt] if self.opt else []))

    @property
    def label(self):
        return self.route + ("+void" if self.void else "")


A, B, C, D = (1, 40, 56), (2, 37, 61), (3, 17, 9), (1, 480, 854)     # B: ceil-mode pooling at 3 of 4 pools; C: stage 5 2x1
# prior: "trunk" = the 13 trunk weights only (the side branch takes its fresh-buffer path); "weights" = the trunk and
# side_prep weights (some side-branch gradients exist, others do not: still the fresh path); "bucket" = the views of a
# GradientBucket, as parent_epoch has them
CASES = [
    Case("plain", False, False, "online", "none", A),
    Case("plain", True, False, "parent", "all", B, seed=1),
    Case("plain", False, True, "mixed", "trunk", C, seed=2),
    Case("plain", True, True, "parent", "bucket", A, seed=3),
    Case("objective", False, False, "mixed", "weights", B, seed=4),
    Case("objective", True, False, "online", "all", C, seed=5),
    Case("objective", False, True, "online", "bucket", B, seed=6),
    Case("objective", True, True, "mixed", "trunk", A, seed=7),
    Case("objective", True, False, "parent", "bucket", B, opt="fused", seed=8),
    Case("objective", False, False, "parent", "all", B, void=True, seed=9),
    Case("objective", True, False, "mixed", "trunk", C, void=True, seed=10),
    Case("objective", True, False, "online", "none", D, void=True, seed=11),
    Case("objective", False, False, "online", "bucket", A, void=True, seed=12),
    Case("graphed", False, False, "online", "none", D, opt="fused_ext", seed=13),
    Case("graphed", True, False, "parent", "bucket", B, opt="torch", seed=14),
    Case("graphed", False, True, "mixed", "none", C, opt="fused_ext", seed=15),
    Case("graphed", True, True, "online", "all", A, opt="torch", seed=16),
    Case("graphed", True, False, "mixed", "weights", C, void=True, opt="fused", seed=17),
]


@contextlib.contextmanager
def det_mode(on):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def make_net(case):
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS
    params = oc.he_params(seed=case.seed, include_upscale=True)
    if case.general:
        params.update(deconv_weights(case.seed + 100, "dense"))
    net = OSVOS(pretrained=0, verbose=False)
    net.load_state_dict(params)
    net.learn_upsampling = case.general
    return net.cuda().train()


def trainable(net):
    return [(n, p) for n, p in net.named_parameters() if net.learn_upsampling or not n.startswith("upscale")]


def samples(case, window):
    """K = 3 different samples for the graphed route, one otherwise; void: 20 % void pixels, and with a batch > 1 the
    last element entirely void."""
    n, h, w = case.shape
    out = []
    for k in range(3 if case.route == "graphed" else 1):
        x, gt = oc.synthetic_frame(n, h, w, 7919 * case.seed + 31 * window + k)
        if case.void:
            g = torch.Generator().manual_seed(case.seed * 101 + k)
            gt = torch.where(torch.rand(gt.shape, generator=g) < 0.2, torch.full_like(gt, -1.0), gt)
            if n > 1:
                gt[-1] = -1.0
        out.append((x.cuda(), gt.cuda()))
    return out


def capture(net, x):
    """The 13 trunk activations (NCHW fp32) of one eager training forward; no backward runs."""
    from osvos_pytorch_b200 import ops
    cap = {}
    net._engine.debug_capture = cap
    try:
        with torch.enable_grad():
            outs = net(x)
        acts = [ops.act_to_nchw(a) for stage in cap["acts"] for a in stage]
    finally:
        net._engine.debug_capture = None
    del outs, cap
    return acts


def set_prior(net, case, scale):
    """Seeded non-zero prior gradients; ``scale(name)``: their rms for that parameter."""
    g = torch.Generator().manual_seed(977 + case.seed)
    for name, p in trainable(net):
        if case.prior == "none":
            continue
        if case.prior == "trunk" and not (name.startswith("stages.") and name.endswith(".weight")):
            continue
        if case.prior == "weights" and not ((name.startswith("stages.") or name.startswith("side_prep."))
                                            and name.endswith(".weight")):
            continue
        val = (torch.randn(p.shape, generator=g) * scale(name)).float().cuda()
        if p.grad is not None:                      # GradientBucket views, GraphedTrainStep's static buffers
            p.grad.copy_(val)
        else:
            p.grad = val


def written(net, prior):
    """{name: gradient the step wrote (p.grad - prior), or None when p.grad is None or unchanged}."""
    got = {}
    for name, p in trainable(net):
        if p.grad is None or (name in prior and torch.equal(p.grad, prior[name])):
            got[name] = None
        else:
            got[name] = p.grad.double() - prior[name].double() if name in prior else p.grad.double()
    return got


def run_window(net, case, batch, grad_scale, step, want_dx):
    """The route over the samples of one window -> {maps, per_map, loss, dx} (per sample) and the activations the
    non-graphed routes saw."""
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss as cbce
    w = WEIGHTS[case.weights]
    res = {"maps": [], "per_map": [], "loss": [], "dx": [], "acts": []}
    for x, gt in batch:
        if case.route == "graphed":
            loss = step({"image": x, "gt": gt})
            res["loss"].append(loss.clone())
            res["per_map"].append(step.per_map.clone())
            continue
        xin = x.clone().requires_grad_(want_dx)
        cap = {}
        net._engine.debug_capture = cap
        try:
            if case.route == "plain":
                outs = net(xin)
                per = [cbce(o, gt, size_average=False) for o in outs]
                total = sum(wk * grad_scale * lk for wk, lk in zip(w, per) if wk != 0.0)
                total.backward()
                per = torch.stack([lk.detach() for lk in per])
            else:
                outs, total, per = net.forward_objective(xin, gt, [wk * grad_scale for wk in w], void=case.void)
                with net._engine.direct_grad_accumulation():
                    total.backward()
        finally:
            net._engine.debug_capture = None
        res["acts"].append([ops.act_to_nchw(a) for stage in cap["acts"] for a in stage])
        res["maps"].append(torch.cat([o.detach() for o in outs]))
        res["per_map"].append(per.detach().clone())
        res["loss"].append(total.detach().clone())
        res["dx"].append(xin.grad.clone() if want_dx else None)
    return res


def optimizer_step(net, case, step):
    """One SGD step (momentum 0.9) whose per-parameter lr moves each weight by about 1e-3 of its norm."""
    from osvos_pytorch_b200.optim import FusedSGD
    groups = []
    for _, p in trainable(net):
        if p.grad is None:
            continue
        gn, pn = float(p.grad.double().norm()), float(p.detach().double().norm())
        groups.append({"params": [p], "lr": 1e-3 * pn / gn if gn > 0 else 0.0})
    if case.opt in ("fused", "fused_ext"):
        opt = FusedSGD(groups, lr=0.0, momentum=0.9, engine=net._engine)
        opt.step(zero_grad=True)
        if step is not None:
            step.zero_grads(skip=[g["params"][0] for g in groups])
    else:
        opt = torch.optim.SGD(groups, lr=0.0, momentum=0.9)
        opt.step()
        if step is not None:
            step.zero_grads()
        else:
            for g in groups:
                g["params"][0].grad.zero_()


def run_case(case, check=True):
    """Everything case runs on the device; with ``check`` it is held to the gated fp64 reference as it goes.  ->
    the CUDA results (maps, losses, input gradients, final gradients and parameters) for the bit-identity checks."""
    from osvos_pytorch_b200.parallel import GradientBucket, trainable_parameters
    from osvos_pytorch_b200.training import GraphedTrainStep
    k_samples = 3 if case.route == "graphed" else 1
    grad_scale = 1.0 / k_samples
    want_dx = case.route != "graphed" and not case.void
    out = {"maps": [], "per_map": [], "loss": [], "dx": []}
    with det_mode(case.det):
        net = make_net(case)
        bucket = GradientBucket(trainable_parameters(net)) if case.prior == "bucket" else None
        batch = samples(case, 0)
        step = None
        if case.route == "graphed":
            step = GraphedTrainStep(net, WEIGHTS[case.weights], {"image": batch[0][0], "gt": batch[0][1]},
                                    grad_scale=grad_scale, external_pack=case.opt == "fused_ext", void=case.void)
    for window in range(2 if case.opt else 1):
        if window:
            batch = samples(case, window)
        with det_mode(case.det):
            acts = [capture(net, x) for x, _ in batch]
            if case.route == "graphed":      # the graph's activations cannot be read: its gates come from these
                assert all(torch.equal(u, v) for u, v in zip(capture(net, batch[0][0]), acts[0])), \
                    "two eager forwards differ"
        refs = None
        if check:
            params64 = {k: v.detach().double() for k, v in net.state_dict().items()}
            refs = [reference_step(params64, x.double(), gt.double(), WEIGHTS[case.weights], grad_scale, void=case.void,
                                   gates=gates_of(a), general=case.general, learn_upsampling=case.general,
                                   want_dx=want_dx) for a, (x, gt) in zip(acts, batch)]
        if window == 0:
            ref_rms = {} if refs is None else {k: float(g.pow(2).mean().sqrt()) for k, g in refs[0]["grads"].items()}
            set_prior(net, case, lambda name: ref_rms.get(name, 1e-3))
        prior = {n: p.grad.detach().clone() for n, p in trainable(net) if p.grad is not None}
        with det_mode(case.det):
            res = run_window(net, case, batch, grad_scale, step, want_dx)
            torch.cuda.synchronize()
        for a_route, a_eager in zip(res["acts"], acts):          # the training forward is deterministic in both modes
            assert all(torch.equal(u, v) for u, v in zip(a_route, a_eager)), "two eager forwards differ"
        if check:
            got = written(net, prior)
            ref_sum = {k: sum(r["grads"][k] for r in refs) for k in refs[0]["grads"]}
            worst, name = check_gradients(got, ref_sum)
            if worst > WORST.get(case.label, (-1.0,))[0]:
                WORST[case.label] = (worst, name, str(case) + (f" window {window}" if window else ""))
            for r, per, loss in zip(refs, res["per_map"], res["loss"]):
                want = r["per_map"].cpu()
                assert (per.double().cpu() - want).abs().max() <= LOSS_TOL * want.abs().max(), (per, want)
                want_loss = float(r["loss"]) / (grad_scale if case.route == "graphed" else 1.0)
                assert abs(float(loss) - want_loss) <= LOSS_TOL * abs(want_loss), (float(loss), want_loss)
            for r, dx in zip(refs, res["dx"]):
                if want_dx:
                    assert relnorm(dx, r["dx"]) < GATED_TOL
        if bucket is not None:                            # the gradients stay views of the bucket
            base = bucket.flat.untyped_storage().data_ptr()
            assert all(p.grad.untyped_storage().data_ptr() == base for p in bucket.params)
        for key in ("maps", "per_map", "loss", "dx"):
            out[key] += res[key]
        if window == 0 and case.route == "graphed" and case.det:
            eager_equals_graph(case, batch, grad_scale, prior, net)
        if case.opt and window == 0:
            with det_mode(case.det):
                optimizer_step(net, case, step)
    out["grads"] = {n: None if p.grad is None else p.grad.detach().clone() for n, p in trainable(net)}
    out["params"] = {n: p.detach().clone() for n, p in net.named_parameters()}
    del step, net
    return out


def eager_equals_graph(case, batch, grad_scale, prior, graphed_net):
    """Deterministic kernels: the graph's window is bit-identical to the same micro-batches run eagerly
    (forward_objective + a direct backward) on a fresh network with the same prior gradients."""
    with det_mode(True):
        net = make_net(case)
        for n, p in trainable(net):
            p.grad = prior[n].clone() if n in prior else torch.zeros_like(p)
        w = [wk * grad_scale for wk in WEIGHTS[case.weights]]
        for x, gt in batch:
            _, total, _ = net.forward_objective(x, gt, w, void=case.void)
            with net._engine.direct_grad_accumulation():
                total.backward()
    for (n, p), q in zip(trainable(net), [q for _, q in trainable(graphed_net)]):
        assert torch.equal(p.grad, q.grad), n


@pytest.mark.parametrize("case", CASES, ids=str)
def test_route_matches_the_gated_reference(case):
    run_case(case)


def test_matrix_covers_every_axis_value():
    axes = {"route": {"plain", "objective", "graphed"}, "det": {False, True}, "general": {False, True},
            "weights": set(WEIGHTS), "prior": {"none", "all", "trunk", "weights", "bucket"}, "shape": {A, B, C, D},
            "void": {False, True}, "opt": {"", "fused", "fused_ext", "torch"}}
    for axis, values in axes.items():
        assert {getattr(c, axis) for c in CASES} == values, axis
    assert {(c.label, c.det) for c in CASES} >= {(r, d) for r in ("plain", "objective", "objective+void", "graphed")
                                                   for d in (False, True)}
    assert not any(c.void and c.general for c in CASES)          # refused: the general tail has no void form
    assert {c.label for c in CASES if c.shape == D} == {"objective+void", "graphed"}


def _assert_bit_identical(a, b, what=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _assert_bit_identical(a[k], b[k], f"{what}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for i, (u, v) in enumerate(zip(a, b)):
            _assert_bit_identical(u, v, f"{what}[{i}]")
    elif a is None or b is None:
        assert a is None and b is None, what
    else:
        assert not torch.isnan(a).any() and not torch.isnan(b).any(), f"NaN in {what}"
        assert torch.equal(a, b), what


@contextlib.contextmanager
def uninitialized_fill(monkeypatch):
    """torch.use_deterministic_algorithms(True) with torch's NaN / max-integer fill of torch.empty left on inside the
    autograd node too."""
    from osvos_pytorch_b200 import ops
    import torch.utils.deterministic as d
    with monkeypatch.context() as m:
        m.setattr(ops, "no_uninitialized_fill", contextlib.nullcontext)
        m.setattr(d, "fill_uninitialized_memory", True)
        with det_mode(True):
            yield


@pytest.mark.parametrize("case", [c for c in CASES if c.det], ids=str)
def test_route_writes_every_buffer_before_reading_it(case, monkeypatch):
    plain = run_case(case, check=False)
    with uninitialized_fill(monkeypatch):
        filled = run_case(case, check=False)
    _assert_bit_identical(plain, filled)


def _finetune(use_graph, fused):
    from osvos_pytorch_b200 import training
    case = Case("objective", True, False, "online", "none", A, seed=21)
    net = make_net(case)
    (x, gt), = samples(case, 0)
    hist = training.online_finetune(net, lambda it: {"image": x, "gt": gt}, 10, n_ave_grad=5, lr=1e-6, log_every=1,
                                    log=lambda s: None, use_graph=use_graph, fused_optimizer=fused)
    torch.cuda.synchronize()
    return {"hist": [torch.tensor(hist)], "params": {n: p.detach().clone() for n, p in net.named_parameters()}}


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("fused", [True, False])
def test_online_finetune_writes_every_buffer_before_reading_it(use_graph, fused, monkeypatch):
    with det_mode(True):
        plain = _finetune(use_graph, fused)
    with uninitialized_fill(monkeypatch):
        filled = _finetune(use_graph, fused)
    _assert_bit_identical(plain, filled)
    init = make_net(Case("objective", True, False, "online", "none", A, seed=21))
    assert not torch.equal(plain["params"]["stages.2.1.weight"], init.stages[2][1].weight.detach())  # it trained


def _parent(fused):
    from osvos_pytorch_b200 import training
    from osvos_pytorch_b200.parallel import GradientBucket, trainable_parameters
    case = Case("objective", True, False, "parent", "bucket", B, void=True, seed=22)
    net = make_net(case)
    opt = training.make_optimizer(net, "parent", lr=1e-6, fused=fused)
    bucket = GradientBucket(trainable_parameters(net))
    batches = [{"image": x, "gt": gt} for w in range(2) for x, gt in samples(case, w)]
    totals = training.parent_epoch(net, opt, bucket, batches, 84, 240, n_ave_grad=2, void=True)
    torch.cuda.synchronize()
    return {"totals": totals.clone(), "params": {n: p.detach().clone() for n, p in net.named_parameters()}}


@pytest.mark.parametrize("fused", [True, False])
def test_parent_epoch_writes_every_buffer_before_reading_it(fused, monkeypatch):
    with det_mode(True):
        plain = _parent(fused)
    with uninitialized_fill(monkeypatch):
        filled = _parent(fused)
    _assert_bit_identical(plain, filled)


@pytest.mark.parametrize("general", [False, True])
def test_checker_fails_on_a_one_percent_error_and_on_a_missing_gradient(general):
    assert 0.01 >= 20 * GATED_TOL and 0.01 >= 5 * SUM_TOL
    case = Case("plain", False, general, "mixed", "none", A, seed=23)
    net = make_net(case)
    (x, gt), = samples(case, 0)
    params64 = {k: v.detach().double() for k, v in net.state_dict().items()}
    ref = reference_step(params64, x.double(), gt.double(), WEIGHTS["mixed"], gates=gates_of(capture(net, x)),
                         general=general, learn_upsampling=general)["grads"]
    names = [n for n, _ in trainable(net)]
    got = {n: ref[n].clone() if n in ref else None for n in names}
    assert check_gradients(got, ref)[0] == 0.0
    for n in ref:
        scaled = dict(got, **{n: 1.01 * ref[n]})
        with pytest.raises(AssertionError):
            check_gradients(scaled, ref)
        with pytest.raises(AssertionError):
            check_gradients(dict(got, **{n: None}), ref)
    extra = next(n for n in names if n not in ref)                      # score_dsn or an upscale_ at weight 0
    with pytest.raises(AssertionError):
        check_gradients(dict(got, **{extra: torch.zeros(1)}), ref)

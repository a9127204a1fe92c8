"""Online adaptation on the GPU (csrc/adapt.cu, training.OnlineAdaptation, SequenceSegmenter(adapt=...), DESIGN.md §28):
the targets kernel against the numpy / scipy restatement (tests/adaptation_ref.py, pinned in test_adaptation.py) bit for
bit, and the adapted test loop against a restatement built from eager public calls."""
import gc
import json
import os
import random

import numpy as np
import pytest
import torch
from scipy import ndimage

import adaptation_ref as ref
import davis_fixture

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def release_graphs():
    """Each test's networks and their engines reference each other, and they and the adaptation own captured CUDA
    graphs: free them when the test ends, not in a collection inside a later test (or a later file's capture)."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def _mask(rng, h, w, kind):
    if kind == "empty":
        return np.zeros((h, w), np.uint8)
    if kind == "full":
        return np.full((h, w), 255, np.uint8)
    if kind == "border":                                # blobs cut by all four edges
        m = np.zeros((h, w), np.uint8)
        m[:max(1, h // 3), :max(1, w // 2)] = 255
        m[h - max(1, h // 4):, w // 3:] = 1
        m[h // 3:2 * h // 3 + 1, :max(1, w // 5)] = 7
        m[:, w - max(1, w // 6):] = 200
        return m
    blur = max(1.0, min(h, w) / 12)                     # random blobs
    return (ndimage.gaussian_filter(rng.random((h, w)), blur) > 0.5).astype(np.uint8) * 255


def _logits(rng, h, w, alpha):
    x = (rng.standard_normal((h, w)) * 4).astype(np.float32)
    x[rng.random((h, w)) < 0.1] = ref.threshold(alpha)   # exactly on the threshold: not positive
    return x


def _check(logits, masks, alpha, e, d):
    from osvos_pytorch_b200 import ops
    lt, mt = torch.from_numpy(logits).cuda(), torch.from_numpy(masks).cuda()
    labels, counts = ops.adaptation_labels(lt, mt, alpha, e, d)
    want_l, want_c = ref.adaptation_labels(logits, masks, alpha, e, d)
    np.testing.assert_array_equal(counts.cpu().numpy(), want_c)
    assert np.array_equal(labels.cpu().numpy(), want_l)
    return want_c


PARAMS = [(0.97, 15, 220), (0.5, 0, 0), (0.9, 3, 40), (0.99, 1, 5000), (0.7, 40, 12)]


@pytest.mark.parametrize("shape", [(1, 1), (7, 5), (33, 45), (480, 854), (1080, 1920), (5, 13000)])
@pytest.mark.parametrize("kind", ["blobs", "empty", "full", "border"])
def test_labels_match_restatement(shape, kind):
    h, w = shape
    rng = np.random.default_rng(h * 7 + w + len(kind))
    for i, (alpha, e, d) in enumerate(PARAMS if h * w < 10 ** 5 else PARAMS[:2]):
        masks = _mask(rng, h, w, kind)[None]
        _check(_logits(rng, h, w, alpha)[None, None], masks, alpha, e, d)


@pytest.mark.parametrize("alpha,e,d", PARAMS)
def test_batch_of_different_masks(alpha, e, d):
    rng = np.random.default_rng(17)
    h, w = 61, 83
    masks = np.stack([_mask(rng, h, w, k) for k in ("blobs", "border", "empty")])
    logits = np.stack([_logits(rng, h, w, alpha) for _ in range(3)])[:, None]
    c = _check(logits, masks, alpha, e, d)
    assert c[2].tolist()[0] == 0 and c[2, 2] == 0          # the empty mask: E empty, no negatives


def test_blob_erosion_and_distance_are_not_trivial():
    """A 480x854 blob under the defaults: E is a strict non-empty subset of M and both labels occur."""
    rng = np.random.default_rng(5)
    m = np.zeros((480, 854), np.uint8)
    m[150:330, 300:560] = 255
    c = _check(_logits(rng, 480, 854, 0.97)[None, None], m[None], 0.97, 15, 220)
    assert 0 < c[0, 0] < (m != 0).sum() and c[0, 1] > 0 and c[0, 2] > 0


def test_misaligned_mask_gives_the_same_result():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(9)
    h, w = 47, 61
    mask = torch.from_numpy(_mask(rng, h, w, "blobs")[None]).cuda()
    logits = torch.from_numpy(_logits(rng, h, w, 0.9)[None, None]).cuda()
    want = ops.adaptation_labels(logits, mask, 0.9, 2, 9)
    for off in (1, 2, 3):
        buf = torch.zeros(mask.numel() + 8, dtype=torch.uint8, device="cuda")
        shifted = buf[off:off + mask.numel()].view(mask.shape)
        shifted.copy_(mask)
        got = ops.adaptation_labels(logits, shifted, 0.9, 2, 9)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_out_receives_the_labels():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(2)
    mask = torch.from_numpy(_mask(rng, 20, 30, "blobs")[None]).cuda()
    logits = torch.from_numpy(_logits(rng, 20, 30, 0.97)[None, None]).cuda()
    out = torch.full((1, 1, 20, 30), 5.0, device="cuda")
    labels, _ = ops.adaptation_labels(logits, mask, 0.97, 1, 4, out=out)
    assert labels is out and torch.equal(out, ops.adaptation_labels(logits, mask, 0.97, 1, 4)[0])


def test_invalid_arguments_raise_before_any_launch():
    from osvos_pytorch_b200 import ops
    logits = torch.zeros(1, 1, 8, 9, device="cuda")
    mask = torch.zeros(1, 8, 9, dtype=torch.uint8, device="cuda")
    bad = [
        (logits, mask, 0.0, 1, 1), (logits, mask, 1.0, 1, 1), (logits, mask, 1.5, 1, 1), (logits, mask, True, 1, 1),
        (logits, mask, float("nan"), 1, 1), (logits, mask, 0.9, -1, 1), (logits, mask, 0.9, 1.5, 1),
        (logits, mask, 0.9, True, 1), (logits, mask, 0.9, 1, -3), (logits, mask, 0.9, 1, 2.0),
        (logits[:, 0], mask, 0.9, 1, 1), (logits.half(), mask, 0.9, 1, 1), (logits, mask.float(), 0.9, 1, 1),
        (logits, mask[:, :, :8], 0.9, 1, 1), (torch.zeros(2, 1, 8, 9, device="cuda"), mask, 0.9, 1, 1),
    ]
    before = ops.KERNEL_LAUNCHES[0]
    for args in bad:
        with pytest.raises(ValueError):
            ops.adaptation_labels(*args)
    with pytest.raises(ValueError, match="out"):
        ops.adaptation_labels(logits, mask, 0.9, 1, 1, out=torch.zeros(1, 8, 9, device="cuda"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.adaptation_labels(logits.cpu(), mask, 0.9, 1, 1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.adaptation_labels(logits, mask.cpu(), 0.9, 1, 1)
    torch.cuda.synchronize()
    assert ops.KERNEL_LAUNCHES[0] == before


# ---- the adapted test loop ------------------------------------------------------------------------------------------

def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


def _sequence(tree):
    """Five collated 33x45 frames: sequence aa's three and two of them flipped."""
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True, seq_name=None)
    items = [d[i] for i in range(3)]
    for it in items[:2]:
        items.append(dict(it, image=np.ascontiguousarray(it["image"][:, ::-1]), gt=np.ascontiguousarray(it["gt"][:, ::-1])))
    return [davis.collate([it]) for it in items]


def _frames(batches):
    from osvos_pytorch_b200 import davis
    for b in batches:
        img, _ = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
        yield img


def _sampler(batches, seed):
    """The fine-tuning's sampler over the annotated frame, on its own generator."""
    from osvos_pytorch_b200 import augment, davis
    img_u8, gt_u8, stats = davis.upload(batches[0], torch.device("cuda"))
    rng = random.Random(seed)

    def sample_fn(it):
        return augment.affine_warp_u8(img_u8, gt_u8, augment.draw_params(1, rng=rng), stats)
    return sample_fn, gt_u8


OPTS = dict(steps=4, current_steps=2, weight=0.5, alpha=0.9, distance=10, erosion=1)
LR, WD = 1e-10, 0.0002


def _adapted_run(net, batches, first_mask, sample_fn, **kw):
    from osvos_pytorch_b200 import training
    from osvos_pytorch_b200.inference import SequenceSegmenter
    adapt = training.OnlineAdaptation(net, sample_fn, first_mask, LR, WD, **dict(OPTS, **kw))
    seg = SequenceSegmenter(net, output="bytescale", depth=2, frames="bgr8", adapt=adapt)
    return [r.clone() for r in seg(_frames(batches))], adapt


def _restated(net, batches, first_mask, sample_fn, steps, current_steps, weight, alpha, distance, erosion):
    """The adapted loop from eager public calls: forward_inference, adaptation_labels, forward_objective + backward,
    FusedSGD.step and logits_to_u8."""
    from osvos_pytorch_b200 import davis, ops, parallel, training
    dev = torch.device("cuda")
    eng = net._engine
    opt = training.make_optimizer(net, "online", LR, WD, fused=True)
    opt.zero_grad()
    in_opt = {id(p) for g in opt.param_groups for p in g["params"]}
    params = parallel.trainable_parameters(net)
    for p in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
    current_at = {i * steps // current_steps for i in range(current_steps)}
    last, results, counts, draws = first_mask.clone(), [], [], 0
    for i, b in enumerate(batches):
        x = davis.to_device(b, dev)["image"]
        if i > 0:
            labels, c = ops.adaptation_labels(eng.forward_inference(x)[-1], last, alpha, erosion, distance)
            counts.append(c[0].cpu())
            if int(c[0, 0]) > 0:
                for s in range(steps):
                    if s in current_at:
                        xs, gts, w, void = x, labels, (0.0, 0.0, 0.0, 0.0, weight), True
                    else:
                        smp = sample_fn(draws)
                        draws += 1
                        xs, gts, w, void = smp["image"], smp["gt"], training.ONLINE_WEIGHTS, False
                    _, total, _ = net.forward_objective(xs, gts, w, void=void)
                    with eng.direct_grad_accumulation():
                        total.backward()
                    opt.step(zero_grad=True)
                    for p in params:
                        if id(p) not in in_opt:
                            p.grad.zero_()
        fused = eng.forward_inference(x)[-1]
        if i > 0:
            last = ops.logits_to_u8(fused, "mask")[:, 0].contiguous()
        results.append(ops.logits_to_u8(fused, "bytescale").cpu())
    return results, counts


@pytest.fixture
def deterministic():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def test_adapted_loop_matches_eager_restatement(tree, deterministic):
    batches = _sequence(tree)
    net_a, net_b = _he_net(seed=4).cuda(), _he_net(seed=4).cuda()
    init = {k: v.clone() for k, v in net_a.state_dict().items()}
    fn_a, first = _sampler(batches, 7)
    fn_b, _ = _sampler(batches, 7)
    got, adapt = _adapted_run(net_a, batches, first, fn_a)
    want, want_counts = _restated(net_b, batches, first, fn_b, **OPTS)
    assert len(got) == 5 and all(torch.equal(a, b) for a, b in zip(got, want))
    assert len(adapt.counts) == 4 and all(torch.equal(a, b) for a, b in zip(adapt.counts, want_counts))
    assert any(int(c[0]) > 0 for c in adapt.counts) and adapt.skipped == sum(int(c[0]) == 0 for c in adapt.counts)
    assert net_a._engine._graphs == {}                  # every forward of the adapted run was eager
    sa, sb = net_a.state_dict(), net_b.state_dict()
    assert all(torch.equal(sa[k], sb[k]) for k in sa)
    assert any(not torch.equal(sa[k], init[k]) for k in sa)


def test_zero_steps_is_the_eager_segmenter(tree, monkeypatch):
    from osvos_pytorch_b200.inference import SequenceSegmenter
    batches = _sequence(tree)
    fn, first = _sampler(batches, 1)
    net = _he_net(seed=6).cuda().eval()
    init = {k: v.clone() for k, v in net.state_dict().items()}
    got, adapt = _adapted_run(net, batches, first, fn, steps=0, current_steps=0)
    assert len(adapt.counts) == 4 and net._engine._graphs == {}
    assert adapt._first is None and adapt._current is None      # no step taken: no training graph captured
    assert all(torch.equal(v, init[k]) for k, v in net.state_dict().items())
    monkeypatch.setenv("OSVOS_CUDA_GRAPH", "0")
    plain = _he_net(seed=6).cuda().eval()
    want = [r.clone() for r in SequenceSegmenter(plain, output="bytescale", depth=2, frames="bgr8")(_frames(batches))]
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_mask_eroded_to_nothing_takes_no_step(tree):
    batches = _sequence(tree)[:2]                       # frame 1 is the only adapted frame; its last mask is `first`
    fn, first = _sampler(batches, 3)
    first = torch.zeros_like(first)
    first[0, 10:13, 20:23] = 255                        # a 3x3 square: gone under erosion 2
    net = _he_net(seed=8).cuda()
    init = {k: v.clone() for k, v in net.state_dict().items()}
    _, adapt = _adapted_run(net, batches, first, fn, erosion=2)
    assert adapt.skipped == 1 and int(adapt.counts[0][0]) == 0
    assert adapt._first is None and adapt._current is None
    assert all(torch.equal(v, init[k]) for k, v in net.state_dict().items())


def test_segmenter_refuses_adapt_combinations(tree):
    from osvos_pytorch_b200 import training
    from osvos_pytorch_b200.inference import SequenceSegmenter
    batches = _sequence(tree)
    fn, first = _sampler(batches, 0)
    net = _he_net().cuda()
    adapt = training.OnlineAdaptation(net, fn, first, LR, WD, **OPTS)
    for kw in (dict(nets=[net]), dict(net=net, output="labels"), dict(net=net, output="bytescale"),
               dict(net=_he_net().cuda(), output="bytescale", frames="bgr8")):
        with pytest.raises(ValueError, match="adapt"):
            SequenceSegmenter(adapt=adapt, **kw)
    seg = SequenceSegmenter(net, output="bytescale", frames="bgr8", adapt=adapt)
    two = (torch.cat([f, f]) for f in _frames(batches))
    with pytest.raises(ValueError, match="adapt"):
        list(seg(two))
    with pytest.raises(ValueError, match="current_steps"):
        training.OnlineAdaptation(net, fn, first, LR, WD, steps=2, current_steps=3)


def _online(tree, save, monkeypatch, extra):
    import train_online
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    try:
        return train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed",
                                  "1", "--parent-epoch", "1", "--log-every", "1", "--no-save", "--loader", "native",
                                  "--adapt", "--adapt-steps", "3", "--adapt-current-steps", "1", "--adapt-erosion",
                                  "2", "--adapt-distance", "30"] + extra)
    finally:
        gc.collect()                                    # the run's network, engine and graphs


def _outputs(save):
    root = save / "Results"
    return {os.path.join(dp, f): open(os.path.join(dp, f), "rb").read()
            for dp, _, fs in os.walk(root) for f in fs}


@pytest.mark.parametrize("extra", [[], ["--input-res", "40", "56", "--output-res", "stored", "--encode", "device",
                                        "--evaluate"]])
def test_train_online_adapt(tree, tmp_path, monkeypatch, capsys, extra):
    from PIL import Image
    save = tmp_path / "models"
    save.mkdir()
    torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
    hist = _online(tree, save, monkeypatch, extra)
    assert len(hist) == 4 and all(np.isfinite(hist))
    pngs = sorted(os.listdir(save / "Results" / "cc"))
    assert pngs == ["00000.png", "00001.png"]
    assert np.asarray(Image.open(save / "Results" / "cc" / pngs[1])).shape == (97, 131)
    assert "Online adaptation time" in capsys.readouterr().out
    if "--evaluate" in extra:
        with open(save / "Results" / "cc_scores.json") as f:
            res = json.load(f)
        ad = res["adaptation"]
        assert (ad["steps"], ad["current_steps"], ad["erosion"], ad["distance"]) == (3, 1, 2, 30)
        assert len(ad["counts"]) == 1 and len(ad["counts"][0]) == 3


def test_train_online_adapt_deterministic_runs_are_identical(tree, tmp_path, monkeypatch):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    runs = []
    try:
        for r in range(2):
            save = tmp_path / f"run{r}"
            save.mkdir()
            torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
            _online(tree, save, monkeypatch, ["--deterministic", "--evaluate", "--overlay"])
            runs.append({os.path.relpath(k, save): v for k, v in _outputs(save).items()})
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    assert len(runs[0]) == 5 and runs[0] == runs[1]     # 2 PNGs, 2 overlays, the scores

"""Void labels on the GPU (DESIGN.md §26): the void forms of the class-balanced BCE kernels against the fp64
restatement (void_loss_ref), their identity with the plain forms on labels without void, the whole network's void
objective against the plain route, the id ingest and id-mode warp against the two-mask composition of the existing
kernels, and train_parent.py --davis 2017 / train_online.py --ignore-void on a synthetic DAVIS-2017 tree."""
import gc
import os
import re

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import osvos_oracle as oc
import void_loss_ref as V

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _labels(g, shape, p_void, p_pos=0.3):
    u = torch.rand(shape, generator=g)
    return torch.where(u < p_void, -1.0, torch.where(u < p_void + p_pos, 1.0, 0.0))


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------- standalone loss (osvos_cbce_fwd / _bwd_void)
def _cbce(x, y, det, void, divisor=2.0):
    from osvos_pytorch_b200 import _native as nat
    lib = nat.load()
    flags = (nat.FLAG_DETERMINISTIC if det else 0) | (nat.FLAG_VOID_LABELS if void else 0)
    sums = torch.empty(lib.osvos_cbce_fwd_sums(x.numel(), flags), dtype=torch.float64, device=x.device)
    loss = torch.empty((), dtype=torch.float32, device=x.device)
    s = torch.cuda.current_stream().cuda_stream
    nat.check(lib.osvos_cbce_fwd(x.data_ptr(), y.data_ptr(), x.numel(), divisor, sums.data_ptr(), loss.data_ptr(),
                                 flags, s), "osvos_cbce_fwd")
    dx = torch.empty_like(x)
    bwd = lib.osvos_cbce_bwd_void if void else lib.osvos_cbce_bwd
    nat.check(bwd(x.data_ptr(), y.data_ptr(), sums.data_ptr(), None, divisor, x.numel(), dx.data_ptr(), s), "bwd")
    return loss, dx, sums


def _loss_shapes():
    """numel in each regime of loss_grid: one block with a numel % 4 tail, several blocks, the capped grid."""
    cap = _sm_count() * 8
    return [7, 4 * 256 * 3 + 2, 4 * 256 * cap * 2 + 3]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("p_void", [0.0, 0.25, 1.0])
def test_cbce_void_vs_fp64(dev, det, p_void):
    g = torch.Generator().manual_seed(11)
    for numel in _loss_shapes():
        x = torch.randn(numel, generator=g) * 4
        y = _labels(g, (numel,), p_void)
        loss, dx, _ = _cbce(x.to(dev), y.to(dev), det, True)
        want, gwant = V.void_loss(x.numpy(), y.numpy(), 2.0)
        # fp32 per-pixel terms summed in fp32 per thread, fp64 across blocks: bound steps * 2^-23 * sum|terms|
        sp = np.maximum(x.numpy(), 0) + np.log1p(np.exp(-np.abs(x.numpy())))
        bound = 4e-7 * (numel / (256 * 4) + 64) * float(sp.sum()) / 2.0 + 1e-30
        assert abs(float(loss) - want) <= bound, (numel, float(loss), want)
        gd = dx.cpu().double().numpy()
        assert np.all(gd[y.numpy() < 0] == 0)
        assert np.abs(gd - gwant).max() <= 1e-6 * max(np.abs(gwant).max(), 1e-30), numel
        if det:
            loss2, dx2, _ = _cbce(x.to(dev), y.to(dev), det, True)
            assert torch.equal(loss, loss2) and torch.equal(dx, dx2)


@pytest.mark.parametrize("det", [False, True])
def test_cbce_void_without_void_is_the_plain_loss(dev, det):
    g = torch.Generator().manual_seed(12)
    for numel in _loss_shapes():
        x = (torch.randn(numel, generator=g) * 4).to(dev)
        y = _labels(g, (numel,), 0.0).to(dev)
        l0, d0, s0 = _cbce(x, y, det, False)
        l1, d1, s1 = _cbce(x, y, det, True)
        assert torch.equal(d0, d1) and torch.equal(s0[2:4], s1[2:4])       # P and N: exact counts
        if det:
            assert torch.equal(l0, l1) and torch.equal(s0[:2], s1[:2])
        else:
            assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l0))


# ---------------------------------------------------------------- tail forward + fused backward, void forms
def _random_pqs(n, h, w, g, scale=5.0):
    pqs, hk, wk = [], h, w
    for _ in range(4):
        hk, wk = oc.pooled_size(hk), oc.pooled_size(wk)
        pqs.append(torch.randn(n, hk, wk, 2, generator=g) * scale)
    return pqs


def _tail_shapes():
    """The tail backward's regimes need width: one narrow, one odd, one with several row groups and a multi-block
    forward, one wave past the SM count (the forward's row striding)."""
    rows = _sm_count() * 8 + 5
    return [(1, 17, 3), (2, 33, 45), (3, 64, 96), (1, rows, 70), (2, 480, 854)]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("p_void", [0.0, 0.3, 1.0])
def test_tail_void_vs_fp64(dev, det, p_void):
    from osvos_pytorch_b200 import ops
    weights = (0.5, 0.0, 2.0, 0.25, 1.0)
    g = torch.Generator().manual_seed(13)
    for n, h, w in _tail_shapes():
        pqs = [p.to(dev) for p in _random_pqs(n, h, w, g)]
        fb = torch.tensor([0.3], device=dev)
        y = _labels(g, (n, 1, h, w), p_void).to(dev)
        out, sums, losses = ops.tail_fwd(pqs, fb, n, h, w, label=y, loss_weights=weights, divisor=float(n),
                                         deterministic=det, void=True)
        maps = out.cpu().double().numpy()
        yn = y.cpu().numpy()
        grads = []
        for k in range(5):
            lk, gk = V.void_loss(maps[k], yn, float(n))
            sp = np.maximum(maps[k], 0) + np.log1p(np.exp(-np.abs(maps[k])))
            bound = 4e-7 * (h + 64) * float(sp.sum()) / n + 1e-30
            assert abs(float(losses[k]) - lk) <= bound, (n, h, w, k, float(losses[k]), lk)
            grads.append(torch.from_numpy(weights[k] * gk).float().to(dev))
        assert float(sums[11]) == float((y >= 0).sum())
        upstream = torch.tensor([1.5], device=dev)
        dpq, dfb = ops.tail_loss_bwd(out, y, sums, weights, float(n), upstream, n, h, w, deterministic=det, void=True)
        want = ops.tail_bwd([gk * 1.5 for gk in grads], n, h, w, deterministic=det)
        for k in range(4):
            scale = float(want[k].abs().max()) + 1e-30
            assert float((dpq[k] - want[k]).abs().max()) <= 2e-5 * scale, (n, h, w, k)
        fb_want = 1.5 * float(grads[4].double().sum())
        assert abs(float(dfb) - fb_want) <= 1e-5 * max(abs(fb_want), float(grads[4].abs().sum())) + 1e-30
        if det:
            out2, sums2, losses2 = ops.tail_fwd(pqs, fb, n, h, w, label=y, loss_weights=weights, divisor=float(n),
                                                deterministic=True, void=True)
            dpq2, dfb2 = ops.tail_loss_bwd(out2, y, sums2, weights, float(n), upstream, n, h, w, deterministic=True,
                                           void=True)
            assert torch.equal(losses, losses2) and torch.equal(dfb, dfb2)
            assert all(torch.equal(a, b) for a, b in zip(dpq, dpq2))


# ---------------------------------------------------------------- whole network
@pytest.fixture(scope="module")
def net(dev):
    from osvos_pytorch_b200.networks import vgg_osvos as vo
    m = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(m, seed=0)
    return m.to(dev).train()


def _objective_grads(net, x, gt, weights, void):
    net.zero_grad(set_to_none=True)
    _, total, per_map = net.forward_objective(x, gt, weights, void=void)
    total.backward()
    return total.detach().clone(), per_map.detach().clone(), \
        {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("n,h,w", [(2, 64, 96), (12, 480, 854)])
def test_void_objective_is_bit_identical_without_void(net, dev, n, h, w):
    """Labels without void: void=True gives the same bits as void=False under deterministic algorithms, and agrees to
    the run-to-run bound without them."""
    x, gt = oc.synthetic_frame(n, h, w, 17)
    x, gt = x.to(dev), gt.to(dev)
    weights = (0.5, 0.5, 0.5, 0.5, 1.0)
    torch.use_deterministic_algorithms(True)
    try:
        t0, m0, g0 = _objective_grads(net, x, gt, weights, False)
        t1, m1, g1 = _objective_grads(net, x, gt, weights, True)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(t0, t1) and torch.equal(m0, m1)
    assert set(g0) == set(g1) and all(torch.equal(g0[k], g1[k]) for k in g0)
    t0, m0, g0 = _objective_grads(net, x, gt, weights, False)
    t1, m1, g1 = _objective_grads(net, x, gt, weights, True)
    assert abs(float(t0) - float(t1)) <= 1e-5 * abs(float(t0))
    for k in g0:
        err = float((g0[k].double() - g1[k].double()).norm() / g0[k].double().norm().clamp(min=1e-30))
        assert err < 2e-4, (k, err)
    del g0, g1
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("h,w", [(64, 96), (480, 854)])
@pytest.mark.parametrize("weights", [(0, 0, 0, 0, 1), (0.5, 0.5, 0.5, 0.5, 1)])
def test_void_objective_vs_plain_route(net, dev, weights, h, w):
    """forward_objective(void=True) against net(x) + the restated void loss per map through autograd, with a void band
    and with a frame that is void only; at 480x854 the tail backward runs its wide, multi-segment rows."""
    n = 3
    x, gt = oc.synthetic_frame(n, h, w, 23)
    x, gt = x.to(dev), gt.to(dev).clone()
    gt[0, :, h // 6:h // 3, :] = -1                  # a void band
    gt[2] = -1                                       # a void-only frame
    net.zero_grad(set_to_none=True)
    outs = net(x)
    losses = [V.void_loss_torch(o, gt, float(n)) for o in outs]
    total = sum(wk * l for wk, l in zip(weights, losses) if wk != 0)
    total.backward()
    ref = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
    tot2, per_map, got = _objective_grads(net, x, gt, weights, True)
    assert abs(float(tot2) - float(total)) <= 1e-5 * abs(float(total))
    for k in range(5):
        assert abs(float(per_map[k]) - float(losses[k])) <= 1e-5 * abs(float(losses[k])) + 1e-30
    assert set(got) == set(ref)
    for k in ref:
        err = float((got[k].double() - ref[k].double()).norm() / ref[k].double().norm().clamp(min=1e-30))
        assert err < 2e-4, (k, err)


def test_void_objective_refusals(net, dev):
    x = torch.zeros(1, 3, 32, 32, device=dev)
    gt = torch.zeros(1, 1, 32, 32, device=dev)
    with pytest.raises(ValueError, match="size_average"):
        net.forward_objective(x, gt, (0, 0, 0, 0, 1), size_average=True, void=True)
    from osvos_pytorch_b200.networks import vgg_osvos as vo
    m = vo.OSVOS(pretrained=0, verbose=False, learn_upsampling=True).to(dev)
    with pytest.raises(ValueError, match="general tail"):
        m.forward_objective(x, gt, (0, 0, 0, 0, 1), void=True)


# ---------------------------------------------------------------- id ingest and id-mode warp
def _ids(g, n, h, w):
    ids = torch.randint(0, 5, (n, h, w), generator=g, dtype=torch.uint8)
    ids[torch.rand(n, h, w, generator=g) < 0.1] = 255
    ids[:, :, : max(1, w // 10)] = 255               # a void band
    return ids


@pytest.mark.parametrize("n,h,w", [(1, 480, 854), (12, 480, 854), (3, 37, 61), (1, 1, 5)])
def test_labels_from_ids(dev, n, h, w):
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(n * 1000 + h)
    ids = _ids(g, n, h, w)
    for obj in (None, "all", 3):
        got = ops.labels_from_ids(ids.to(dev), obj).cpu().numpy()
        want = V.labels_of_ids(ids.numpy(), None if obj == "all" else obj)[:, None]
        assert np.array_equal(got, want)


@pytest.mark.parametrize("n,h,w", [(1, 480, 854), (12, 480, 854), (3, 37, 61), (33, 21, 13)])
@pytest.mark.parametrize("indexed", [False, True])
def test_id_warp_equals_two_mask_composition(dev, n, h, w, indexed):
    """The id mode of the fused warp equals, bit for bit, the existing warp's label of the 0/255 object mask, set to -1
    where the existing warp of the 0/255 void mask is 1; the image half is the existing warp's.  Also held to the host
    restatement (void_loss_ref.warp_ids) at the first sample."""
    import random
    from osvos_pytorch_b200 import augment, ops
    g = torch.Generator().manual_seed(n + h)
    store = _ids(g, n + 2, h, w).to(dev)
    img = torch.randint(0, 256, (n + 2, h, w, 3), generator=g, dtype=torch.uint8).to(dev)
    params = augment.draw_params(n, rng=random.Random(n * 7 + w))
    index = [(5 * i + 1) % (n + 2) for i in range(n)] if indexed else None
    src_ids = store if indexed else store[:n]
    src_img = img if indexed else img[:n]
    void = torch.where(src_ids == 255, 255, 0).to(torch.uint8)
    for obj in (None, 2):
        fg = torch.where((src_ids >= 1) & (src_ids <= 254) if obj is None else src_ids == obj, 255, 0).to(torch.uint8)
        kw = {} if index is None else {"index": index}
        got = augment.affine_warp_u8(src_img, src_ids, params, ids="all" if obj is None else obj, **kw)
        a = augment.affine_warp_u8(src_img, fg, params, ops.label_stats_u8(fg), **kw)
        b = augment.affine_warp_u8(src_img, void, params, ops.label_stats_u8(void), **kw)
        want = torch.where(b["gt"] == 1, torch.full_like(a["gt"], -1.0), a["gt"])
        assert torch.equal(got["gt"], want)
        assert torch.equal(got["image"], a["image"])
        i0 = index[0] if indexed else 0
        flip, rot, sc = params[0]
        host = V.warp_ids(src_ids[i0].cpu().numpy(), rot, sc, flip, obj)
        assert np.array_equal(got["gt"][0, 0].cpu().numpy(), host)


# ---------------------------------------------------------------- the scripts on a synthetic DAVIS-2017 tree
SEQS = {"train": {"t1": 2, "t2": 3}, "val": {"v1": 2, "v2": 1}}


def _scene(rng, h, w, k, void):
    yy, xx = np.mgrid[:h, :w]
    gt = np.zeros((h, w), np.uint8)
    for j in range(1, k + 1):
        cy, cx = rng.integers(0, h), rng.integers(0, w)
        ry, rx = rng.integers(3, h // 3), rng.integers(3, w // 3)
        gt[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1] = j
    if void:
        gt[h // 2:h // 2 + 4, :] = 255
    return gt


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """A DAVIS-2017 layout with train.txt and val.txt: JPEG frames (cv2), palette annotations (Pillow) with void bands
    in even frames."""
    cv2 = pytest.importorskip("cv2")
    from osvos_pytorch_b200.png import davis_palette
    root = tmp_path_factory.mktemp("davis2017_train")
    rng = np.random.default_rng(31)
    for split, seqs in SEQS.items():
        for seq, k in seqs.items():
            os.makedirs(root / "JPEGImages" / "480p" / seq)
            os.makedirs(root / "Annotations" / "480p" / seq)
            for f in range(4):
                cv2.imwrite(str(root / "JPEGImages" / "480p" / seq / f"{f:05d}.jpg"),
                            rng.integers(0, 256, (40, 56, 3), dtype=np.uint8))
                gt = _scene(rng, 40, 56, k, f % 2 == 0)    # void bands in the first annotation too
                gt[0, 0] = k
                im = Image.fromarray(gt, "P")
                im.putpalette(davis_palette(256))
                im.save(str(root / "Annotations" / "480p" / seq / f"{f:05d}.png"))
        os.makedirs(root / "ImageSets" / "2017", exist_ok=True)
        (root / "ImageSets" / "2017" / f"{split}.txt").write_text("\n".join(seqs) + "\n")
    return str(root)


def _run_parent(tmp_path, tree, monkeypatch, capsys, extra):
    import train_parent
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    torch.manual_seed(0)
    import random
    random.seed(0)
    try:
        train_parent.main(["--davis", "2017", "--loader", "native", "--epochs", "2", "--test-interval", "1",
                           "--snapshot", "1", "--pretrained", "0", "--lr", "1e-9", "--workers", "0", "--batch", "2",
                           "--n-ave-grad", "2"] + extra)
    finally:
        torch.use_deterministic_algorithms(False)
    gc.collect()
    return capsys.readouterr().out


def _union_scores(tree, net_state, dev):
    """Host restatement of --val-measures for 2017: the fused map > 0 against the union of the objects, void ignored
    (davis_objects_ref with one object), J and F per frame, each sequence's mean over its frames (davis_measures_ref),
    then the mean over sequences."""
    import davis_measures_ref as M
    import davis_objects_ref as O
    from osvos_pytorch_b200 import davis
    from osvos_pytorch_b200.networks import vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    net.load_state_dict(net_state)
    net.to(dev).eval()
    ds = davis.DAVIS2017Frames("val", tree)
    per_seq = {}
    for i in range(len(ds)):
        item = ds[i]
        x = davis.to_device(davis.collate([item]), dev, ids="all")["image"]
        with torch.no_grad():
            fused = net.forward(x)[-1][0, 0].cpu().numpy()
        ids = np.asarray(item["gt"])
        union = np.where(ids == 255, 255, (ids != 0).astype(np.uint8)).astype(np.uint8)
        c = O.object_counts((fused > 0).astype(np.uint8), union, 1, M.bound_pix(*ids.shape))[0]
        per_seq.setdefault(ds.seq_of[i], []).append(M.j_and_f(c))
    js = [M.statistics([v[0] for v in jf])[0] for jf in per_seq.values()]
    fs = [M.statistics([v[1] for v in jf])[0] for jf in per_seq.values()]
    return float(np.mean(js)), float(np.mean(fs))


def test_train_parent_2017(tmp_path, tree, monkeypatch, capsys, dev):
    out = _run_parent(tmp_path, tree, monkeypatch, capsys, ["--val-measures"])
    epochs = re.findall(r"\[Epoch: \d+\] (.*?)  Execution", out)
    assert len(epochs) == 2
    for line in epochs:
        vals = [float(v) for v in re.findall(r"Loss \d: (\S+)", line)]
        assert len(vals) == 5 and all(np.isfinite(vals))
    ckpt = tmp_path / "parent_epoch-1.pth"
    assert ckpt.exists()
    jf = re.findall(r"J M/O/D: (\S+) / \S+ / \S+  F M/O/D: (\S+) /", out)
    assert len(jf) == 2
    j, f = _union_scores(tree, torch.load(ckpt, map_location="cpu"), dev)
    assert abs(float(jf[-1][0]) - j) <= 1e-4 and abs(float(jf[-1][1]) - f) <= 1e-4, (jf[-1], j, f)


def test_train_parent_2017_deterministic_cache_equals_streaming(tmp_path, tree, monkeypatch, capsys):
    runs = []
    for extra in ([], ["--cache", "device"]):
        d = tmp_path / ("cache" if extra else "stream")
        d.mkdir()
        out = _run_parent(d, tree, monkeypatch, capsys, ["--deterministic"] + extra)
        runs.append(re.findall(r"\[Epoch: \d+\] (.*?)  Execution", out) + re.findall(r"\*\*\*Testing \*\*\* (.*)", out))
    assert len(runs[0]) == 4 and runs[0] == runs[1]


def _recording_finetune(monkeypatch):
    """Wraps training.online_finetune: records, per call, its ``void`` argument and the smallest label it trained on."""
    from osvos_pytorch_b200 import training
    calls, real = [], training.online_finetune

    def finetune(net, sample_fn, *args, **kw):
        seen = []

        def recorded(it):
            s = sample_fn(it)
            seen.append(float(s["gt"].min()))
            return s
        out = real(net, recorded, *args, **kw)
        calls.append((kw.get("void", False), min(seen)))
        return out
    monkeypatch.setattr(training, "online_finetune", finetune)
    return calls


def test_train_online_2017_ignore_void(tmp_path, tree, monkeypatch):
    """With --ignore-void each object trains on labels with void (-1) pixels through the void objective; without it
    on 0 / 1 labels as before.  Both write the same set of files."""
    import train_online
    from osvos_pytorch_b200.networks import vgg_osvos as vo
    m = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(m, seed=3)
    torch.save(m.state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    calls = _recording_finetune(monkeypatch)
    files = {}
    for flag in ([], ["--ignore-void"]):
        d = tmp_path / ("void" if flag else "plain")
        d.mkdir()
        torch.save(m.state_dict(), d / "parent_epoch-0.pth")
        monkeypatch.setenv("OSVOS_SAVE_ROOT", str(d))
        train_online.main(["--seq-name", "v1", "--iters", "10", "--n-ave-grad", "5", "--lr", "1e-10", "--seed", "1",
                           "--parent-epoch", "1", "--loader", "native", "--davis", "2017", "--evaluate"] + flag)
        gc.collect()
        files[bool(flag)] = sorted(str(p.relative_to(d)) for p in d.rglob("*") if p.is_file())
    assert files[True] == files[False] and "Results/v1/00000.png" in files[True]
    k = SEQS["val"]["v1"]
    assert calls == [(False, 0.0)] * k + [(True, -1.0)] * k, calls


def test_train_online_ignore_void_refuses_a_general_tail_parent(tmp_path, tree, monkeypatch):
    """A parent whose deconvolution weights are not the bilinear taps is refused before any fine-tune starts."""
    import train_online
    from osvos_pytorch_b200.networks import vgg_osvos as vo
    m = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(m, seed=3)
    with torch.no_grad():
        m.upscale[0].weight.mul_(1.5)
    torch.save(m.state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    calls = _recording_finetune(monkeypatch)
    with pytest.raises(SystemExit, match="bilinear taps"):
        train_online.main(["--seq-name", "v1", "--iters", "10", "--n-ave-grad", "5", "--lr", "1e-10",
                           "--parent-epoch", "1", "--loader", "native", "--davis", "2017", "--ignore-void"])
    assert calls == []

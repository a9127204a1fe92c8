"""ops.connected_components and ops.filter_components (csrc/components.cu, DESIGN.md §30) bit for bit against scipy and
the restatement tests/components_ref.py, and the filter in SequenceSegmenter and train_online.py."""
import ctypes
import gc
import json
import os
import random

import numpy as np
import pytest
import torch

import components_ref as ref
import davis_fixture

pytestmark = pytest.mark.gpu

TILE_H, TILE_W = 16, 32


@pytest.fixture(autouse=True)
def release_graphs():
    yield
    gc.collect()
    torch.cuda.empty_cache()


# ---- masks ----------------------------------------------------------------------------------------------------------

def _serpentine(h, w):
    """One 1-pixel-wide path through every row pair: full rows joined alternately at the right and the left end."""
    m = np.zeros((h, w), np.uint8)
    m[0::2] = 1
    for y in range(1, h, 2):
        m[y, w - 1 if (y // 2) % 2 == 0 else 0] = 1
    return m


def _blobs(rng, h, w, count, on_borders=False):
    m = np.zeros((h, w), np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    for _ in range(count):
        if on_borders:                                  # centred on tile borders and on the frame's edges
            cy = int(rng.integers(0, h // TILE_H + 1)) * TILE_H
            cx = int(rng.integers(0, w // TILE_W + 1)) * TILE_W
        else:
            cy, cx = int(rng.integers(0, h)), int(rng.integers(0, w))
        r = float(rng.uniform(0.5, max(1.0, min(h, w) / 6)))
        m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 1
    return m


def _masks(seed, h, w):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    kinds = {
        "empty": np.zeros((h, w), np.uint8),
        "full": np.full((h, w), 7, np.uint8),
        "checkerboard": ((yy + xx) % 2).astype(np.uint8),
        "serpentine": _serpentine(h, w),
        "random0.3": (rng.random((h, w)) < 0.3).astype(np.uint8) * 255,
        "random0.5": (rng.random((h, w)) < 0.5).astype(np.uint8),
        "random0.59": (rng.random((h, w)) < 0.59).astype(np.uint8),
        "blobs": _blobs(rng, h, w, 12),
        "blobs_on_borders": _blobs(rng, h, w, 12, on_borders=True),
    }
    return list(kinds), np.stack(list(kinds.values()))


SHAPES = [(1, 1), (7, 5), (33, 45), (480, 854), (1080, 1920), (5, 13000), (13000, 5),
          (TILE_H, TILE_W), (TILE_H + 1, TILE_W + 1), (TILE_H - 1, TILE_W - 1), (TILE_H, 3 * TILE_W + 1),
          (2 * TILE_H - 1, TILE_W)]


@pytest.mark.parametrize("connectivity", [4, 8])
@pytest.mark.parametrize("hw", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_labels_equal_scipy(hw, connectivity):
    from osvos_pytorch_b200 import ops
    names, masks = _masks(hash(hw) % 1000, *hw)
    labels, counts = ops.connected_components(torch.from_numpy(masks).cuda(), connectivity)
    labels, counts = labels.cpu().numpy(), counts.cpu().numpy()
    for f, name in enumerate(names):
        want, n = ref.label(masks[f], connectivity)
        assert counts[f] == n, name
        assert np.array_equal(labels[f], want), name


def test_n_frames_in_one_call_equal_one_frame_calls_and_misaligned_masks():
    from osvos_pytorch_b200 import ops
    _, masks = _masks(5, 70, 100)
    x = torch.from_numpy(masks).cuda()
    for c in (4, 8):
        lab, cnt = ops.connected_components(x, c)
        for f in range(x.shape[0]):
            l1, c1 = ops.connected_components(x[f:f + 1].clone(), c)
            assert torch.equal(lab[f:f + 1], l1) and torch.equal(cnt[f:f + 1], c1)
        buf = torch.empty(x.numel() + 1, dtype=torch.uint8, device="cuda")
        view = buf[1:].view(x.shape)
        view.copy_(x)
        assert view.data_ptr() % 2 == 1
        l2, c2 = ops.connected_components(view, c)
        assert torch.equal(lab, l2) and torch.equal(cnt, c2)


# ---- the filter -----------------------------------------------------------------------------------------------------

def _maps(seed, k, n, h, w):
    """Logits whose foreground is blobs (a few large, many small), with NaN and ±0 sprinkled over both sides."""
    rng = np.random.default_rng(seed)
    z = np.empty((k, n, h, w), np.float32)
    for o in range(k):
        for j in range(n):
            fg = _blobs(rng, h, w, 3 + int(rng.integers(0, 8))) | (rng.random((h, w)) < 0.004)
            z[o, j] = np.where(fg > 0, rng.uniform(0.01, 8, (h, w)), -rng.uniform(0, 8, (h, w)))
            for v in (np.nan, 0.0, -0.0):
                z[o, j][rng.random((h, w)) < 0.003] = v
    return z


def _prior(seed, k, h, w):
    rng = np.random.default_rng(seed + 50)
    return np.stack([_blobs(rng, h, w, 2) for _ in range(k)])


def _filter(z, params, prior=None, **kw):
    from osvos_pytorch_b200 import ops
    maps = [torch.from_numpy(m).cuda().unsqueeze(1) for m in z]
    p = None if prior is None else torch.from_numpy(prior).cuda()
    out, kept, stats = ops.filter_components(maps, params, prior=p, **kw)
    return out, kept, stats


def _check(z, params, prior, got):
    out, kept, stats = got
    w_out, w_kept, w_stats = ref.filter_components(z, params.mode, params.radius, params.connectivity, prior)
    assert np.array_equal(stats.cpu().numpy(), w_stats)
    assert np.array_equal(kept.cpu().numpy(), w_kept)
    assert out.cpu().numpy()[:, :, 0].tobytes() == w_out.tobytes()


FILTER_CASES = ([("largest", 32, k, c, False) for k in (1, 2, 3, 4) for c in (4, 8)]
                + [("near", r, k, 8, p) for r in (0, 1, 32, 5000) for k in (1, 2, 3, 4) for p in (False, True)]
                + [("near", 5, 2, 4, True)])


@pytest.mark.parametrize("mode,radius,k,connectivity,with_prior", FILTER_CASES)
def test_filter_equals_restatement(mode, radius, k, connectivity, with_prior):
    from osvos_pytorch_b200 import ops
    n, h, w = 3, 61, 97
    z = _maps(radius * 10 + k, k, n, h, w)
    prior = _prior(k, k, h, w) if with_prior else None
    params = ops.Components(mode, radius=radius, connectivity=connectivity)
    _check(z, params, prior, _filter(z, params, prior))


@pytest.mark.parametrize("mode", ["largest", "near"])
def test_filter_at_480x854(mode):
    from osvos_pytorch_b200 import ops
    z = _maps(7, 2, 2, 480, 854)
    prior = _prior(7, 2, 480, 854)
    params = ops.Components(mode)
    _check(z, params, prior, _filter(z, params, prior))


def test_one_component_largest_is_the_map_bit_for_bit():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(9)
    z = (rng.standard_normal((1, 2, 40, 50)) - 8).astype(np.float32)
    z[0, :, 5:30, 10:40] = np.abs(z[0, :, 5:30, 10:40]) + 0.1
    z[0, 0, 0, 0], z[0, 0, 0, 1] = -0.0, np.nan
    out, _, stats = _filter(z, ops.Components("largest"))
    assert out.cpu().numpy()[:, :, 0].tobytes() == z.tobytes()
    assert stats[..., 0].tolist() == [[1, 1]]


def _same(a, b):
    """Bit equality (the maps hold NaN)."""
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return torch.equal(a, b)


@pytest.mark.parametrize("det", [False, True])
def test_two_runs_are_bit_identical(det):
    from osvos_pytorch_b200 import ops
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    z, prior = _maps(11, 3, 2, 120, 200), _prior(11, 3, 120, 200)
    _, masks = _masks(11, 120, 200)
    try:
        torch.use_deterministic_algorithms(det)
        runs = [[_filter(z, ops.Components(m), prior) for m in ("largest", "near")]
                + [ops.connected_components(torch.from_numpy(masks).cuda(), c) for c in (4, 8)] for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    runs.append([_filter(z, ops.Components(m), prior) for m in ("largest", "near")]
                + [ops.connected_components(torch.from_numpy(masks).cuda(), c) for c in (4, 8)])
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert all(_same(x, y) for x, y in zip(a, b))


def test_filter_misaligned_prior_and_out():
    from osvos_pytorch_b200 import ops
    k, n, h, w = 2, 2, 37, 45
    z, prior = _maps(13, k, n, h, w), _prior(13, k, h, w)
    params = ops.Components("near", radius=4)
    want = _filter(z, params, prior)
    buf = torch.empty(prior.size + 1, dtype=torch.uint8, device="cuda")
    view = buf[1:].view(prior.shape)
    view.copy_(torch.from_numpy(prior))
    out = torch.full((k * n * h * w,), float("nan"), device="cuda")
    got = ops.filter_components([torch.from_numpy(m).cuda() for m in z], params, prior=view, out=out)
    assert got[0].data_ptr() == out.data_ptr()
    assert all(_same(a, b) for a, b in zip(want, got))


def test_invalid_arguments_raise_before_any_launch():
    from osvos_pytorch_b200 import _native as nat, ops
    m = torch.zeros((1, 8, 9), dtype=torch.uint8, device="cuda")
    z = torch.zeros((1, 1, 8, 9), device="cuda")
    before = ops.KERNEL_LAUNCHES[0]
    for kw in (dict(masks=m.float()), dict(masks=m[0]), dict(masks=m, connectivity=6), dict(masks=m.cpu()),
               dict(masks=m, connectivity=True), dict(masks=m[:0])):
        with pytest.raises((ValueError, RuntimeError)):
            ops.connected_components(**kw)
    p = ops.Components("near")
    for kw in (dict(maps=[z], params=dict(mode="near")), dict(maps=[z], params="largest"),
               dict(maps=[z.double()], params=p), dict(maps=[], params=p), dict(maps=[z] * 255, params=p),
               dict(maps=[z], params=p, prior=m.float()), dict(maps=[z], params=p, prior=m[:, :, :8]),
               dict(maps=[z, z], params=p, prior=m), dict(maps=[z], params=p, prior=m.cpu()),
               dict(maps=[z], params=p, out=torch.empty(71, device="cuda")),
               dict(maps=[z], params=p, out=torch.empty(72, device="cuda", dtype=torch.float64)),
               dict(maps=[z.cpu()], params=p)):
        with pytest.raises((ValueError, RuntimeError)):
            ops.filter_components(**kw)
    with pytest.raises(ValueError, match="32767"):
        ops.connected_components(torch.zeros((1, 1, 32768), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="32767"):
        ops.filter_components([torch.zeros((1, 32768, 1), device="cuda")], ops.Components("largest"))
    assert ops.KERNEL_LAUNCHES[0] == before
    # the library's own checks, with placeholder device addresses that are never dereferenced
    lib, addr, s = nat.load(), 1 << 20, None
    ptrs = (ctypes.c_void_p * 2)(addr, addr)
    assert lib.osvos_filter_components(ptrs, None, addr, addr, addr, addr, 8, 2, 1 << 14, 1 << 14, 0, 1, 8, s) == 1
    assert b"sizes_ok" in lib.osvos_last_error()
    assert lib.osvos_filter_components(ptrs, None, addr, addr, addr, addr, 1, 1, 32768, 4, 0, 1, 8, s) == 1
    assert lib.osvos_filter_components(ptrs, None, addr, addr, addr, addr, 1, 1, 8, 8, 2, 1, 8, s) == 1
    assert lib.osvos_filter_components(ptrs, None, addr, addr, addr, addr, 1, 1, 8, 8, 0, -1, 8, s) == 1
    assert lib.osvos_filter_components(ptrs, None, addr, addr, addr, addr, 1, 1, 8, 8, 0, 1, 6, s) == 1
    assert lib.osvos_connected_components(addr, addr, addr, addr, 1 << 11, 1 << 10, 1 << 10, 8, s) == 1
    assert lib.osvos_connected_components(addr, addr, addr, addr, 1, 4, 32768, 8, s) == 1
    assert lib.osvos_filter_components_workspace_bytes(8, 2, 1 << 14, 1 << 14, 0) == 0
    assert lib.osvos_connected_components_workspace_bytes(1, 32768, 1) == 0


# ---- the segmenter --------------------------------------------------------------------------------------------------

def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


def _scene(seed, n, h, w):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), (xx + yy) % 256], -1)
    frames = np.empty((n, h, w, 3), np.uint8)
    for i in range(n):
        f = base + rng.integers(-20, 21, size=(h, w, 3))
        blob = (xx - w * (0.3 + 0.1 * i)) ** 2 + (yy - h / 2) ** 2 < (min(h, w) / 3) ** 2
        f[blob] = (200, 40 + 30 * i, 90)
        frames[i] = np.clip(f, 0, 255)
    return frames


def _items(seed, n_frames, h, w, k_ids=None):
    rng = np.random.default_rng(seed)
    frames = [torch.from_numpy(_scene(seed + i, 1, h, w)).pin_memory() for i in range(n_frames)]
    hi = 2 if k_ids is None else k_ids + 1
    gts = [torch.from_numpy((rng.integers(0, hi, (1, h, w)) * (255 if k_ids is None else 1)).astype(np.uint8))
           for _ in range(n_frames)]
    return frames, gts


def _centred(net, frame):
    """Move the fused map's threshold to its median on ``frame``, so the foreground breaks into several components."""
    from osvos_pytorch_b200 import ops
    with torch.no_grad():
        z = net(ops.image_from_bgr8(frame.cuda()))[-1]
        net.fuse.bias -= z.median()
    return net


def _files(x):
    if isinstance(x, tuple) and len(x) == 2 and torch.is_tensor(x[0]):
        buf, lens = x[0].cpu().numpy(), x[1].cpu().tolist()
        return [bytes(buf[j, :int(n)]) for j, n in enumerate(lens)]
    return [bytes(v) for v in x]


@pytest.mark.parametrize("case", ["2016", "2016_near", "2016_f32", "2017", "crf"])
def test_segmenter_with_components_equals_the_eager_restatement(case):
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    from png_palette_ref import davis_palette
    h, w = 40, 56
    crf = ops.CRF(iterations=2, bilateral_weight=6.0, bilateral_xy=20.0, bilateral_rgb=15.0) if case == "crf" else None
    params = ops.Components("near" if case in ("2016_near", "2017") else "largest", radius=6)
    kw = {}
    if case == "2017":
        nets = [_he_net(seed=1).cuda().eval(), _he_net(seed=2).cuda().eval()]
        frames, gts = _items(5, 4, h, w, k_ids=2)
        pal = davis_palette(3)
        res = dict(input_res=(24, 32))
        prior = torch.zeros((2, 24, 32), dtype=torch.uint8)
        prior[0, 4:12, 4:14] = 1
        prior[1, 14:22, 18:30] = 1
        seg = SequenceSegmenter(nets=nets, output="labels", depth=2, frames="bgr8", score=True, encode="png",
                                palette=pal, output_res="stored", components=params, components_prior=prior, **res)
    else:
        frames, gts = _items(6, 4, h, w)
        nets = [_centred(_he_net(seed=3).cuda().eval(), frames[0])]
        res = {}
        prior = None
        if case == "2016_near":
            prior = torch.zeros((1, h, w), dtype=torch.uint8)
            prior[0, 10:30, 5:25] = 1
        fmode = "nchw_f32" if case == "2016_f32" else "bgr8"
        if fmode == "nchw_f32":
            frames = [ops.image_from_bgr8(f.cuda()).cpu().pin_memory() for f in frames]
        seg = SequenceSegmenter(nets[0], output="bytescale", depth=2, frames=fmode, score=True,
                                encode="png" if fmode == "bgr8" else None, overlay="jpeg" if case == "2016" else None,
                                crf=crf, components=params, components_prior=prior)
    got = []
    for r in seg(iter(list(zip(frames, gts)))):
        if isinstance(r, tuple):
            got.append((_files(r[0]), _files(r[1])))
        elif torch.is_tensor(r):
            got.append(r.clone())
        else:
            got.append(_files(r))
    counts, cstats = seg.frame_counts(), seg.component_stats()
    fmode = "nchw_f32" if case == "2016_f32" else "bgr8"
    logits = [[r.clone() for r in SequenceSegmenter(net, output="logits", depth=2, frames=fmode, **res)(iter(frames))]
              for net in nets]
    want, want_counts, want_stats = [], [], []
    p = None if prior is None else prior.cuda()
    with torch.no_grad():
        for i, (f, g) in enumerate(zip(frames, gts)):
            gd = g.cuda()
            fused = [lg[i].cuda() for lg in logits]
            if crf is not None:
                fused = list(ops.dense_crf(f.cuda(), fused, crf).unbind(0))
            filtered, kept, stats = ops.filter_components(fused, params, prior=p if params.mode == "near" else None)
            p = kept[:, -1].contiguous()
            want_stats.append(stats.permute(1, 0, 2))
            maps = list(filtered.unbind(0))
            if case == "2017":
                labels = ops.upsample_merge_objects(maps, (h, w)).view(1, 1, h, w)
                want_counts.append(ops.davis_measures_objects(labels, gd, 2))
                want.append(_files(ops.encode_png(labels, palette=pal)))
            else:
                r = maps[0]
                want_counts.append(ops.davis_measures(r, gd))
                u8 = ops.logits_to_u8(r, "bytescale")
                if fmode == "nchw_f32":
                    want.append(u8.cpu())
                    continue
                files = _files(ops.encode_png(u8))
                if case == "2016":
                    want.append((files, _files(ops.encode_jpeg(ops.overlay_mask(f.cuda(), r), 95))))
                else:
                    want.append(files)
    assert counts.tolist() == torch.cat(want_counts).cpu().tolist()
    assert cstats.tolist() == torch.cat(want_stats).cpu().tolist()
    if fmode == "nchw_f32":
        assert all(torch.equal(a, b) for a, b in zip(got, want))
    else:
        assert got == want
    assert int(cstats[..., 2].sum()) > 0                 # the filter saw foreground
    if case == "2017":                                   # and there it removed some
        assert int(cstats[..., 3].sum()) > 0


def test_segmenter_refuses_bad_components():
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda()
    with pytest.raises(ValueError, match="components"):
        SequenceSegmenter(net, output="bytescale", components=dict(mode="largest"))
    with pytest.raises(ValueError, match="components_prior"):
        SequenceSegmenter(net, output="bytescale", components_prior=torch.zeros((1, 4, 4), dtype=torch.uint8))
    with pytest.raises(ValueError, match="components_prior"):
        SequenceSegmenter(net, output="bytescale", components=ops.Components("near"),
                          components_prior=torch.zeros((1, 4, 4)))
    seg = SequenceSegmenter(net, output="bytescale", depth=2, frames="bgr8", components=ops.Components("near"),
                            components_prior=torch.zeros((1, 4, 4), dtype=torch.uint8))
    with pytest.raises(ValueError, match="components_prior"):
        list(seg(iter([torch.zeros((1, 8, 8, 3), dtype=torch.uint8)])))
    with pytest.raises(RuntimeError, match="component_stats"):
        SequenceSegmenter(net, output="bytescale").component_stats()


# ---- adaptation with the filter ---------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def _sequence(tree):
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True, seq_name=None)
    items = [d[i] for i in range(3)]
    for it in items[:2]:
        items.append(dict(it, image=np.ascontiguousarray(it["image"][:, ::-1]), gt=np.ascontiguousarray(it["gt"][:, ::-1])))
    return [davis.collate([it]) for it in items]


def _adapted(tree, components):
    from osvos_pytorch_b200 import augment, davis, training
    from osvos_pytorch_b200.inference import SequenceSegmenter
    batches = _sequence(tree)
    img_u8, gt_u8, stats = davis.upload(batches[0], torch.device("cuda"))
    rng = random.Random(7)

    def sample_fn(it):
        return augment.affine_warp_u8(img_u8, gt_u8, augment.draw_params(1, rng=rng), stats)

    def frames():
        for b in batches:
            img, _ = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
            yield img
    net = _he_net(seed=4).cuda()
    adapt = training.OnlineAdaptation(net, sample_fn, gt_u8, 1e-10, 0.0002, steps=4, current_steps=2, weight=0.5,
                                      alpha=0.9, distance=10, erosion=1)
    seg = SequenceSegmenter(net, output="logits", depth=2, frames="bgr8", adapt=adapt, components=components,
                            components_prior=None if components is None else (gt_u8 != 0).to(torch.uint8))
    res = [r.clone() for r in seg(frames())]
    return res, adapt, {k: v.clone() for k, v in net.state_dict().items()}


def test_adapt_with_components_adapts_as_without(tree):
    from osvos_pytorch_b200 import ops
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        plain, ad_plain, w_plain = _adapted(tree, None)
        filtered, ad_f, w_f = _adapted(tree, ops.Components("near", radius=2))
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    assert all(torch.equal(a, b) for a, b in zip(ad_plain.counts, ad_f.counts)) and ad_plain.skipped == ad_f.skipped
    assert all(torch.equal(w_plain[k], w_f[k]) for k in w_plain)
    for a, b in zip(plain, filtered):                    # the filter only ever negates positive logits
        assert torch.equal(torch.where(b != a, -b, b), a) and bool((a[b != a] > 0).all())


# ---- train_online.py --components -------------------------------------------------------------------------------------

def test_train_online_components_2016(tree, tmp_path, monkeypatch, capsys):
    import train_online
    torch.save(_he_net(seed=3).state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    try:
        train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                           "--parent-epoch", "1", "--no-save", "--loader", "native", "--evaluate", "--encode", "device",
                           "--components", "near", "--components-radius", "3", "--components-connectivity", "4"])
    finally:
        gc.collect()
    res = json.load(open(tmp_path / "Results" / "cc_scores.json"))
    comp = res["components"]
    assert (comp["mode"], comp["radius"], comp["connectivity"]) == ("near", 3, 4)
    stats = np.array(comp["stats"])
    assert stats.shape == (2, 1, 4) and (stats[..., 1] <= stats[..., 0]).all()
    assert sorted(os.listdir(tmp_path / "Results" / "cc")) == ["00000.png", "00001.png"]
    assert f"covering {int(stats[..., 3].sum())} pixel(s)" in capsys.readouterr().out


def _tree_2017(root):
    cv2 = pytest.importorskip("cv2")
    from PIL import Image
    from png_palette_ref import davis_palette
    rng = np.random.default_rng(21)
    os.makedirs(root / "JPEGImages" / "480p" / "s2")
    os.makedirs(root / "Annotations" / "480p" / "s2")
    frames = _scene(9, 4, 40, 56)
    for f in range(4):
        cv2.imwrite(str(root / "JPEGImages" / "480p" / "s2" / f"{f:05d}.jpg"), frames[f])
        gt = np.zeros((40, 56), np.uint8)
        gt[5:20, 5 + f:25 + f] = 1
        gt[22:35, 30:50 - f] = 2
        if f % 2:
            gt[:, 27] = 255
        gt[rng.integers(0, 40, 20), rng.integers(0, 56, 20)] = 2
        im = Image.fromarray(gt, "P")
        im.putpalette(davis_palette(256))
        im.save(str(root / "Annotations" / "480p" / "s2" / f"{f:05d}.png"))
    os.makedirs(root / "ImageSets" / "2017")
    (root / "ImageSets" / "2017" / "val.txt").write_text("s2\n")
    return str(root)


@pytest.mark.parametrize("mode", ["largest", "near"])
def test_train_online_components_2017_scores_equal_score_results(mode, tmp_path, monkeypatch):
    import train_online
    from osvos_pytorch_b200 import evaluation
    db = _tree_2017(tmp_path / "db")
    torch.save(_he_net(seed=3).state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", db)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    try:
        train_online.main(["--seq-name", "s2", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                           "--parent-epoch", "1", "--no-save", "--loader", "native", "--davis", "2017", "--evaluate",
                           "--input-res", "24", "32", "--output-res", "stored", "--encode", "device",
                           "--components", mode])
    finally:
        gc.collect()
    results = tmp_path / "Results"
    written = json.load(open(results / "s2_scores.json"))
    assert written["components"]["mode"] == mode and np.array(written["components"]["stats"]).shape == (4, 2, 4)
    scored = evaluation.score_results(str(results), db, sequences=["s2"], device="cuda", davis="2017")
    assert written["counts"] == scored["sequences"]["s2"]["counts"]

"""ops.dense_crf (csrc/crf.cu, DESIGN.md §29) against the float64 restatement tests/crf_ref.py, and the CRF in
SequenceSegmenter and train_online.py.

Error bound of the refined maps (u = 2^-24, fp32 round-off; all sums on the device run in a fixed order):
  - splat: a vertex's value is a sum of m positive products w·Q, m its occupancy, added by 256 threads (each a
    sequential sum of at most ceil(m/256) terms) and a tree of depth 8: relative error <= (ceil(m/256) + 9)u;
  - 6 blur passes, each ½v + ¼(v⁻ + v⁺) of positive terms: <= 3u each; slice, 6 positive products: <= 7u; Q itself
    (expf, a sum of K + 1 terms, a division) <= (K + 6)u.  B = F(Q)·(1/F(1)), both ratios of such terms, B in [0, 1]:
    |ΔB| <= e_B = 2(ceil(m_max/256) + 9 + 18 + 7 + K + 6)u + 2u;
  - S, (2R+1)-tap rows then columns of positive terms, and the in-frame tap sums: |ΔS| <= e_S = 2(3(2R+1) + 8)u,
    R = ceil(3θγ);
  - a = a⁰ + w_α B + w_γ S and r = a_k - a_0: a fresh error per iteration of e_a = w_α e_B + w_γ e_S
    + 4u(max|z| + w_α + w_γ);
  - an error Δa in one iteration's a moves Q by at most ½|Δa| (the softmax Jacobian's ∞-norm is max 2Q(1-Q) <= ½),
    and B and S, convex combinations of Q, by no more; so after T iterations |Δa| <= e_a Σ_{t<T} L^t, L = (w_α + w_γ)/2,
    and |Δr| <= 2 e_a Σ_{t<T} L^t.  The test allows twice that for the neglected second-order terms.
T = 1 runs with w_γ = 0 see the lattice alone: the vertex counts are compared exactly, and any vertex or weight that
differed from the restatement's would move B by far more than e_B."""
import gc
import json
import math
import os
import random

import numpy as np
import pytest
import torch

import crf_ref as ref
import davis_fixture

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture(autouse=True)
def release_graphs():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _scene(seed, n, h, w):
    """Frames with structure (a colour ramp, two flat blobs, noise) and logits that roughly follow it."""
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


def _maps(seed, k, n, h, w):
    rng = np.random.default_rng(seed + 100)
    return (rng.standard_normal((k, n, h, w)) * 3).astype(np.float32)


def _bound(lat, z, iterations, w_a, w_g, theta_g, k):
    m = int(lat.occupancy.max())
    r = math.ceil(3 * theta_g)
    e_b = 2 * (-(-m // 256) + 9 + 18 + 7 + k + 6) * U + 2 * U
    e_s = 2 * (3 * (2 * r + 1) + 8) * U
    e_a = w_a * e_b + w_g * e_s + 4 * U * (float(np.abs(z).max()) + w_a + w_g)
    lip = (w_a + w_g) / 2
    return 2 * 2 * e_a * sum(lip ** t for t in range(iterations))


def _run(frames, z, crf, **kw):
    from osvos_pytorch_b200 import ops
    f = torch.from_numpy(frames).cuda()
    maps = torch.from_numpy(z).cuda()
    verts = torch.zeros(frames.shape[0], dtype=torch.int32, device="cuda")
    out = ops.dense_crf(f, maps, crf, vertices=verts, **kw)
    return out, verts


PARAMS = {
    "default": dict(),
    "lattice": dict(iterations=1, gaussian_weight=0.0),
    "lattice_fine": dict(iterations=1, gaussian_weight=0.0, bilateral_xy=9.0, bilateral_rgb=5.0, bilateral_weight=4.0),
    "two": dict(iterations=2, bilateral_weight=3.0, bilateral_xy=30.0, bilateral_rgb=20.0, gaussian_weight=1.5,
                gaussian_xy=1.3),
    "smooth_only": dict(iterations=1, bilateral_weight=0.0, gaussian_xy=7.5),
}

CASES = [((1, 1), 1, 1, "default"), ((1, 1), 2, 3, "lattice"), ((7, 5), 1, 1, "lattice_fine"),
         ((7, 5), 5, 3, "default"), ((7, 5), 2, 1, "two"), ((33, 45), 1, 1, "lattice"), ((33, 45), 2, 3, "default"),
         ((33, 45), 5, 1, "lattice_fine"), ((33, 45), 1, 3, "smooth_only"), ((480, 854), 1, 1, "lattice"),
         ((480, 854), 1, 1, "default"), ((480, 854), 2, 1, "two"), ((5, 4000), 5, 3, "lattice"),
         ((5, 4000), 1, 1, "default")]


@pytest.mark.parametrize("hw,k,n,params", CASES)
def test_dense_crf_matches_restatement(hw, k, n, params):
    from osvos_pytorch_b200 import ops
    crf = ops.CRF(**PARAMS[params])
    h, w = hw
    frames, z = _scene(h * w + n, n, h, w), _maps(k + n, k, n, h, w)
    out, verts = _run(frames, z, crf)
    assert out.shape == (k, n, 1, h, w)
    lat = ref.Lattice(frames, crf.bilateral_xy, crf.bilateral_rgb, weights_f32=True)
    assert verts.cpu().tolist() == lat.per_frame.tolist()          # the keys, exactly
    want = ref.dense_crf(frames, z, crf.iterations, crf.bilateral_weight, crf.bilateral_xy, crf.bilateral_rgb,
                         crf.gaussian_weight, crf.gaussian_xy, lattice=lat)
    got = out[:, :, 0].double().cpu().numpy()
    bound = _bound(lat, z, crf.iterations, float(np.float32(crf.bilateral_weight)),
                   float(np.float32(crf.gaussian_weight)), crf.gaussian_xy, k)
    err = float(np.abs(got - want).max())
    assert err <= bound, (err, bound)
    if crf.iterations == 1:
        assert bound < 0.05                                        # a wrong vertex or weight moves B by ~0.1 or more


def test_zero_iterations_are_bit_exact():
    from osvos_pytorch_b200 import ops
    frames, z = _scene(1, 2, 9, 13), _maps(1, 3, 2, 9, 13)
    z[0, 0, 0, 0] = -0.0
    out, _ = _run(frames, z, ops.CRF(iterations=0))
    assert torch.equal(out[:, :, 0].cpu(), torch.from_numpy(z))
    assert np.signbit(out[0, 0, 0, 0, 0].item())


@pytest.mark.parametrize("det", [False, True])
def test_two_calls_are_bit_identical(det):
    from osvos_pytorch_b200 import ops
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    frames, z = _scene(2, 2, 120, 200), _maps(2, 2, 2, 120, 200)
    try:
        torch.use_deterministic_algorithms(det)
        a, va = _run(frames, z, ops.CRF())
        b, vb = _run(frames, z, ops.CRF())
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    c, _ = _run(frames, z, ops.CRF())
    assert torch.equal(a, b) and torch.equal(a, c) and torch.equal(va, vb)


def test_misaligned_frames_and_out():
    from osvos_pytorch_b200 import ops
    n, h, w = 2, 17, 23
    frames, z = _scene(3, n, h, w), _maps(3, 2, n, h, w)
    want, _ = _run(frames, z, ops.CRF())
    buf = torch.empty(n * h * w * 3 + 1, dtype=torch.uint8, device="cuda")
    view = buf[1:].view(n, h, w, 3)
    view.copy_(torch.from_numpy(frames))
    assert view.data_ptr() % 2 == 1
    out = torch.full((2 * n * h * w,), float("nan"), device="cuda")
    got = ops.dense_crf(view, [torch.from_numpy(m).cuda() for m in z], ops.CRF(), out=out)
    assert got is out and torch.equal(out.view(want.shape), want)


def test_invalid_arguments_raise_before_any_launch():
    from osvos_pytorch_b200 import _native as nat, ops
    f = torch.zeros((1, 8, 9, 3), dtype=torch.uint8, device="cuda")
    m = torch.zeros((1, 1, 8, 9), device="cuda")
    before = ops.KERNEL_LAUNCHES[0]
    bad = [
        dict(frames=f.float(), maps=[m]),
        dict(frames=f[..., :2], maps=[m]),
        dict(frames=f, maps=[m[..., :8]]),
        dict(frames=f, maps=[m.double()]),
        dict(frames=f, maps=[]),
        dict(frames=f, maps=[m] * 255),
        dict(frames=f, maps=[m], out=torch.empty(71, device="cuda")),
        dict(frames=f, maps=[m], crf=dict(iterations=1)),
        dict(frames=f, maps=[m], vertices=torch.empty(2, dtype=torch.int32, device="cuda")),
        dict(frames=f.cpu(), maps=[m]),
    ]
    for kw in bad:
        with pytest.raises((ValueError, RuntimeError)):
            ops.dense_crf(**kw)
    big = torch.zeros((1, 480, 854, 3), dtype=torch.uint8, device="cuda")
    bm = torch.zeros((1, 1, 480, 854), device="cuda")
    with pytest.raises(nat.NativeLibraryError, match="crf_fits"):     # the keys' range: θα 0.5 on 854 columns
        ops.dense_crf(big, [bm], ops.CRF(bilateral_xy=0.5))
    with pytest.raises(nat.NativeLibraryError, match="crf_fits"):
        ops.dense_crf(big, [bm], ops.CRF(bilateral_rgb=0.05))
    assert ops.KERNEL_LAUNCHES[0] == before
    ops.dense_crf(big, [bm], ops.CRF(bilateral_xy=40.0))             # well inside the range
    torch.cuda.synchronize()


# ---- the segmenter ----------------------------------------------------------------------------------------------------

def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


CRF_SEG = dict(iterations=3, bilateral_weight=6.0, bilateral_xy=20.0, bilateral_rgb=15.0)


def _bgr_items(seed, n_frames, h, w, k_ids=None):
    rng = np.random.default_rng(seed)
    frames = [torch.from_numpy(_scene(seed + i, 1, h, w)).pin_memory() for i in range(n_frames)]
    hi = 2 if k_ids is None else k_ids + 1
    gts = [torch.from_numpy((rng.integers(0, hi, (1, h, w)) * (255 if k_ids is None else 1)).astype(np.uint8))
           for _ in range(n_frames)]
    return frames, gts


@pytest.mark.parametrize("case", ["2016", "input_res", "2017"])
def test_segmenter_with_crf_equals_the_eager_restatement(case):
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    from png_palette_ref import davis_palette
    crf = ops.CRF(**CRF_SEG)
    h, w = 40, 56
    if case == "2017":
        nets = [_he_net(seed=1).cuda().eval(), _he_net(seed=2).cuda().eval()]
        frames, gts = _bgr_items(5, 3, h, w, k_ids=2)
        pal = davis_palette(3)
        seg = SequenceSegmenter(nets=nets, output="labels", depth=2, frames="bgr8", score=True, encode="png",
                                palette=pal, crf=crf)
    else:
        nets = [_he_net(seed=3).cuda().eval()]
        frames, gts = _bgr_items(6, 3, h, w)
        kw = dict(input_res=(24, 32), output_res="stored") if case == "input_res" else {}
        seg = SequenceSegmenter(nets[0], output="bytescale", depth=2, frames="bgr8", score=True, encode="png",
                                overlay="jpeg" if case == "2016" else None, crf=crf, **kw)
    got = []
    for r in seg(iter(list(zip(frames, gts)))):
        if isinstance(r, tuple):
            got.append(([bytes(x) for x in r[0]], [bytes(x) for x in r[1]]))
        else:
            got.append([bytes(x) for x in r])
    counts = seg.frame_counts()
    # the forwards as the segmenter without crf runs them: its fp32 logits at the network resolution
    res = dict(input_res=(24, 32)) if case == "input_res" else {}
    logits = [[r.clone() for r in SequenceSegmenter(net, output="logits", depth=2, frames="bgr8", **res)(iter(frames))]
              for net in nets]
    want, want_counts = [], []
    with torch.no_grad():
        for i, (f, g) in enumerate(zip(frames, gts)):
            raw, gd = f.cuda(), g.cuda()
            if case == "input_res":
                raw = ops.resize_u8(raw, (24, 32), "bilinear")
            fused = [lg[i].cuda() for lg in logits]
            refined = list(ops.dense_crf(raw, fused, crf).unbind(0))
            if case == "2017":
                labels = ops.merge_objects(refined).view(1, 1, h, w)
                want_counts.append(ops.davis_measures_objects(labels, gd, 2))
                pngs = ops.encode_png(labels, palette=pal)
            else:
                r = refined[0]
                if case == "input_res":
                    r = ops.resize_f32(r, (h, w))
                want_counts.append(ops.davis_measures(r, gd))
                pngs = ops.encode_png(ops.logits_to_u8(r, "bytescale"))
            files = [bytes(p) for p in pngs] if isinstance(pngs, list) else pngs
            if case == "2016":
                jpg = ops.encode_jpeg(ops.overlay_mask(f.cuda(), refined[0]), 95)
                want.append((files, jpg))
            else:
                want.append(files)
    assert counts.tolist() == torch.cat(want_counts).cpu().tolist()
    assert _as_bytes(got) == _as_bytes(want)


def _as_bytes(items):
    """Results as lists of bytes: memoryviews, or ops.encode_png / encode_jpeg's (buffer, lengths) pairs."""
    def files(x):
        if isinstance(x, tuple) and len(x) == 2 and torch.is_tensor(x[0]):
            buf, lens = x[0].cpu().numpy(), x[1].cpu().tolist()
            return [bytes(buf[j, :int(n)]) for j, n in enumerate(lens)]
        return [bytes(v) for v in x]
    out = []
    for it in items:
        if isinstance(it, tuple) and len(it) == 2 and not torch.is_tensor(it[0]):
            out.append((files(it[0]), files(it[1])))
        else:
            out.append(files(it))
    return out


def test_segmenter_refuses_crf_without_bytes():
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda()
    with pytest.raises(ValueError, match="crf"):
        SequenceSegmenter(net, output="bytescale", crf=ops.CRF())
    with pytest.raises(ValueError, match="crf"):
        SequenceSegmenter(net, output="bytescale", frames="bgr8", crf=dict(iterations=1))


# ---- adaptation with the CRF ------------------------------------------------------------------------------------------

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


def _frames(batches):
    from osvos_pytorch_b200 import davis
    for b in batches:
        img, _ = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
        yield img


def _adapted(tree, crf):
    from osvos_pytorch_b200 import augment, davis, training
    from osvos_pytorch_b200.inference import SequenceSegmenter
    batches = _sequence(tree)
    img_u8, gt_u8, stats = davis.upload(batches[0], torch.device("cuda"))
    rng = random.Random(7)

    def sample_fn(it):
        return augment.affine_warp_u8(img_u8, gt_u8, augment.draw_params(1, rng=rng), stats)
    net = _he_net(seed=4).cuda()
    adapt = training.OnlineAdaptation(net, sample_fn, gt_u8, 1e-10, 0.0002, steps=4, current_steps=2, weight=0.5,
                                      alpha=0.9, distance=10, erosion=1)
    seg = SequenceSegmenter(net, output="logits", depth=2, frames="bgr8", adapt=adapt, crf=crf)
    res = [r.clone() for r in seg(_frames(batches))]
    return res, adapt, {k: v.clone() for k, v in net.state_dict().items()}


def test_adapt_with_crf_adapts_as_without(tree):
    from osvos_pytorch_b200 import ops
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        plain, ad_plain, w_plain = _adapted(tree, None)
        refined, ad_crf, w_crf = _adapted(tree, ops.CRF(**CRF_SEG))
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    assert all(torch.equal(a, b) for a, b in zip(ad_plain.counts, ad_crf.counts)) and ad_plain.skipped == ad_crf.skipped
    assert all(torch.equal(w_plain[k], w_crf[k]) for k in w_plain)
    assert any(not torch.equal(a, b) for a, b in zip(plain, refined))     # the CRF did change the results


# ---- train_online.py --crf --------------------------------------------------------------------------------------------

def test_train_online_crf_2016(tree, tmp_path, monkeypatch):
    import train_online
    torch.save(_he_net(seed=3).state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    try:
        train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                           "--parent-epoch", "1", "--no-save", "--loader", "native", "--evaluate", "--encode", "device",
                           "--crf", "--crf-iterations", "2", "--crf-bilateral", "5", "30", "10"])
    finally:
        gc.collect()
    res = json.load(open(tmp_path / "Results" / "cc_scores.json"))
    assert res["crf"] == dict(iterations=2, bilateral_weight=5.0, bilateral_xy=30.0, bilateral_rgb=10.0,
                              gaussian_weight=3.0, gaussian_xy=3.0)
    assert sorted(os.listdir(tmp_path / "Results" / "cc")) == ["00000.png", "00001.png"]
    assert len(res["J"]) == len(res["counts"]) == 2


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


def test_train_online_crf_2017_scores_equal_score_results(tmp_path, monkeypatch):
    import train_online
    from osvos_pytorch_b200 import evaluation
    db = _tree_2017(tmp_path / "db")
    torch.save(_he_net(seed=3).state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", db)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    try:
        train_online.main(["--seq-name", "s2", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                           "--parent-epoch", "1", "--no-save", "--loader", "native", "--davis", "2017", "--evaluate",
                           "--input-res", "24", "32", "--output-res", "stored", "--encode", "device", "--crf"])
    finally:
        gc.collect()
    results = tmp_path / "Results"
    written = json.load(open(results / "s2_scores.json"))
    assert written["crf"] == dict(iterations=5, bilateral_weight=10.0, bilateral_xy=80.0, bilateral_rgb=13.0,
                                  gaussian_weight=3.0, gaussian_xy=3.0)
    scored = evaluation.score_results(str(results), db, sequences=["s2"], device="cuda", davis="2017")
    assert written["counts"] == scored["sequences"]["s2"]["counts"]
    for k in (1, 2):
        assert written["objects"][str(k)]["J"] == scored["sequences"]["s2"]["objects"][k]["J"]
        assert written["objects"][str(k)]["F"] == scored["sequences"]["s2"]["objects"][k]["F"]

"""DAVIS-2017 on the device (DESIGN.md §24): ops.merge_objects, ops.davis_measures_objects, palette PNG decode and
encode, SequenceSegmenter(nets=..., output="labels"), score_results(davis="2017") and train_online.py --davis 2017,
each against its numpy restatement (tests/davis_objects_ref.py, tests/png_palette_ref.py) or Pillow."""
import gc
import io
import json
import os

import numpy as np
import pytest
import torch

import davis_measures_ref as M
import davis_objects_ref as O
import png_palette_ref as PP
import png_ref as P
from png_palette_ref import davis_palette, pillow_palette_png

pytestmark = pytest.mark.gpu
Image = pytest.importorskip("PIL.Image")


# ---- merge ------------------------------------------------------------------------------------------------------------

def _maps(k, n, h, w, seed):
    rng = np.random.default_rng(seed)
    m = rng.normal(0, 2, (k, n, 1, h, w)).astype(np.float32)
    m = np.round(m * 2) / 2                                      # many exact ties
    flat = m.reshape(k, -1)
    sel = rng.random(flat.shape[1])
    flat[:, sel < 0.05] = np.nan
    flat[:, (sel >= 0.05) & (sel < 0.1)] = 0.0
    flat[:, (sel >= 0.1) & (sel < 0.15)] = -0.0
    flat[rng.integers(0, k), sel > 0.97] = np.nan                 # NaN in one map beside finite values
    return m


@pytest.mark.parametrize("k", range(1, 9))
@pytest.mark.parametrize("n,h,w", [(1, 17, 23), (3, 40, 57), (2, 480, 854)])
def test_merge_objects_equals_numpy(k, n, h, w):
    from osvos_pytorch_b200 import ops
    m = _maps(k, n, h, w, seed=k * 100 + w)
    want = O.merge(m).reshape(n, h, w)
    dev = torch.from_numpy(m).cuda()
    assert np.array_equal(ops.merge_objects(dev).cpu().numpy(), want)
    # K separate tensors, an output one byte off alignment, maps 4- but not 16-byte aligned
    buf = torch.empty(n * h * w + 1, dtype=torch.uint8, device="cuda")
    flat = torch.empty(k * n * h * w + 1, dtype=torch.float32, device="cuda")
    parts = []
    for j in range(k):
        t = flat[1 + j * n * h * w:1 + (j + 1) * n * h * w].view(n, 1, h, w)
        t.copy_(dev[j])
        parts.append(t)
    got = ops.merge_objects(parts, out=buf[1:].view(n, h, w))
    assert np.array_equal(got.cpu().numpy(), want)


def test_merge_objects_refuses_bad_input():
    from osvos_pytorch_b200 import ops
    a = torch.zeros(1, 1, 4, 4, device="cuda")
    with pytest.raises(ValueError):
        ops.merge_objects([])
    with pytest.raises(ValueError):
        ops.merge_objects([a, torch.zeros(1, 1, 4, 5, device="cuda")])
    with pytest.raises(ValueError):
        ops.merge_objects([a] * 255)
    with pytest.raises(ValueError):
        ops.merge_objects([a.double()])


# ---- per-object measures ----------------------------------------------------------------------------------------------

def _scene(kind, h, w, k, seed):
    """(labels, gt) uint8 [H,W] with objects 1..k."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:h, :w]
    gt = np.zeros((h, w), np.uint8)
    lab = np.zeros((h, w), np.uint8)
    for j in range(1, k + 1):
        if kind == "absent" and j == k:
            continue
        cy, cx = rng.integers(0, h), rng.integers(0, w)
        ry, rx = rng.integers(2, max(3, h // 3)), rng.integers(2, max(3, w // 3))
        blob = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1
        gt[blob] = j
        dy, dx = rng.integers(-3, 4, 2)
        lab[np.roll(np.roll(blob, dy, 0), dx, 1)] = j
    if kind == "lines":
        gt[h // 2, :] = 1
        lab[:, w // 3] = min(2, k)
        lab[h // 4, w // 5:w // 2] = 1
    if kind == "edges":
        gt[0, :] = 1
        gt[:, -1] = k
        lab[-1, :] = 1
        lab[:, 0] = k
    if kind == "void":
        gt[:, w // 3:w // 3 + 3] = 255
        gt[h // 2:h // 2 + 2, :] = 255
    noise = rng.random((h, w)) < 0.01
    lab[noise] = rng.integers(0, k + 1, int(noise.sum()))
    return lab, gt


@pytest.mark.parametrize("kind", ["blobs", "lines", "edges", "void", "absent"])
@pytest.mark.parametrize("n,h,w,k", [(2, 37, 53, 3), (1, 64, 96, 1), (3, 30, 33, 8)])
def test_measures_objects_equal_the_restatement(kind, n, h, w, k):
    from osvos_pytorch_b200 import ops
    scenes = [_scene(kind, h, w, k, seed=i + 7 * k + h) for i in range(n)]
    lab = np.stack([s[0] for s in scenes])
    gt = np.stack([s[1] for s in scenes])
    r = M.bound_pix(h, w)
    buf = torch.empty(n * h * w + 3, dtype=torch.uint8, device="cuda")
    lab_dev = buf[3:].view(n, h, w)                               # any alignment
    lab_dev.copy_(torch.from_numpy(lab))
    got = ops.davis_measures_objects(lab_dev, torch.from_numpy(gt).cuda(), k).cpu().numpy()
    want = np.array([O.object_counts(lab[i], gt[i], k, r) for i in range(n)])
    assert got.shape == (n, k, 6) and np.array_equal(got, want)


@pytest.mark.parametrize("h,w", [(480, 854), (1080, 1920)])
def test_measures_objects_full_size(h, w):
    from osvos_pytorch_b200 import ops
    k = 3
    scenes = [_scene(kind, h, w, k, seed=i) for i, kind in enumerate(["blobs", "void"])]
    lab = np.stack([s[0] for s in scenes])
    gt = np.stack([s[1] for s in scenes])
    got = ops.davis_measures_objects(torch.from_numpy(lab).cuda(), torch.from_numpy(gt).cuda(), k).cpu().numpy()
    r = M.bound_pix(h, w)
    want = np.array([O.object_counts(lab[i], gt[i], k, r) for i in range(2)])
    assert np.array_equal(got, want)


def test_single_object_equals_davis_measures():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(4)
    for n, h, w in [(1, 45, 61), (4, 480, 854)]:
        lab = (rng.random((n, h, w)) > 0.7).astype(np.uint8)
        lab[:, h // 4:h // 2, w // 4:w // 2] = 1
        gt = (rng.random((n, h, w)) > 0.8).astype(np.uint8)
        gt[:, h // 3:2 * h // 3, w // 3:2 * w // 3] = 1
        logits = torch.from_numpy(np.where(lab == 1, 1.0, -1.0).astype(np.float32)).cuda()
        a = ops.davis_measures(logits, torch.from_numpy(gt).cuda())
        b = ops.davis_measures_objects(torch.from_numpy(lab).cuda(), torch.from_numpy(gt).cuda(), 1)
        assert torch.equal(a, b[:, 0])


# ---- palette PNGs -----------------------------------------------------------------------------------------------------

def _decode_index(datas):
    from osvos_pytorch_b200 import ops, png
    parsed = [png.parse(d, palette="index") for d in datas]
    assert all(isinstance(p, png.Parsed) for p in parsed), parsed
    blob = png.pack(parsed)
    n, h, w = len(parsed), parsed[0].h, parsed[0].w
    buf = torch.empty(n * h * w + 1, dtype=torch.uint8, device="cuda")
    out, status = ops.decode_png(torch.from_numpy(blob).cuda(), n, h, w, png.segment_count(blob),
                                 out=buf[1:].view(n, h, w))
    return out.cpu().numpy(), status.cpu().tolist()


@pytest.mark.parametrize("entries", [2, 4, 16, 256])
@pytest.mark.parametrize("w", [1, 9, 31, 854])
def test_palette_decode_equals_pillow(entries, w):
    rng = np.random.default_rng(entries + w)
    datas, want = [], []
    for i in range(3):
        idx = rng.integers(0, entries, (23, w)).astype(np.uint8)
        idx[:5] = 0
        datas.append(pillow_palette_png(idx, entries, transparency=0 if i == 1 else None))
        want.append(np.array(Image.open(io.BytesIO(datas[-1]))))
    got, status = _decode_index(datas)
    assert status == [0, 0, 0]
    assert np.array_equal(got, np.stack(want))


def test_palette_encode_equals_the_restatement_and_decodes_back():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(9)
    for (n, h, w), entries in [((1, 1, 1), 1), ((3, 37, 53), 4), ((2, 480, 854), 256), ((1, 7, 17000), 3)]:
        idx = rng.integers(0, entries, (n, h, w)).astype(np.uint8)
        idx[:, : h // 2] = 0
        pal = davis_palette(entries)
        buf = torch.empty(n * h * w + 1, dtype=torch.uint8, device="cuda")
        src = buf[1:].view(n, h, w)
        src.copy_(torch.from_numpy(idx))
        out, lengths = ops.encode_png(src, palette=pal)
        assert out.shape[1] == ops.png_max_bytes(h, w, pal) == ops.png_max_bytes(h, w) + 12 + 3 * entries
        files = [bytes(out[i, :int(lengths[i])].cpu().numpy()) for i in range(n)]
        for i in range(n):
            assert files[i] == PP.encode(idx[i], pal)
            im = Image.open(io.BytesIO(files[i]))
            assert im.mode == "P" and np.array_equal(np.array(im), idx[i])
            assert bytes(im.getpalette())[:3 * entries] == pal
        got, status = _decode_index(files)
        assert status == [0] * n and np.array_equal(got, idx)
        # without a palette: byte-identical to the grayscale restatement, as before
        out0, len0 = ops.encode_png(src)
        assert out0.shape[1] == ops.png_max_bytes(h, w)
        for i in range(n):
            assert bytes(out0[i, :int(len0[i])].cpu().numpy()) == P.encode(idx[i])
    with pytest.raises(ValueError):
        ops.encode_png(src, palette=b"\0" * 4)


# ---- segmenter, scorer, online loop -----------------------------------------------------------------------------------

def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


@pytest.mark.parametrize("opts", [dict(), dict(score=True), dict(score=True, encode="png")])
def test_segmenter_labels_equal_the_merge_of_each_net(opts):
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    nets = [_he_net(seed=1).cuda().eval(), _he_net(seed=2).cuda().eval()]
    rng = np.random.default_rng(3)
    frames = [torch.from_numpy(rng.integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)).pin_memory() for _ in range(4)]
    gts = [torch.from_numpy(rng.integers(0, 3, (2, 40, 56)).astype(np.uint8)).pin_memory() for _ in range(4)]
    for g in gts:
        g[:, :, 20:22] = 255
    score = opts.get("score", False)
    items = list(zip(frames, gts)) if score else frames
    logits = []
    for net in nets:
        seg = SequenceSegmenter(net, output="logits", depth=2, frames="bgr8")
        logits.append([r.clone() for r in seg(iter(frames))])
    pal = davis_palette(3) if opts.get("encode") else None
    seg = SequenceSegmenter(nets=nets, output="labels", depth=2, frames="bgr8", palette=pal, **opts)
    got = [[bytes(f) for f in r] if pal else r.clone() for r in seg(iter(items))]
    assert len(got) == 4
    counts = []
    for i, res in enumerate(got):
        want = ops.merge_objects([logits[0][i].cuda(), logits[1][i].cuda()])
        if pal:
            assert res == [PP.encode(m, pal) for m in want.cpu().numpy()]
        else:
            assert res.shape == (2, 1, 40, 56) and torch.equal(res[:, 0], want.cpu())
        if score:
            counts.append(ops.davis_measures_objects(want, gts[i].cuda(), 2).cpu())
    if score:
        assert torch.equal(seg.frame_counts(), torch.cat(counts))
    with pytest.raises(ValueError):
        SequenceSegmenter(nets=nets, output="labels", frames="bgr8", input_res=(24, 32))
    with pytest.raises(ValueError):
        SequenceSegmenter(nets=nets, output="labels", frames="bgr8", overlay="jpeg")
    with pytest.raises(ValueError):
        SequenceSegmenter(nets=nets, output="mask", frames="bgr8")


SEQS = {"s1": 2, "s2": 3}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """A DAVIS-2017 layout: JPEG frames (cv2), palette annotations with a void band (Pillow), ImageSets/2017/val.txt."""
    cv2 = pytest.importorskip("cv2")
    root = tmp_path_factory.mktemp("davis2017")
    rng = np.random.default_rng(21)
    for s, (seq, k) in enumerate(SEQS.items()):
        os.makedirs(root / "JPEGImages" / "480p" / seq)
        os.makedirs(root / "Annotations" / "480p" / seq)
        for f in range(5):
            img = rng.integers(0, 256, (40, 56, 3), dtype=np.uint8)
            cv2.imwrite(str(root / "JPEGImages" / "480p" / seq / f"{f:05d}.jpg"), img)
            _, gt = _scene("void" if f % 2 else "blobs", 40, 56, k, seed=100 * s + f)
            if f == 0:
                gt[gt == 255] = 0
                gt[0, 0] = k                                     # every object id present in the first frame
            im = Image.fromarray(gt, "P")
            im.putpalette(davis_palette(256))
            im.save(str(root / "Annotations" / "480p" / seq / f"{f:05d}.png"))
    os.makedirs(root / "ImageSets" / "2017")
    (root / "ImageSets" / "2017" / "val.txt").write_text("\n".join(SEQS) + "\n")
    return str(root)


def _restated_scores(results, root, seq, k):
    stems = sorted(x[:-4] for x in os.listdir(os.path.join(root, "Annotations", "480p", seq)))
    counts = []
    for s in stems:
        res = np.array(Image.open(os.path.join(results, seq, s + ".png")))
        ann = np.array(Image.open(os.path.join(root, "Annotations", "480p", seq, s + ".png")))
        counts.append(O.object_counts(res, ann, k, M.bound_pix(*ann.shape)))
    return np.array(counts)


@pytest.mark.parametrize("decode", ["device", "host"])
def test_score_results_2017_equals_the_restatement(tmp_path, tree, decode):
    from osvos_pytorch_b200 import davis, evaluation
    rng = np.random.default_rng(5)
    for seq in SEQS:
        os.makedirs(tmp_path / seq)
        for f in range(5):
            lab = rng.integers(0, SEQS[seq] + 2, (40, 56)).astype(np.uint8)
            if f % 2:                                             # another method's grayscale files score the same
                Image.fromarray(lab, "L").save(str(tmp_path / seq / f"{f:05d}.png"))
            else:
                im = Image.fromarray(lab, "P")
                im.putpalette(davis_palette(8))
                im.save(str(tmp_path / seq / f"{f:05d}.png"))
    res = evaluation.score_results(str(tmp_path), tree, device="cuda", decode=decode, davis="2017", batch=2)
    assert list(res["sequences"]) == list(SEQS) and res["frames"] == 10
    stats = []
    for seq, k in SEQS.items():
        want = _restated_scores(str(tmp_path), tree, seq, k)
        r = res["sequences"][seq]
        assert np.array_equal(np.array(r["counts"]), want)
        for j in range(k):
            jf = [M.j_and_f(c) for c in want[:, j]]
            assert np.allclose(r["objects"][j + 1]["J"], [x for x, _ in jf])
            stats.append(M.statistics([x for x, _ in jf])[0])
    assert res["dataset"]["objects"] == 5 and np.isclose(res["dataset"]["J"]["M"], np.mean(stats))
    ds = davis.DAVIS2017Frames("val", tree)
    assert len(ds) == 10 and ds.n_objects == SEQS and ds.palettes["s1"] == davis_palette(256)
    item = ds[1]
    assert item["n_objects"] == 2 and item["image"].shape == (40, 56, 3)
    assert np.array_equal(item["gt"], np.array(Image.open(os.path.join(tree, "Annotations/480p/s1/00001.png"))))


@pytest.mark.parametrize("extra", [["--encode", "device", "--decode", "device"], []])
def test_online_2017_scores_equal_score_results(tmp_path, tree, monkeypatch, extra):
    import train_online
    from osvos_pytorch_b200 import evaluation
    seq = "s2"
    torch.save(_he_net(seed=3).state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    train_online.main(["--seq-name", seq, "--iters", "10", "--n-ave-grad", "5", "--lr", "1e-10", "--seed", "1",
                       "--parent-epoch", "1", "--loader", "native", "--davis", "2017", "--evaluate"] + extra)
    gc.collect()
    results = tmp_path / "Results"
    files = sorted(os.listdir(results / seq))
    assert files == [f"{f:05d}.png" for f in range(5)]
    for f in files:
        im = Image.open(results / seq / f)
        assert im.mode == "P" and bytes(im.getpalette())[:6] == davis_palette(2)
    assert sorted(x for x in os.listdir(tmp_path) if x.endswith(".pth")) == \
        ["parent_epoch-0.pth"] + [f"{seq}_object-{k}_epoch-9.pth" for k in range(1, 4)]
    written = json.load(open(results / f"{seq}_scores.json"))
    scored = evaluation.score_results(str(results), tree, sequences=[seq], device="cuda", davis="2017")
    assert written["n_objects"] == 3 and written["counts"] == scored["sequences"][seq]["counts"]
    for k in range(1, 4):
        assert written["objects"][str(k)]["J"] == scored["sequences"][seq]["objects"][k]["J"]
        assert written["objects"][str(k)]["F"] == scored["sequences"][seq]["objects"][k]["F"]

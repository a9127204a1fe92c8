"""DAVIS-2016 J and F on the GPU (csrc/measures.cu, ops.davis_measures): the kernel's integer counts equal the numpy
oracle's (tests/davis_measures_ref.py) exactly, scoring inside SequenceSegmenter leaves its outputs unchanged, and
``train_online.py --evaluate`` writes the oracle's scores without changing the PNGs."""
import json
import os

import numpy as np
import pytest
import torch

import davis_fixture
import davis_measures_ref as ref

pytestmark = pytest.mark.gpu

MAX_R = 31


def blobs(rng, h, w, k=4):
    y, x = np.mgrid[0:h, 0:w]
    m = np.zeros((h, w), dtype=bool)
    for _ in range(k):
        cy, cx = rng.uniform(-0.1, 1.1) * h, rng.uniform(-0.1, 1.1) * w
        ry, rx = rng.uniform(0.05, 0.4) * h + 1, rng.uniform(0.05, 0.4) * w + 1
        m |= ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 <= 1
    return m


def speckle(rng, h, w, p=0.5):
    return rng.random((h, w)) < p


def edges(h, w):
    """Foreground along every edge and in every corner, with a hole in the middle."""
    m = np.zeros((h, w), dtype=bool)
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = True
    m[: max(1, h // 4), : max(1, w // 4)] = True
    m[-max(1, h // 5):, -max(1, w // 3):] = True
    return m


def to_logits(rng, m):
    """fp32 logits with sign(m): foreground strictly positive, background negative or exactly ±0.0."""
    mag = rng.uniform(1e-6, 5.0, m.shape).astype(np.float32)
    bg = -mag
    z = rng.random(m.shape)
    bg[z < 0.15] = 0.0
    bg[(z >= 0.15) & (z < 0.3)] = -0.0
    fg = mag
    fg[rng.random(m.shape) < 0.05] = np.float32(1e-38)
    return np.where(m, fg, bg).astype(np.float32)


def to_u8(rng, m):
    """Annotation bytes: foreground any of 1, 128, 255."""
    return np.where(m, rng.choice(np.array([1, 128, 255], dtype=np.uint8), m.shape), 0).astype(np.uint8)


def misaligned(a, offset):
    buf = torch.empty(a.size + 16, dtype=torch.uint8, device="cuda")
    out = buf[offset:offset + a.size].view(a.shape)
    out.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return out


def run(logits, gts, r=None, offset=0):
    from osvos_pytorch_b200 import ops
    lg = torch.from_numpy(np.stack(logits)).cuda()
    gt = misaligned(np.stack(gts), offset) if offset else torch.from_numpy(np.stack(gts)).cuda()
    got = ops.davis_measures(lg, gt, r=r).cpu().tolist()
    want = [ref.counts(l, g, r) for l, g in zip(logits, gts)]
    return got, want


def frame_set(rng, h, w):
    empty, full = np.zeros((h, w), bool), np.ones((h, w), bool)
    preds = [blobs(rng, h, w), speckle(rng, h, w), empty, full, edges(h, w), blobs(rng, h, w), empty, speckle(rng, h, w, 0.1)]
    gts = [blobs(rng, h, w), blobs(rng, h, w), blobs(rng, h, w), full, edges(h, w), empty, empty, speckle(rng, h, w, 0.9)]
    return preds, gts


@pytest.mark.parametrize("w", [1, 31, 32, 33, 45, 854])
@pytest.mark.parametrize("h", [1, 5, 40])
def test_counts_equal_the_oracle_across_shapes(h, w):
    rng = np.random.default_rng(h * 1000 + w)
    preds, gts = frame_set(rng, h, w)
    logits = [to_logits(rng, p) for p in preds]
    masks = [to_u8(rng, g) for g in gts]
    for r in (None, 1, 4, 8):
        for offset in (0, 1, 3):
            got, want = run(logits, masks, r=r, offset=offset)
            assert got == want, (h, w, r, offset)


def test_counts_equal_the_oracle_at_every_radius():
    from osvos_pytorch_b200 import _native as nat
    assert nat.DAVIS_MAX_RADIUS == MAX_R
    rng = np.random.default_rng(7)
    h, w = 70, 97
    preds = [blobs(rng, h, w), speckle(rng, h, w, 0.02), edges(h, w)]
    gts = [blobs(rng, h, w), blobs(rng, h, w, 9), speckle(rng, h, w, 0.03)]
    logits = [to_logits(rng, p) for p in preds]
    masks = [to_u8(rng, g) for g in gts]
    for r in range(1, MAX_R + 1):
        got, want = run(logits, masks, r=r, offset=r % 4)
        assert got == want, r


def test_signed_zero_logits_are_background():
    from osvos_pytorch_b200 import ops
    lg = torch.tensor([[[0.0, -0.0, 1e-45, -1e-45]]], dtype=torch.float32, device="cuda")
    gt = torch.tensor([[[255, 255, 255, 0]]], dtype=torch.uint8, device="cuda")
    assert ops.davis_measures(lg, gt, r=1).cpu().tolist() == [ref.counts(lg[0].cpu().numpy(), gt[0].cpu().numpy(), 1)]
    assert ops.davis_measures(lg, gt, r=1)[0, :2].tolist() == [1, 3]


@pytest.mark.parametrize("n,h,w", [(12, 480, 854), (1, 1080, 1920)])
def test_counts_equal_the_oracle_at_the_served_sizes(n, h, w):
    rng = np.random.default_rng(n)
    preds = [blobs(rng, h, w, 6) if k % 3 else speckle(rng, h, w, 0.002) | blobs(rng, h, w) for k in range(n)]
    gts = [blobs(rng, h, w, 6) for _ in range(n)]
    logits = [to_logits(rng, p) for p in preds]
    masks = [to_u8(rng, g) for g in gts]
    got, want = run(logits, masks, offset=1 if n > 1 else 0)
    assert got == want
    from osvos_pytorch_b200 import ops
    lg = torch.from_numpy(np.stack(logits)).cuda()[:, None]            # [N,1,H,W] as the network returns it
    assert ops.davis_measures(lg, torch.from_numpy(np.stack(masks)).cuda()).cpu().tolist() == want


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


@pytest.mark.parametrize("frames", ["nchw_f32", "bgr8"])
def test_sequence_segmenter_scores_without_changing_outputs(frames):
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net(seed=1).cuda().eval()
    rng = np.random.default_rng(3)
    g = torch.Generator().manual_seed(11)
    n, h, w, count = 2, 48, 67, 6
    raw = [torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8) for _ in range(count)]
    mean = np.array(ops.MEANVAL, dtype=np.float32)
    if frames == "bgr8":
        inputs = [f.pin_memory() for f in raw]
    else:
        inputs = [torch.from_numpy(np.subtract(f.numpy().astype(np.float32), mean).transpose(0, 3, 1, 2).copy()).pin_memory()
                  for f in raw]
    gts = [torch.from_numpy(np.stack([to_u8(rng, blobs(rng, h, w)) for _ in range(n)])).pin_memory() for _ in range(count)]
    for output in ("logits", "bytescale"):
        plain = [o.clone() for o in SequenceSegmenter(net, output=output, frames=frames)(iter(inputs))]
        seg = SequenceSegmenter(net, output=output, frames=frames, score=True)
        scored = [o.clone() for o in seg(zip(inputs, gts))]
        assert len(plain) == len(scored) == count
        for a, b in zip(plain, scored):
            assert torch.equal(a, b), output
        counts = seg.frame_counts()
        assert counts.shape == (count * n, 6) and counts.dtype == torch.int32
        if output == "logits":
            want = ops.davis_measures(torch.cat(plain).cuda(), torch.cat(gts).cuda()).cpu()
            assert torch.equal(counts, want)
            assert counts.tolist() == [ref.counts(l[0].numpy(), m.numpy()) for l, m in zip(torch.cat(plain), torch.cat(gts))]
            logit_counts = counts
        else:
            assert torch.equal(counts, logit_counts)


def test_online_evaluate_writes_the_oracle_scores(tmp_path, monkeypatch):
    """``train_online.py --loader native --evaluate`` on the fixture tree: the JSON's per-frame counts, J and F are the
    oracle's on logits recomputed from the saved checkpoint, and the PNGs equal those of a run without --evaluate."""
    pytest.importorskip("cv2")
    import train_online
    from osvos_pytorch_b200 import davis, evaluation, ops
    tree = davis_fixture.write_tree(davis_fixture.load(), tmp_path / "davis")
    save = tmp_path / "models"
    save.mkdir()
    torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    iters = 4
    common = ["--seq-name", "aa", "--iters", str(iters), "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "5",
              "--parent-epoch", "1", "--log-every", "1", "--loader", "native"]
    out_dir = save / "Results" / "aa"
    train_online.main(common + ["--no-save"])
    plain = {f: (out_dir / f).read_bytes() for f in sorted(os.listdir(out_dir))}
    assert sorted(plain) == ["00000.png", "00001.png", "00002.png"]
    assert not (save / "Results" / "aa_scores.json").exists()
    train_online.main(common + ["--evaluate"])
    assert {f: (out_dir / f).read_bytes() for f in sorted(os.listdir(out_dir))} == plain
    res = json.loads((save / "Results" / "aa_scores.json").read_text())

    net = _he_net(seed=0)
    net.load_state_dict(torch.load(save / f"aa_epoch-{iters - 1}.pth", map_location="cpu"))
    net = net.cuda().eval()
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="aa", all_annotations=True)
    want = []
    with torch.no_grad():
        for i in range(len(d)):
            it = d[i]
            img = ops.image_from_bgr8(torch.from_numpy(it["image"])[None].cuda())
            logit = net(img)[-1][0, 0].cpu().numpy()
            want.append(ref.counts(logit, it["gt"]))
    assert res["sequence"] == "aa" and res["counts"] == want
    jf = [ref.j_and_f(c) for c in want]
    assert res["J"] == [j for j, _ in jf] and res["F"] == [f for _, f in jf]
    st = evaluation.statistics([j for j, _ in jf])
    assert res["statistics"]["J"] == pytest.approx(st, nan_ok=True)

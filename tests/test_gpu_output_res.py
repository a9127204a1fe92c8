"""Segmentations at the annotations' stored size (DESIGN.md §18): the fp32 resize on the GPU (csrc/resize.cu
osvos_resize_f32, ops.resize_f32) against the numpy restatement of Pillow's 'F' resize (tests/resize_f32_ref.py, itself
checked against Pillow in test_resize_f32.py), and ``output_res="stored"`` through SequenceSegmenter, DeviceFrames
and both scripts."""
import gc
import json
import os
import random

import numpy as np
import pytest
import torch

import davis_fixture
import resize_f32_ref

pytestmark = pytest.mark.gpu

SHAPES = [((240, 427), (480, 854)), ((120, 214), (480, 854)), ((360, 640), (480, 854)), ((480, 854), (240, 427)),
          ((7, 9), (30, 41)), ((30, 54), (1080, 1920)), ((240, 427), (480, 427)), ((240, 427), (240, 854)),
          ((33, 45), (1, 1)), ((33, 45), (1, 45)), ((33, 45), (33, 1)), ((1, 1), (5, 7)), ((31, 29), (31, 29)),
          ((5, 70), (64, 3)), ((97, 131), (40, 300))]


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    pytest.importorskip("cv2")                            # DAVIS2016Frames decodes with cv2
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def _maps(rng, n, shape, span=30.0):
    """Logit-like fp32 maps [n,H,W]: smooth structure of both signs plus noise."""
    h, w = shape
    yy, xx = np.meshgrid(np.linspace(-1, 1, h), np.linspace(-1, 1, w), indexing="ij")
    out = [span * np.sin(3 * xx + rng.uniform(0, 6)) * np.cos(2 * yy + rng.uniform(0, 6)) + rng.normal(0, span / 10, (h, w))
           for _ in range(n)]
    return np.stack(out).astype(np.float32)


def _check(x, dst):
    """ops.resize_f32 in both layouts equals the restatement bit for bit."""
    from osvos_pytorch_b200 import ops
    want = resize_f32_ref.resize(x, dst).view(np.uint32)
    xd = torch.from_numpy(x).cuda()
    got3 = ops.resize_f32(xd, dst)
    got4 = ops.resize_f32(xd[:, None], dst)
    assert got3.shape == (x.shape[0],) + tuple(dst) and got4.shape == (x.shape[0], 1) + tuple(dst)
    assert np.array_equal(got3.cpu().numpy().view(np.uint32), want)
    assert np.array_equal(got4[:, 0].cpu().numpy().view(np.uint32), want)


@pytest.mark.parametrize("src,dst", SHAPES)
def test_kernel_is_the_restatement(src, dst):
    rng = np.random.default_rng(list(src + dst))
    for n in (1, 3, 12):
        if n == 12 and dst[0] * dst[1] > 480 * 854:
            continue                                     # keeps the CPU restatement's memory small
        _check(_maps(rng, n, src), dst)


def test_kernel_is_the_restatement_on_random_shapes():
    rng = np.random.default_rng(23)
    for _ in range(60):
        src = tuple(int(v) for v in rng.integers(1, 300, 2))
        dst = tuple(int(v) for v in rng.integers(1, 300, 2))
        _check(_maps(rng, int(rng.choice([1, 3, 12])), src), dst)


def test_large_values_and_an_output_view():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(8)
    x = (rng.uniform(-1e4, 1e4, (3, 50, 30)) * 10.0 ** rng.integers(-6, 1, (3, 50, 30))).astype(np.float32)
    buf = torch.zeros(3 * 17 * 77 + 1, dtype=torch.float32, device="cuda")
    out = buf[1:].view(3, 17, 77)                         # 4-byte but not 16-byte aligned
    ops.resize_f32(torch.from_numpy(x).cuda(), (17, 77), out=out)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), resize_f32_ref.resize(x, (17, 77)).view(np.uint32))


def test_identity_is_a_copy():
    from osvos_pytorch_b200 import ops
    x = torch.randn(3, 1, 31, 29, device="cuda")
    before = ops.KERNEL_LAUNCHES[0]
    y = ops.resize_f32(x, (31, 29))
    assert ops.KERNEL_LAUNCHES[0] - before == 1
    assert y.data_ptr() != x.data_ptr() and torch.equal(y, x)


def test_launch_count():
    from osvos_pytorch_b200 import ops
    x = torch.randn(2, 1, 24, 40, device="cuda")
    for size, launches in (((48, 80), 3), ((24, 80), 2), ((48, 40), 2)):
        before = ops.KERNEL_LAUNCHES[0]
        ops.resize_f32(x, size)
        assert ops.KERNEL_LAUNCHES[0] - before == launches, size


def test_error_paths():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import ops
    x = torch.zeros(2, 1, 8, 8, device="cuda")
    for bad in (x.half(), x.to(torch.uint8), x.double(), torch.zeros(2, 2, 8, 8, device="cuda"),
                torch.zeros(8, 8, device="cuda"), torch.zeros(1, 1, 1, 8, 8, device="cuda")):
        with pytest.raises(ValueError, match="fp32"):
            ops.resize_f32(bad, (4, 4))
    for size in ((0, 4), (4, 0), (32768, 4), (4, 32768), (-1, 4)):
        with pytest.raises(ValueError, match="cannot resize"):
            ops.resize_f32(x, size)
    with pytest.raises(ValueError, match="cannot resize"):
        ops.resize_f32(torch.zeros(0, 1, 8, 8, device="cuda"), (4, 4))
    for out in (torch.zeros(2, 1, 4, 5, device="cuda"), torch.zeros(2, 4, 4, device="cuda"),
                torch.zeros(2, 1, 4, 4, device="cuda", dtype=torch.float64), torch.zeros(2, 1, 4, 8, device="cuda")[..., ::2]):
        with pytest.raises(ValueError, match="out must be"):
            ops.resize_f32(x, (4, 4), out=out)
    q = nat.load().osvos_resize_f32_workspace_bytes
    assert q(0, 8, 8, 4, 4) == 0 and q(65536, 8, 8, 4, 4) == 0 and q(1, 8, 8, 0, 4) == 0 and q(1, 8, 40000, 4, 4) == 0
    assert q(1, 8, 8, 4, 4) > 0


@pytest.mark.parametrize("src", [(240, 427), (120, 214), (360, 640)])
def test_upscale_is_close_to_torch_bilinear(src):
    """A sanity bound only: torch's bilinear (align_corners=False) has no antialias and a different operation order."""
    import torch.nn.functional as F
    from osvos_pytorch_b200 import ops
    x = torch.from_numpy(_maps(np.random.default_rng(src[0]), 2, src)).cuda()[:, None]
    got = ops.resize_f32(x, (480, 854))
    want = F.interpolate(x, size=(480, 854), mode="bilinear", align_corners=False)
    assert float((got - want).abs().max()) <= 1e-4 * float(x.abs().max())


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


def _sequence(tree):
    """Five collated 33x45 frames: sequence aa's three and two of them flipped, so a depth-2 ring reuses its slots."""
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True, seq_name=None)
    items = [d[i] for i in range(3)]
    for it in items[:2]:
        items.append(dict(it, image=np.ascontiguousarray(it["image"][:, ::-1]), gt=np.ascontiguousarray(it["gt"][:, ::-1])))
    return [davis.collate([it]) for it in items]


def _frames(batches, score=True):
    from osvos_pytorch_b200 import davis
    for b in batches:
        img, gt = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
        yield (img, gt) if score else img


def test_sequence_segmenter_stored(tree):
    """Each result is logits_to_u8(resize_f32(fused)) of a per-frame forward at the network resolution, and each count
    row is davis_measures of that upsampled map against the original annotation."""
    from osvos_pytorch_b200 import davis, ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    batches = _sequence(tree)
    res, dev = (24, 32), torch.device("cuda")
    for output in ("bytescale", "logits"):
        seg = SequenceSegmenter(net, output=output, depth=2, frames="bgr8", score=True, input_res=res,
                                output_res="stored")
        got = [r.clone() for r in seg(_frames(batches))]
        counts = seg.frame_counts()
        assert len(got) == 5 and counts.shape == (5, 6)
        assert seg.d2h_bytes_per_frame == 33 * 45 * (4 if output == "logits" else 1)
        for i, b in enumerate(batches):
            with torch.no_grad():
                fused = net(davis.to_device(b, dev, input_res=res)["image"])[-1]
            up = ops.resize_f32(fused, (33, 45))
            assert got[i].shape == (1, 1, 33, 45)
            want = up if output == "logits" else ops.logits_to_u8(up, output)
            assert torch.equal(got[i], want.cpu()), (output, i)
            _, gt_u8, _ = davis.upload(b, dev)
            assert torch.equal(counts[i:i + 1], ops.davis_measures(up, gt_u8).cpu()), (output, i)
        assert counts[:, 1].sum() > 0
    with pytest.raises(ValueError, match="output_res"):
        SequenceSegmenter(net, frames="bgr8", input_res=res, output_res="annotation")


def test_stored_without_input_res_is_the_default(tree, monkeypatch):
    """Without input_res, output_res='stored' gives the default's bytes and counts and never resizes."""
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net(seed=2).cuda().eval()
    batches = _sequence(tree)
    runs = []
    for output_res in ("network", "stored"):
        seg = SequenceSegmenter(net, output="bytescale", depth=2, frames="bgr8", score=True, output_res=output_res)
        runs.append(([r.clone() for r in seg(_frames(batches))], seg.frame_counts()))

    def refuse(*args, **kwargs):
        raise AssertionError("resize_f32 called without input_res")
    monkeypatch.setattr(ops, "resize_f32", refuse)
    seg = SequenceSegmenter(net, output="bytescale", depth=2, frames="bgr8", score=True, output_res="stored")
    runs.append(([r.clone() for r in seg(_frames(batches))], seg.frame_counts()))
    for got, counts in runs[1:]:
        assert len(got) == 5 and all(torch.equal(a, b) for a, b in zip(got, runs[0][0]))
        assert torch.equal(counts, runs[0][1])


def test_device_frames_keep_stored_gt(tree):
    from osvos_pytorch_b200 import davis
    dev = torch.device("cuda")
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)             # sequences at 33x45 and 97x131
    plain = davis.DeviceFrames(d, dev, input_res=(30, 40))
    store = davis.DeviceFrames(d, dev, input_res=(30, 40), keep_stored_gt=True)
    assert [g["size"] for g in store.groups] == [(30, 40)]
    assert sorted(g["size"] for g in store.stored_groups) == [(33, 45), (97, 131)]
    assert store.nbytes == plain.nbytes + 3 * 33 * 45 + 2 * 97 * 131
    for i in range(len(d)):
        got, ref = store.ingest(i), plain.ingest(i)
        assert "gt_u8_stored" not in ref
        assert torch.equal(got["image"], ref["image"]) and torch.equal(got["gt_u8"], ref["gt_u8"])
        assert np.array_equal(got["gt_u8_stored"][0].cpu().numpy(), d[i]["gt"]), i
    assert "gt_u8_stored" not in davis.DeviceFrames(d, dev, keep_stored_gt=True).ingest(0)     # no input_res


def test_online_output_res_stored(tree, tmp_path, monkeypatch):
    """``train_online.py --input-res 40 56 --output-res stored --evaluate`` writes PNGs at the sequence's stored size,
    and its scores are those of the saved network's fused maps, upsampled and scored with ops directly."""
    from PIL import Image
    import train_online
    from osvos_pytorch_b200 import davis, ops
    from osvos_pytorch_b200.evaluation import SequenceScores
    save = tmp_path / "models"
    save.mkdir()
    torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    hist = train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                              "--parent-epoch", "1", "--log-every", "1", "--loader", "native", "--input-res", "40", "56",
                              "--output-res", "stored", "--evaluate"])
    assert len(hist) == 4 and all(np.isfinite(hist))
    pngs = sorted(os.listdir(save / "Results" / "cc"))
    assert pngs == ["00000.png", "00001.png"]
    with open(save / "Results" / "cc_scores.json") as f:
        got = json.load(f)
    assert got["network_res"] == [40, 56] and got["scored_res"] == [97, 131]
    net = _he_net().cuda().eval()
    net.load_state_dict(torch.load(save / "cc_epoch-3.pth", map_location="cuda"))
    dev = torch.device("cuda")
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="cc", all_annotations=True)
    scores = SequenceScores()
    for i in range(len(d)):
        b = davis.collate([d[i]])
        with torch.no_grad():
            fused = net(davis.to_device(b, dev, input_res=(40, 56))["image"])[-1]
        up = ops.resize_f32(fused, (97, 131))
        png = np.asarray(Image.open(save / "Results" / "cc" / pngs[i]))
        assert png.shape == (97, 131)
        assert np.array_equal(png, ops.logits_to_u8(up, "bytescale")[0, 0].cpu().numpy()), i
        _, gt_u8, _ = davis.upload(b, dev)
        scores.add(ops.davis_measures(up, gt_u8))
    want = scores.result()
    for key in ("J", "F", "counts", "statistics"):
        np.testing.assert_equal(got[key], want[key])


def _parent_val(argv, save, monkeypatch, capsys):
    """One seeded train_parent.main run -> (its J/F lines, every (logits shape, gt shape, counts) it scored)."""
    import train_parent
    from osvos_pytorch_b200 import ops
    scored, measures = [], ops.davis_measures

    def recording(logits, gt_u8, *args, **kw):
        out = measures(logits, gt_u8, *args, **kw)
        scored.append((tuple(logits.shape), tuple(gt_u8.shape), out.cpu()))
        return out
    monkeypatch.setattr(ops, "davis_measures", recording)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    torch.manual_seed(11)
    random.seed(11)
    train_parent.main(argv)
    monkeypatch.setattr(ops, "davis_measures", measures)
    gc.collect()                                        # free the run's captured graphs here (test_gpu_device_frames)
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("***Testing") and " J M/O/D" in ln]
    return lines, scored


def test_parent_val_measures_stored(tree, tmp_path, monkeypatch, capsys):
    """--val-measures --input-res --output-res stored scores the upsampled fused map against the stored annotations,
    and the streaming and --cache device runs print identical J/F lines from identical counts."""
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    argv = ["--loader", "native", "--pretrained", "0", "--epochs", "1", "--snapshot", "1", "--test-interval", "1",
            "--n-ave-grad", "1", "--workers", "0", "--val-measures", "--lr", "1e-7", "--deterministic",
            "--input-res", "30", "40", "--output-res", "stored"]
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        streamed, s_scored = _parent_val(argv, tmp_path / "streamed", monkeypatch, capsys)
        cached, c_scored = _parent_val(argv + ["--cache", "device"], tmp_path / "cached", monkeypatch, capsys)
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    assert len(streamed) == 1 and cached == streamed and streamed[0].endswith("(1 sequences)")
    assert len(s_scored) == 2 and len(c_scored) == 2                   # the val split: bb's two 48x70 frames
    for (ls, gs, cs), (lc, gc_, cc) in zip(s_scored, c_scored):
        assert ls == lc == (1, 1, 48, 70) and gs == gc_ == (1, 48, 70)
        assert torch.equal(cs, cc)

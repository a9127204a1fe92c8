"""Reduced-resolution DAVIS-2017 on the device (DESIGN.md §27): ops.upsample_merge_objects against the composition it
fuses (ops.merge_objects of ops.resize_f32 of each map), SequenceSegmenter(nets=..., output="labels", input_res=...,
output_res="stored"), and train_online.py --davis 2017 --input-res --output-res stored against the numpy restatement
(tests/upsample_merge_ref.py) and score_results."""
import gc
import json
import os

import numpy as np
import pytest
import torch

import davis_objects_ref as O
import davis_measures_ref as M
import upsample_merge_ref as U
from png_palette_ref import davis_palette

pytestmark = pytest.mark.gpu


def _maps(k, n, h, w, seed, scale=1.0):
    """K fp32 [N,1,h,w] maps: ties across objects, ±0, NaN, one all-negative map, magnitudes 1e-6 .. 1e4."""
    rng = np.random.default_rng(seed)
    m = np.round(rng.normal(0, 2, (k, n, 1, h, w)) * 2) / 2
    m *= 10.0 ** rng.integers(-6, 5, (k, n, 1, h, w))
    flat = m.reshape(k, -1)
    sel = rng.random(flat.shape[1])
    flat[:, sel < 0.04] = np.nan
    flat[:, (sel >= 0.04) & (sel < 0.08)] = 0.0
    flat[:, (sel >= 0.08) & (sel < 0.12)] = -0.0
    flat[rng.integers(0, k), sel > 0.97] = np.nan                 # NaN in one map beside finite values
    if k > 1:
        flat[k - 1, sel > 0.8] = flat[0, sel > 0.8]               # exact ties between objects
        flat[1] = -np.abs(flat[1]) - 1.0                          # all negative
    return torch.from_numpy((m * scale).astype(np.float32)).cuda()


def _composed(maps, size):
    from osvos_pytorch_b200 import ops
    return ops.merge_objects([ops.resize_f32(m, size) for m in maps])


def _check(maps, size):
    from osvos_pytorch_b200 import ops
    want = _composed(maps, size)
    got = ops.upsample_merge_objects(maps, size)
    assert got.shape == want.shape and torch.equal(got, want)
    return want


SIZES = [((240, 427), (480, 854)), ((360, 640), (480, 854)), ((120, 214), (480, 854)), ((30, 54), (1080, 1920)),
         ((480, 854), (240, 427)), ((240, 427), (480, 427)), ((480, 427), (480, 854)), ((240, 427), (240, 427)),
         ((33, 45), (1, 1)), ((33, 45), (1, 45)), ((33, 45), (33, 1)), ((1, 1), (5, 7))]


@pytest.mark.parametrize("src,dst", SIZES)
@pytest.mark.parametrize("k", [1, 2, 3, 4, 17])
def test_equals_the_composition(src, dst, k):
    n = 3 if src[0] * dst[0] < 1e6 else 1
    _check(_maps(k, n, *src, seed=k + src[1] + dst[1]), dst)


@pytest.mark.parametrize("n", [1, 3, 12])
@pytest.mark.parametrize("k", [1, 4, 254])
def test_batches_and_object_counts(n, k):
    src, dst = ((240, 427), (480, 854)) if k * n <= 48 else ((24, 43), (48, 85))
    _check(_maps(k, n, *src, seed=n * 1000 + k), dst)


def test_254_objects_at_the_stored_size():
    _check(_maps(254, 1, 240, 427, seed=254), (480, 854))


def test_random_shape_pairs():
    rng = np.random.default_rng(40)
    for i in range(40):
        src = tuple(int(v) for v in rng.integers(1, 300, 2))
        dst = tuple(int(v) for v in rng.integers(1, 600, 2))
        if src[0] > 22 * dst[0]:
            dst = (src[0] // 22 + 1, dst[1])
        _check(_maps(int(rng.integers(1, 6)), int(rng.integers(1, 4)), *src, seed=i), dst)


def test_matches_the_numpy_restatement():
    maps = _maps(3, 2, 24, 43, seed=9)
    want = U.upsample_merge(maps.cpu().numpy(), (48, 85))
    assert np.array_equal(_check(maps, (48, 85)).cpu().numpy(), want.reshape(2, 48, 85))


def test_input_layouts_and_an_odd_output_offset():
    from osvos_pytorch_b200 import ops
    k, n, src, dst = 3, 2, (60, 107), (120, 214)
    dev = _maps(k, n, *src, seed=3)
    want = _composed(dev, dst)
    assert torch.equal(ops.upsample_merge_objects(dev, dst), want)                           # one [K,N,1,H,W] tensor
    assert torch.equal(ops.upsample_merge_objects(dev[:, :, 0], dst), want)                  # one [K,N,H,W] tensor
    flat = torch.empty(k * n * src[0] * src[1] + 1, dtype=torch.float32, device="cuda")
    parts = []                                                   # K separate tensors, 4- but not 16-byte aligned
    for j in range(k):
        t = flat[1 + j * n * src[0] * src[1]:1 + (j + 1) * n * src[0] * src[1]].view(n, *src)
        t.copy_(dev[j, :, 0])
        parts.append(t)
    buf = torch.empty(n * dst[0] * dst[1] + 1, dtype=torch.uint8, device="cuda")
    got = ops.upsample_merge_objects(parts, dst, out=buf[1:].view(n, 1, *dst))
    assert got.data_ptr() == buf.data_ptr() + 1 and torch.equal(got.view(n, *dst), want)


def test_launch_count():
    from osvos_pytorch_b200 import ops
    for k in (1, 2, 4, 17, 254):
        maps = [torch.zeros(1, 1, 12, 20, device="cuda")] * k
        before = ops.KERNEL_LAUNCHES[0]
        ops.upsample_merge_objects(maps, (24, 40))
        assert ops.KERNEL_LAUNCHES[0] - before == 2, k
        before = ops.KERNEL_LAUNCHES[0]
        ops.upsample_merge_objects(maps, (12, 20))
        assert ops.KERNEL_LAUNCHES[0] - before == 1, k


def test_launches_seen_by_the_profiler():
    """The two launches are the tables kernel and the tile kernel.  Late in a long process torch.profiler can record no
    device activity at all (tests/test_gpu_side_schedules.py's ``ran``), or lose a kernel record from a window
    (tests/test_gpu_conv_schedules.py's ``profiled``; here it was the window's first, the tables kernel).  So each
    window opens with a torch kernel of its own, and a window that records fewer than the two launches is retried, at
    most twice; one that stays blind is skipped.  The package's kernels in a window must be exactly these two."""
    from osvos_pytorch_b200 import ops
    maps = [torch.ones(2, 1, 12, 20, device="cuda")] * 4
    out = torch.empty(2, 24, 40, dtype=torch.uint8, device="cuda")
    first = torch.zeros(1, device="cuda")
    for _ in range(3):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            first.add_(1)
            ops.upsample_merge_objects(maps, (24, 40), out=out)
            torch.cuda.synchronize()
        records = [(ev.key, ev.count) for ev in prof.key_averages() if ev.device_type.name == "CUDA"]
        kernels = [(key, c) for key, c in records if "osvos::" in key]
        if sum(c for _, c in kernels) >= 2:
            break
    if not records:
        pytest.skip("torch.profiler recorded no device activity in this process")
    assert sum(c for _, c in kernels) == 2, records
    assert any("upsample_merge_objects_kernel" in key for key, _ in kernels), kernels
    assert any("resize_f32_tables_kernel" in key for key, _ in kernels), kernels


def test_refuses_bad_input():
    from osvos_pytorch_b200 import ops
    a = torch.zeros(1, 1, 4, 4, device="cuda")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.upsample_merge_objects([a.cpu()], (8, 8))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([], (8, 8))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([a, torch.zeros(1, 1, 4, 5, device="cuda")], (8, 8))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([a] * 255, (8, 8))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([a.double()], (8, 8))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([torch.zeros(1, 2, 4, 4, device="cuda")], (8, 8))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([a], (8, 8), out=torch.empty(1, 8, 9, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.upsample_merge_objects([a], (0, 8))
    with pytest.raises(ValueError, match="downscale"):
        ops.upsample_merge_objects([torch.zeros(1, 1, 1200, 4, device="cuda")], (50, 4))


# ---- segmenter and online loop ----------------------------------------------------------------------------------------

def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


SEQS = {"s1": 2, "s2": 3}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """A DAVIS-2017 layout: 40x56 JPEG frames (cv2), palette annotations with a void band (Pillow), ImageSets/2017."""
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    root = tmp_path_factory.mktemp("davis2017_res")
    rng = np.random.default_rng(27)
    yy, xx = np.mgrid[:40, :56]
    for seq, k in SEQS.items():
        os.makedirs(root / "JPEGImages" / "480p" / seq)
        os.makedirs(root / "Annotations" / "480p" / seq)
        for f in range(5):
            img = rng.integers(0, 256, (40, 56, 3), dtype=np.uint8)
            cv2.imwrite(str(root / "JPEGImages" / "480p" / seq / f"{f:05d}.jpg"), img)
            gt = np.zeros((40, 56), np.uint8)
            for j in range(1, k + 1):
                cy, cx = rng.integers(5, 35), rng.integers(5, 51)
                gt[((yy - cy) / rng.integers(4, 12)) ** 2 + ((xx - cx) / rng.integers(4, 16)) ** 2 <= 1] = j
            gt[0, :k] = np.arange(1, k + 1)                        # every object id present in every frame
            if f % 2:
                gt[:, 20:22] = 255                                 # void
            im = Image.fromarray(gt, "P")
            im.putpalette(davis_palette(256))
            im.save(str(root / "Annotations" / "480p" / seq / f"{f:05d}.png"))
    os.makedirs(root / "ImageSets" / "2017")
    (root / "ImageSets" / "2017" / "val.txt").write_text("\n".join(SEQS) + "\n")
    return str(root)


@pytest.mark.parametrize("frames", ["bgr8", "jpeg"])
def test_segmenter_stored_labels(tree, frames):
    """Each result is upsample_merge_objects of the nets' forwards on to_device(b, input_res), encoded as a palette
    PNG, and each count row is davis_measures_objects of those labels against the stored annotation."""
    import io
    from PIL import Image
    from osvos_pytorch_b200 import davis, ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    nets = [_he_net(seed=1).cuda().eval(), _he_net(seed=2).cuda().eval()]
    res, dev = (24, 32), torch.device("cuda")
    ds = davis.DAVIS2017Frames(db_root_dir=tree, seq_name="s1", all_annotations=True, decode="device" if frames == "jpeg"
                               else "host")
    batches = [davis.collate([ds[i]]) for i in range(len(ds))]

    def items():
        for b in batches:
            yield b if frames == "jpeg" else davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
    pal = davis_palette(3)
    for encode in ("png", None):
        seg = SequenceSegmenter(nets=nets, output="labels", depth=2, frames=frames, score=True, input_res=res,
                                output_res="stored", encode=encode, palette=pal if encode else None)
        got = [[bytes(f) for f in r] if encode else r.clone() for r in seg(items())]
        assert not hasattr(seg, "_dev_up")
        assert seg.d2h_bytes_per_frame == (ops.png_max_bytes(40, 56, pal) + 8 if encode else 40 * 56)
        counts = seg.frame_counts()
        assert len(got) == 5 and counts.shape == (5, 2, 6)
        for i, b in enumerate(batches):
            with torch.no_grad():
                x = davis.to_device(b, dev, input_res=res)["image"]
                fused = [net(x)[-1] for net in nets]
            want = ops.upsample_merge_objects(fused, (40, 56))
            if encode:
                im = Image.open(io.BytesIO(got[i][0]))
                assert im.mode == "P" and im.size == (56, 40) and bytes(im.getpalette())[:9] == pal
                assert np.array_equal(np.array(im), want[0].cpu().numpy()), i
            else:
                assert got[i].shape == (1, 1, 40, 56) and torch.equal(got[i][:, 0], want.cpu()), i
            _, gt_u8, _ = davis.upload(b, dev)
            assert gt_u8.shape == (1, 40, 56)
            assert torch.equal(counts[i:i + 1], ops.davis_measures_objects(want, gt_u8, 2).cpu()), i
        assert counts[:, :, 1].sum() > 0
    with pytest.raises(ValueError):
        SequenceSegmenter(nets=nets, output="labels", frames=frames, input_res=res, output_res="network")
    with pytest.raises(ValueError):
        SequenceSegmenter(nets=nets, output="labels", frames=frames, input_res=res, output_res="stored", overlay="jpeg")


def test_segmenter_stored_without_input_res_changes_nothing(tree):
    from osvos_pytorch_b200 import davis
    from osvos_pytorch_b200.inference import SequenceSegmenter
    nets = [_he_net(seed=1).cuda().eval(), _he_net(seed=2).cuda().eval()]
    ds = davis.DAVIS2017Frames(db_root_dir=tree, seq_name="s2", all_annotations=True)
    batches = [davis.collate([ds[i]]) for i in range(len(ds))]
    runs = []
    for output_res in ("network", "stored"):
        seg = SequenceSegmenter(nets=nets, output="labels", depth=2, frames="bgr8", score=True, output_res=output_res)
        got = [r.clone() for r in seg(davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
                                      for b in batches)]
        runs.append((got, seg.frame_counts()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert torch.equal(runs[0][1], runs[1][1])


@pytest.mark.parametrize("extra", [[], ["--ignore-void"], ["--decode", "device", "--encode", "device"]])
def test_online_2017_input_res_stored(tmp_path, tree, monkeypatch, extra):
    """train_online.py --davis 2017 --input-res 24 32 --output-res stored --evaluate: every object fine-tunes on 24x32
    samples, the files are 40x56 palette PNGs equal to the restatement of the saved nets' fused maps, and the scores
    JSON equals score_results of the written folder."""
    from PIL import Image
    import train_online
    from osvos_pytorch_b200 import davis, evaluation, training
    seq, k = "s2", SEQS["s2"]
    torch.save(_he_net(seed=3).state_dict(), tmp_path / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path))
    samples, finetune = [], training.online_finetune

    def recording(net, sample_fn, *args, **kwargs):
        def fn(it):
            s = sample_fn(it)
            samples.append((tuple(s["image"].shape), tuple(s["gt"].shape)))
            return s
        return finetune(net, fn, *args, **kwargs)
    monkeypatch.setattr(training, "online_finetune", recording)
    train_online.main(["--seq-name", seq, "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                       "--parent-epoch", "1", "--loader", "native", "--davis", "2017", "--input-res", "24", "32",
                       "--output-res", "stored", "--evaluate"] + extra)
    gc.collect()
    assert samples and all(s == ((1, 3, 24, 32), (1, 1, 24, 32)) for s in samples), set(samples)
    results = tmp_path / "Results"
    files = sorted(os.listdir(results / seq))
    assert files == [f"{f:05d}.png" for f in range(5)]
    nets = []
    for j in range(1, k + 1):
        net = _he_net().cuda().eval()
        net.load_state_dict(torch.load(tmp_path / f"{seq}_object-{j}_epoch-3.pth", map_location="cuda"))
        nets.append(net)
    ds = davis.DAVIS2017Frames(db_root_dir=tree, seq_name=seq, all_annotations=True)
    for i, f in enumerate(files):
        im = Image.open(results / seq / f)
        assert im.mode == "P" and im.size == (56, 40) and bytes(im.getpalette())[:6] == davis_palette(2)
        with torch.no_grad():
            x = davis.to_device(davis.collate([ds[i]]), torch.device("cuda"), input_res=(24, 32))["image"]
            fused = np.stack([net(x)[-1].cpu().numpy() for net in nets])
        assert np.array_equal(np.array(im), U.upsample_merge(fused, (40, 56))[0, 0]), f
    written = json.load(open(results / f"{seq}_scores.json"))
    assert written["network_res"] == [24, 32] and written["scored_res"] == [40, 56]
    scored = evaluation.score_results(str(results), tree, sequences=[seq], device="cuda", davis="2017")
    assert written["n_objects"] == k and written["counts"] == scored["sequences"][seq]["counts"]
    counts = np.array(written["counts"])
    for i, f in enumerate(files):                                  # and the restated counts of the written files
        ann = np.array(Image.open(os.path.join(tree, "Annotations", "480p", seq, f)))
        lab = np.array(Image.open(results / seq / f))
        assert np.array_equal(counts[i], np.array(O.object_counts(lab, ann, k, M.bound_pix(40, 56))))
    for j in range(1, k + 1):
        assert written["objects"][str(j)]["J"] == scored["sequences"][seq]["objects"][j]["J"]
        assert written["objects"][str(j)]["F"] == scored["sequences"][seq]["objects"][j]["F"]

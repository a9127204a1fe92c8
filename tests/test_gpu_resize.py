"""Frame resize on the GPU (csrc/resize.cu, ops.resize_u8) and the ``input_res`` paths built on it: the kernel against
the numpy restatement of Pillow (tests/resize_ref.py, itself checked against Pillow in test_resize.py), and the device
data path against the reference dataset with inputRes (tests/golden/reference_resize.npz)."""
import os
import random

import numpy as np
import pytest
import torch

import davis_fixture
import resize_ref

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_resize.npz")


@pytest.fixture(scope="module")
def fx():
    with np.load(GOLDEN, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def _res(fx, key):
    v, kind = fx[key], str(fx[key + ".kind"])
    return tuple(int(x) for x in v) if kind == "tuple" else int(v) if kind == "int" else float(v)


def _misaligned(t, offset):
    buf = torch.empty(t.numel() + 16, dtype=torch.uint8, device="cuda")
    out = buf[offset:offset + t.numel()].view(t.shape)
    out.copy_(t)
    return out


SHAPES = [((480, 854), (240, 427)), ((480, 854), (360, 640)), ((480, 854), (720, 1280)), ((480, 854), (480, 427)),
          ((1080, 1920), (480, 854)), ((48, 70), (33, 45)), ((37, 53), (100, 21)), ((31, 29), (31, 29)),
          ((33, 45), (1, 1)), ((33, 45), (1, 45)), ((33, 45), (33, 1)), ((5, 7), (64, 3)), ((97, 131), (48, 131)),
          ((2, 3), (3, 2)), ((480, 854), (17, 9))]


@pytest.mark.parametrize("src,dst", SHAPES)
@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_kernel_is_pillow(src, dst, mode):
    """Every channel count, batches of 1 and 3, sources 0 / 1 / 3 bytes past an aligned address."""
    from osvos_pytorch_b200 import ops
    g = torch.Generator().manual_seed(src[0] * 7 + dst[1])
    for c, n, offset in ((3, 1, 0), (1, 3, 1), (3, 3, 3)):
        x = torch.randint(0, 256, (n,) + src + ((3,) if c == 3 else ()), generator=g, dtype=torch.uint8)
        got = ops.resize_u8(_misaligned(x.cuda(), offset), dst, mode).cpu().numpy()
        assert got.shape == (n,) + dst + x.shape[3:]
        for i in range(n):
            assert np.array_equal(got[i], resize_ref.resize(x[i].numpy(), dst, mode)), (c, n, offset, i)


def test_kernel_is_pillow_on_random_shapes():
    """Random sizes, batches and channel counts, writing into an odd-offset output view."""
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(11)
    for _ in range(60):
        src = tuple(int(v) for v in rng.integers(1, 300, 2))
        dst = tuple(int(v) for v in rng.integers(1, 300, 2))
        n, c = int(rng.integers(1, 5)), int(rng.choice([1, 3]))
        mode = str(rng.choice(["bilinear", "nearest"]))
        x = rng.integers(0, 256, (n,) + src + ((3,) if c == 3 else ()), dtype=np.uint8)
        shape = (n,) + dst + x.shape[3:]
        out = _misaligned(torch.zeros(shape, dtype=torch.uint8, device="cuda"), int(rng.integers(0, 4)))
        ops.resize_u8(_misaligned(torch.from_numpy(x).cuda(), int(rng.integers(0, 4))), dst, mode, out=out)
        got = out.cpu().numpy()
        for i in range(n):
            assert np.array_equal(got[i], resize_ref.resize(x[i], dst, mode)), (src, dst, n, c, mode, i)


def test_to_device_matches_the_reference_input_res(fx, tree):
    """to_device(input_res=...) is make_img_gt_pair with inputRes + ToTensor, bit for bit, for a downscale, an upscale, a
    non-uniform size, an int percentage and a float fraction; an unannotated frame's mask is all zero at the resized
    size (the reference keeps it at the stored size)."""
    from osvos_pytorch_b200 import davis
    dev = torch.device("cuda")
    checked = nolabel = 0
    for r in range(int(fx["res.n"])):
        res = _res(fx, f"res.{r}")
        for kw in (dict(train=True), dict(train=False), dict(train=False, seq_name="aa")):
            d = davis.DAVIS2016Frames(db_root_dir=tree, **kw)
            for i in range(len(d)):
                it = d[i]
                key = d.img_list[i] + ("" if it["has_gt"] else ":nolabel")
                want_img, want_gt = fx[f"pair.{r}.{key}.image"], fx[f"pair.{r}.{key}.gt"]
                out = davis.to_device(davis.collate([it]), dev, input_res=res)
                got_img = out["image"][0].cpu().numpy().transpose(1, 2, 0)
                got_gt = out["gt"][0, 0].cpu().numpy()
                assert np.array_equal(got_img, want_img), (res, key)
                if it["has_gt"]:
                    assert np.array_equal(got_gt, want_gt), (res, key)
                else:
                    nolabel += 1
                    assert got_gt.shape == want_img.shape[:2] and not got_gt.any() and not want_gt.any()
                checked += 1
    assert checked > 30 and nolabel > 0


def test_augmented_samples_match_the_reference_transforms(fx, tree):
    """RandomHorizontalFlip + ScaleNRotate after the resize: binary masks bit-exact, images (and non-binary masks,
    cubic in float64 in the reference) within 3e-4, as test_gpu_davis.py holds the unresized path."""
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    for k in range(int(fx["aug.n"])):
        res = _res(fx, f"aug.{k}.res")
        flip, rot, sc = fx[f"aug.{k}.draws"]
        idx = int(fx[f"aug.{k}.index"])
        out = davis.to_device(davis.collate([d[idx]]), torch.device("cuda"),
                              augment=[(bool(flip), float(rot), float(sc))], input_res=res)
        got_img = out["image"][0].cpu().numpy().transpose(1, 2, 0)
        got_gt = out["gt"][0, 0].cpu().numpy()
        assert got_img.shape == fx[f"aug.{k}.image"].shape, k
        assert np.abs(got_img - fx[f"aug.{k}.image"]).max() <= 3e-4, k
        src = resize_ref.resize(d[idx]["gt"], got_gt.shape, "nearest")
        if np.isin(src, [0, src.max()]).all():
            assert np.array_equal(got_gt, fx[f"aug.{k}.gt"]), k
        else:
            assert np.abs(got_gt - fx[f"aug.{k}.gt"]).max() <= 3e-4, k


@pytest.mark.parametrize("res", [(40, 60), 50, 1.25])
def test_device_frames_match_to_device(tree, res):
    """A DeviceFrames store with input_res: frames of different stored sizes that resize to one size share a group,
    and its augmented batches and ingest are bit-identical to to_device(..., input_res) of the same items."""
    from osvos_pytorch_b200 import davis
    dev = torch.device("cuda")
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    store = davis.DeviceFrames(d, dev, input_res=res)
    sizes = {davis.imresize_size(res, *d[i]["gt"].shape) for i in range(len(d))}
    assert sorted(g["size"] for g in store.groups) == sorted(sizes)
    assert store.nbytes == sum(g["img"].shape[0] * (h * w * 4 + 8) for g in store.groups for h, w in [g["size"]])
    for i in range(len(d)):
        want = davis.to_device(davis.collate([d[i]]), dev, input_res=res)
        got = store.ingest(i)
        assert torch.equal(got["image"], want["image"]) and torch.equal(got["gt"], want["gt"]), i
    same = [i for i in range(len(d)) if d[i]["gt"].shape == d[0]["gt"].shape]       # one collated batch
    params = [(j % 2 == 0, 7.0 * j - 10.0, 0.9 + 0.05 * j) for j in range(len(same))]
    got = store.augmented(same, params)
    want = davis.to_device(davis.collate([d[i] for i in same]), dev, augment=params, input_res=res)
    assert torch.equal(got["image"], want["image"]) and torch.equal(got["gt"], want["gt"])


def test_store_sizes_merge_under_a_fixed_resolution(tree):
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)        # sequences at 33x45 and 97x131
    store = davis.DeviceFrames(d, torch.device("cuda"), input_res=(30, 40))
    assert [g["size"] for g in store.groups] == [(30, 40)] and store.groups[0]["img"].shape[0] == len(d)


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


def test_sequence_segmenter_input_res(tree):
    """Bytes equal to a forward on to_device(input_res)'s image, and counts equal to ops.davis_measures on the
    nearest-resized annotation; fp32 frames are refused."""
    from osvos_pytorch_b200 import davis, ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="cc", all_annotations=True)
    res = (48, 64)
    batches = [davis.collate([d[i]]) for i in range(len(d))]

    def frames():
        for b in batches:
            img, gt = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
            yield img, gt
    seg = SequenceSegmenter(net, output="bytescale", frames="bgr8", score=True, input_res=res)
    got = [r.clone() for r in seg(frames())]
    counts = seg.frame_counts()
    assert len(got) == len(d)
    dev = torch.device("cuda")
    for i, b in enumerate(batches):
        ing = davis.to_device(b, dev, input_res=res)
        with torch.no_grad():
            fused = net(ing["image"])[-1]
        assert got[i].shape == (1, 1) + res
        assert torch.equal(got[i], ops.logits_to_u8(fused, "bytescale").cpu()), i
        _, gt_u8, _ = davis.upload(b, dev, input_res=res)
        assert torch.equal(counts[i:i + 1], ops.davis_measures(fused, gt_u8).cpu()), i
    with pytest.raises(ValueError, match="bgr8"):
        SequenceSegmenter(net, input_res=res)


def test_input_res_none_launches_no_resize(tree, monkeypatch):
    """Without input_res the ingest, the store and the segmenter enqueue exactly what they did before: no resize."""
    from osvos_pytorch_b200 import davis, ops
    from osvos_pytorch_b200.inference import SequenceSegmenter

    def refuse(*args, **kwargs):
        raise AssertionError("resize_u8 called without input_res")
    monkeypatch.setattr(ops, "resize_u8", refuse)
    dev = torch.device("cuda")
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    before = ops.KERNEL_LAUNCHES[0]
    davis.to_device(davis.collate([d[0]]), dev)
    assert ops.KERNEL_LAUNCHES[0] - before == 5                    # label stats (3), image, label
    store = davis.DeviceFrames(d, dev)
    store.ingest(0)
    net = _he_net().cuda().eval()
    frames = [torch.from_numpy(d[i]["image"])[None].pin_memory() for i in range(2)]
    assert len([r for r in SequenceSegmenter(net, frames="bgr8")(iter(frames))]) == 2


def test_online_native_loader_with_input_res(tree, tmp_path, monkeypatch):
    """A short ``train_online.py --loader native --input-res`` run with --evaluate writes one PNG per frame at the
    resized size and finite losses and scores."""
    import json
    from PIL import Image
    import train_online
    save = tmp_path / "models"
    save.mkdir()
    torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    hist = train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                              "--parent-epoch", "1", "--log-every", "1", "--no-save", "--loader", "native",
                              "--input-res", "40", "56", "--evaluate"])
    assert len(hist) == 4 and all(np.isfinite(hist))
    pngs = sorted(os.listdir(save / "Results" / "cc"))
    assert pngs == ["00000.png", "00001.png"]
    assert np.asarray(Image.open(save / "Results" / "cc" / pngs[0])).shape == (40, 56)
    with open(save / "Results" / "cc_scores.json") as f:
        assert json.load(f)["sequence"] == "cc"

"""Native DAVIS-2016 ingest on the GPU (csrc/frames.cu, osvos_pytorch_b200.davis): bit-exact against the reference's
make_img_gt_pair (tests/golden/reference_davis.npz), the fused warp bit-exact against ingest + augment.affine_warp,
and the ``--loader native`` online loop against the ``--gpu-augment`` loop on the same bytes."""
import random

import numpy as np
import pytest
import torch

import davis_fixture

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

MEAN = (104.00699, 116.66877, 122.67892)


@pytest.fixture(scope="module")
def fx():
    return davis_fixture.load()


@pytest.fixture(scope="module")
def tree(fx, tmp_path_factory):
    return davis_fixture.write_tree(fx, tmp_path_factory.mktemp("davis"))


def _misaligned(t, offset=1):
    """A CUDA copy of ``t`` whose data starts ``offset`` bytes past an aligned address."""
    buf = torch.empty(t.numel() + 16, dtype=torch.uint8, device="cuda")
    out = buf[offset:offset + t.numel()].view(t.shape)
    out.copy_(t)
    return out


@pytest.mark.parametrize("offset", [0, 1, 3])
def test_ingest_is_bit_identical_to_the_reference(fx, tree, offset):
    from osvos_pytorch_b200 import davis, ops
    for mode in (dict(train=True), dict(train=False), dict(train=False, seq_name="aa")):
        d = davis.DAVIS2016Frames(db_root_dir=tree, **mode)
        for i in range(len(d)):
            it = d[i]
            want_img, want_gt = davis_fixture.pair(fx, d.img_list[i], it["has_gt"])
            img = _misaligned(torch.from_numpy(it["image"])[None].cuda(), offset)
            gt = _misaligned(torch.from_numpy(it["gt"])[None].cuda(), offset)
            got_img = ops.image_from_bgr8(img, MEAN)[0].cpu().numpy().transpose(1, 2, 0)
            got_gt = ops.label_from_u8(gt)[0, 0].cpu().numpy()
            assert np.array_equal(got_img, want_img), (d.img_list[i], offset)
            assert np.array_equal(got_gt, want_gt.astype(np.float32)), (d.img_list[i], offset)


def test_label_stats_flag_binary_masks():
    from osvos_pytorch_b200 import ops
    m = torch.zeros(5, 7, 9, dtype=torch.uint8)
    m[1, 2, 3] = 255                                     # 0 / 255
    m[2, :, :] = 7                                       # all equal, non-zero
    m[3, 0, 0], m[3, 1, 1] = 200, 100                    # non-binary
    m[4, 6, 8] = 1                                       # 0 / 1, in the frame's last byte
    stats = ops.label_stats_u8(m.cuda()).cpu().tolist()
    assert stats == [[0, 1], [255, 1], [7, 1], [200, 0], [1, 1]]


def _batch(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8)
    gt = (torch.rand(n, h, w, generator=g) > 0.6).to(torch.uint8) * 255
    for k in range(0, n, 3):                             # every third mask non-binary
        gt[k] = torch.where(torch.rand(h, w, generator=g) > 0.8, 90, gt[k].long()).to(torch.uint8)
    gt[1] = 0                                            # an empty mask
    return img, gt


@pytest.mark.parametrize("shape", [(37, 33, 45), (35, 24, 31), (3, 97, 131)])
def test_fused_warp_is_ingest_then_affine_warp(shape):
    """Bit-identical to osvos_image_from_bgr8 / osvos_label_from_u8 followed by osvos_affine_warp, over more than 32
    samples (two parameter chunks), odd widths, both flip outcomes; each mask in the mode its binary flag selects."""
    from osvos_pytorch_b200 import augment, ops
    n, h, w = shape
    img, gt = _batch(n, h, w, seed=n)
    img, gt = img.cuda(), gt.cuda()
    params = augment.draw_params(n, rng=random.Random(n))
    params = [(k % 2 == 0, rot, sc) for k, (_, rot, sc) in enumerate(params)]
    out = augment.affine_warp_u8(img, gt, params)
    stats = ops.label_stats_u8(gt)
    want_img = augment.affine_warp(ops.image_from_bgr8(img), params, "cubic")
    assert torch.equal(out["image"], want_img)
    lab = ops.label_from_u8(gt, stats)
    binary = stats[:, 1].cpu().tolist()
    assert 0 in binary and 1 in binary
    near = augment.affine_warp(lab, params, "nearest")
    cub = augment.affine_warp(lab, params, "cubic")
    for k in range(n):
        want = near[k] if binary[k] else cub[k]
        assert torch.equal(out["gt"][k], want), (k, binary[k])
        if binary[k] and gt[k].any():
            assert not torch.equal(near[k], cub[k])      # the mode choice is visible in the output


def test_fused_warp_matches_the_reference_transforms(fx, tree):
    """Against the reference's own RandomHorizontalFlip + ScaleNRotate on its dataset's samples: binary masks bit-exact,
    the image and the non-binary mask (cubic, in float64 in the reference) to fp32 summation order."""
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    seen_nonbinary = False
    for k in range(int(fx["aug.n"])):
        flip, rot, sc = fx[f"aug.{k}.draws"]
        batch = davis.collate([d[int(fx[f"aug.{k}.index"])]])
        out = davis.to_device(batch, torch.device("cuda"), augment=[(bool(flip), float(rot), float(sc))])
        got_img = out["image"][0].cpu().numpy().transpose(1, 2, 0)
        got_gt = out["gt"][0, 0].cpu().numpy()
        assert np.abs(got_img - fx[f"aug.{k}.image"]).max() <= 3e-4, k
        want_gt = fx[f"aug.{k}.gt"]
        src = d[int(fx[f"aug.{k}.index"])]["gt"]
        if np.isin(src, [0, src.max()]).all():
            assert np.array_equal(got_gt, want_gt), k
        else:
            seen_nonbinary = True
            assert np.abs(got_gt - want_gt).max() <= 3e-4, k
    assert seen_nonbinary


def test_to_device_without_augmentation_is_the_ingest(fx, tree):
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    out = davis.to_device(davis.collate([d[0], d[1], d[2]]), torch.device("cuda"))
    for i in range(3):
        want_img, want_gt = davis_fixture.pair(fx, d.img_list[i])
        assert np.array_equal(out["image"][i].cpu().numpy().transpose(1, 2, 0), want_img)
        assert np.array_equal(out["gt"][i, 0].cpu().numpy(), want_gt.astype(np.float32))


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


def test_sequence_segmenter_bgr8_matches_fp32_frames():
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    g = torch.Generator().manual_seed(5)
    frames = [torch.randint(0, 256, (1, 40, 57, 3), generator=g, dtype=torch.uint8) for _ in range(5)]
    mean = np.array(MEAN, dtype=np.float32)
    f32 = [torch.from_numpy(np.subtract(f.numpy().astype(np.float32), mean).transpose(0, 3, 1, 2).copy()).pin_memory()
           for f in frames]
    seg_a = SequenceSegmenter(net, output="logits")
    a = [r.clone() for r in seg_a(iter(f32))]
    seg_b = SequenceSegmenter(net, output="logits", frames="bgr8")
    b = [r.clone() for r in seg_b(f.pin_memory() for f in frames)]
    assert len(a) == len(b) == 5
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert seg_b.h2d_bytes_per_frame * 4 == seg_a.h2d_bytes_per_frame


def test_online_native_loader_matches_gpu_augment(tree, tmp_path, monkeypatch):
    """A short ``train_online.py --loader native`` run writes one PNG per frame, and on a sequence whose first mask is
    binary its losses equal, bit for bit, those of the --gpu-augment loop fed the same bytes ingested to fp32."""
    import os
    import train_online
    from osvos_pytorch_b200 import augment, davis, training
    save = tmp_path / "models"
    save.mkdir()
    torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    iters, n_ave, seed = 4, 5, 9
    common = ["--seq-name", "aa", "--iters", str(iters), "--n-ave-grad", str(n_ave), "--lr", "1e-10",
              "--seed", str(seed), "--parent-epoch", "1", "--log-every", "1", "--no-save"]
    hist_native = train_online.main(common + ["--loader", "native"])
    pngs = sorted(os.listdir(save / "Results" / "aa"))
    assert pngs == ["00000.png", "00001.png", "00002.png"]

    net = _he_net(seed=0)
    net.load_state_dict(torch.load(save / "parent_epoch-0.pth", map_location="cpu"))
    net.cuda()
    first = davis.DAVIS2016Frames(db_root_dir=tree, train=True, seq_name="aa")
    base = davis.to_device(davis.collate([first[0]]), torch.device("cuda"))
    rng = random.Random(seed)
    hist_ref = training.online_finetune(net, lambda it: augment.augment_batch(base, rng=rng), iters, n_ave, 1e-10,
                                        0.0002, log_every=1, log=lambda s: None)
    assert len(hist_native) == iters and all(np.isfinite(hist_native))
    assert hist_native == hist_ref

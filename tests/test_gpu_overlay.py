"""ops.encode_jpeg and ops.overlay_mask (csrc/jpeg_encode.cu) against the numpy restatements (tests/jpeg_encode_ref.py,
tests/overlay_ref.py) and cv2's golden bytes, and the paths that use them: SequenceSegmenter(overlay="jpeg") and
train_online.py --overlay."""
import gc
import json
import os

import numpy as np
import pytest
import torch

import jpeg_encode_cases as C
import jpeg_encode_ref as R
import overlay_ref

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_jpeg_encode.npz")


def _files(out, lengths):
    out, lengths = out.cpu().numpy(), lengths.cpu().tolist()
    return [out[i, :ln].tobytes() for i, ln in enumerate(lengths)]


def _encode(frames_np, q, shift=0):
    """Encodes [N,H,W,3] from a device buffer ``shift`` bytes past an allocation's start."""
    from osvos_pytorch_b200 import ops
    n, h, w, _ = frames_np.shape
    buf = torch.empty(frames_np.size + shift, dtype=torch.uint8, device="cuda")
    x = buf[shift:].view(n, h, w, 3)
    x.copy_(torch.from_numpy(np.ascontiguousarray(frames_np)))
    out, lengths = ops.encode_jpeg(x, q)
    assert out.shape == (n, R.max_bytes(h, w))
    return _files(out, lengths)


@pytest.mark.parametrize("h,w", C.SIZES)
def test_encode_equals_the_restatement(h, w):
    frames = np.stack([C.frame(h, w, k) for k in C.KINDS])
    for q in C.QUALITIES:
        got = _encode(frames, q)
        for f, g in zip(frames, got):
            assert g == R.encode(f, q), (h, w, q)


def test_encode_equals_the_golden_cv2_files():
    g = np.load(GOLDEN)
    keys = [k for k in g.files if k.startswith("jpg:")]
    assert len(keys) >= 10
    for k in keys:
        _, hw, kind, q = k.split(":")
        h, w = (int(v) for v in hw.split("x"))
        assert _encode(C.frame(h, w, kind)[None], int(q))[0] == g[k].tobytes(), k


def test_random_shapes_batches_and_misalignment():
    for i, (h, w) in enumerate(C.random_shapes(30, seed=11)):
        n = (1, 3, 12)[i % 3]
        frames = np.stack([C.frame(h, w, C.KINDS[(i + j) % len(C.KINDS)], seed=j) for j in range(n)])
        q = (30, 75, 95, 100)[i % 4]
        got = _encode(frames, q, shift=i % 4)
        assert got == [R.encode(f, q) for f in frames], (h, w, n, q)


def test_deterministic_and_independent_of_batch_mates():
    frames = np.stack([C.frame(480, 854, k, seed=3) for k in C.KINDS] * 2 + [C.frame(480, 854, "noise", seed=9)] * 2)
    a = _encode(frames, 95)
    b = _encode(frames, 95, shift=1)
    assert a == b
    for j in (0, 4, 11):
        assert _encode(frames[j:j + 1], 95)[0] == a[j]


def test_device_decoder_reads_the_files_as_cv2_does():
    cv2 = pytest.importorskip("cv2")
    from osvos_pytorch_b200 import jpeg, ops
    h, w = 97, 131
    frames = np.stack([C.frame(h, w, k) for k in C.KINDS])
    files = _encode(frames, 95)
    blob_np = jpeg.pack([jpeg.parse(f) for f in files])
    blob = torch.from_numpy(blob_np).cuda()
    out, status = ops.decode_jpeg(blob, len(files), h, w, nseg=jpeg.segment_count(blob_np))
    assert int(status.abs().sum()) == 0
    for f, got in zip(files, out.cpu().numpy()):
        assert np.array_equal(got, cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR))


def test_bad_arguments_are_refused():
    from osvos_pytorch_b200 import ops
    x = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device="cuda")
    for bad in (dict(quality=0), dict(quality=101)):
        with pytest.raises(ValueError):
            ops.encode_jpeg(x, **bad)
    with pytest.raises(ValueError):
        ops.encode_jpeg(torch.zeros(1, 8, 8, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.encode_jpeg(torch.zeros(1, 8, 8, 3, dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):
        ops.encode_jpeg(torch.zeros(1, 1, 65501, 3, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.encode_jpeg(x, out=torch.zeros(1, 10, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.overlay_mask(x, torch.zeros(1, 1, 8, 9, device="cuda"))
    with pytest.raises(ValueError):
        ops.overlay_mask(x, torch.zeros(1, 1, 8, 8, device="cuda"), color=(0, 0, 256))
    assert ops.jpeg_max_bytes(0, 5) == 0 and ops.jpeg_max_bytes(65501, 5) == 0


def test_overlay_equals_the_restatement():
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(5)
    for n, h, w in [(1, 1, 1), (3, 17, 33), (2, 97, 131), (1, 480, 854)]:
        frames = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
        logits = rng.standard_normal((n, 1, h, w)).astype(np.float32)
        logits[rng.random(logits.shape) > 0.9] = 0.0
        logits[rng.random(logits.shape) > 0.9] = -0.0
        logits[rng.random(logits.shape) > 0.95] = np.nan
        for color in ((0, 0, 255), (17, 200, 3)):
            buf = torch.empty(frames.size + 1, dtype=torch.uint8, device="cuda")
            x = buf[1:].view(n, h, w, 3)                             # one byte off alignment
            x.copy_(torch.from_numpy(frames))
            got = ops.overlay_mask(x, torch.from_numpy(logits).cuda(), color=color).cpu().numpy()
            assert np.array_equal(got, overlay_ref.overlay(frames, logits, color)), (n, h, w, color)


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


def _bytes_at_result_size(frame_u8, opts):
    """The frame bytes the overlay is drawn on: the resized frame under input_res (network size results)."""
    from osvos_pytorch_b200 import ops
    if opts.get("input_res") is not None and opts.get("output_res", "network") == "network":
        return ops.resize_u8(frame_u8, opts["input_res"], "bilinear")
    return frame_u8


@pytest.mark.parametrize("opts", [dict(), dict(input_res=(24, 32)), dict(input_res=(24, 32), output_res="stored"),
                                  dict(score=True, encode="png"),
                                  dict(score=True, input_res=(24, 32), output_res="stored", encode="png")])
def test_segmenter_overlay_bgr8(opts):
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    rng = np.random.default_rng(3)
    frames = [torch.from_numpy(rng.integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)).pin_memory() for _ in range(5)]
    score = opts.get("score", False)
    gts = [torch.from_numpy((rng.random((2, 40, 56)) > 0.5).astype(np.uint8) * 255).pin_memory() for _ in range(5)]
    items = list(zip(frames, gts)) if score else frames
    png = opts.get("encode") == "png"
    a = SequenceSegmenter(net, output="bytescale", depth=2, frames="bgr8", **opts)
    want = [[bytes(f) for f in r] if png else r.clone() for r in a(iter(items))]
    base = {k: v for k, v in opts.items() if k != "encode"}
    logit_seg = SequenceSegmenter(net, output="logits", depth=2, frames="bgr8", **base)
    logits = [r.clone() for r in logit_seg(iter(items))]
    b = SequenceSegmenter(net, output="bytescale", depth=2, frames="bgr8", overlay="jpeg", overlay_quality=90, **opts)
    got = [(([bytes(f) for f in r] if png else r.clone()), [bytes(o) for o in ov]) for r, ov in b(iter(items))]
    assert len(got) == len(want) == 5
    for (res, ovs), ref, frame, lg in zip(got, want, frames, logits):
        assert res == ref if png else torch.equal(res, ref)
        img = ops.overlay_mask(_bytes_at_result_size(frame.cuda(), opts), lg.cuda())
        out, lengths = ops.encode_jpeg(img, 90)
        assert ovs == _files(out, lengths)
        assert ovs == [R.encode(f, 90) for f in img.cpu().numpy()]
    if score:
        assert torch.equal(a.frame_counts(), b.frame_counts())
    rh, rw = logits[0].shape[2:]
    assert b.d2h_bytes_per_frame == a.d2h_bytes_per_frame + 2 * (R.max_bytes(rh, rw) + 8)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    import davis_fixture
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


@pytest.mark.parametrize("opts", [dict(), dict(score=True, input_res=(24, 32), output_res="stored")])
def test_segmenter_overlay_jpeg_frames(tree, opts):
    from osvos_pytorch_b200 import davis, ops
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    devd = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="cc", all_annotations=True, decode="device")
    jb = [davis.collate([devd[i]]) for i in range(len(devd))] * 2
    host = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="cc", all_annotations=True)
    a = SequenceSegmenter(net, output="logits", depth=2, frames="jpeg", **opts)
    logits = [r.clone() for r in a(iter(jb))]
    b = SequenceSegmenter(net, output="logits", depth=2, frames="jpeg", overlay="jpeg", **opts)
    got = [(r.clone(), [bytes(o) for o in ov]) for r, ov in b(iter(jb))]
    assert int(b.jpeg_status) == 0 and len(got) == len(logits) == 2 * len(host)
    for i, ((res, ovs), lg) in enumerate(zip(got, logits)):
        assert torch.equal(res, lg)
        img_u8, _ = davis.views(davis.pinned(davis.collate([host[i % len(host)]])["data"]),
                                *(int(v) for v in davis.collate([host[i % len(host)]])["size"]))
        img = ops.overlay_mask(_bytes_at_result_size(img_u8.cuda(), opts), lg.cuda())
        assert ovs == [R.encode(f, 95) for f in img.cpu().numpy()]
    if opts.get("score"):
        assert torch.equal(a.frame_counts(), b.frame_counts())


def test_segmenter_refuses_overlay_without_bytes():
    from osvos_pytorch_b200.inference import SequenceSegmenter
    with pytest.raises(ValueError):
        SequenceSegmenter(_he_net(), frames="nchw_f32", overlay="jpeg")
    with pytest.raises(ValueError):
        SequenceSegmenter(_he_net(), frames="bgr8", overlay="png")
    with pytest.raises(ValueError):
        SequenceSegmenter(_he_net(), frames="bgr8", overlay="jpeg", overlay_quality=0)


@pytest.mark.parametrize("extra", [[], ["--decode", "device", "--input-res", "24", "32", "--output-res", "stored",
                                        "--encode", "device"]])
def test_online_overlay_writes_one_jpeg_per_frame(tmp_path, tree, monkeypatch, extra):
    cv2 = pytest.importorskip("cv2")
    import train_online
    out = {}
    for overlay in (False, True):
        save = tmp_path / str(overlay)
        save.mkdir()
        torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
        monkeypatch.setenv("OSVOS_DB_ROOT", tree)
        monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
        try:
            train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                               "--parent-epoch", "1", "--loader", "native", "--evaluate", "--deterministic"]
                              + extra + (["--overlay"] if overlay else []))
        finally:
            torch.use_deterministic_algorithms(False)
        gc.collect()
        res = save / "Results"
        pngs = {p: (res / "cc" / p).read_bytes() for p in sorted(os.listdir(res / "cc"))}
        out[overlay] = (pngs, json.load(open(res / "cc_scores.json")), res)
    (p0, s0, _), (p1, s1, res) = out[False], out[True]
    assert p0 == p1 and s0 == s1
    jpgs = sorted(os.listdir(res / "cc_overlay"))
    assert [j[:-4] for j in jpgs] == [p[:-4] for p in sorted(p1)] and all(j.endswith(".jpg") for j in jpgs)
    for j in jpgs:
        img = cv2.imread(str(res / "cc_overlay" / j))
        assert img is not None and img.ndim == 3

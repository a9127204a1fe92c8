"""ops.encode_png (csrc/png.cu) against the numpy restatement (tests/png_ref.py) byte for byte, its determinism, and
the paths that use it: SequenceSegmenter(encode="png") and train_online.py --encode device."""
import gc
import io
import json
import os

import numpy as np
import pytest
import torch

import png_cases as C
import png_ref as P

pytestmark = pytest.mark.gpu


def _files(out, lengths):
    out, lengths = out.cpu().numpy(), lengths.cpu().tolist()
    return [out[i, :ln].tobytes() for i, ln in enumerate(lengths)]


def _encode(maps_np, shift=0, four_d=False):
    from osvos_pytorch_b200 import ops
    n, h, w = maps_np.shape
    buf = torch.empty(n * h * w + shift, dtype=torch.uint8, device="cuda")
    x = buf[shift:].view(n, h, w)
    x.copy_(torch.from_numpy(maps_np))
    out, lengths = ops.encode_png(x.view(n, 1, h, w) if four_d else x)
    assert out.shape == (n, P.max_bytes(h, w))
    return _files(out, lengths)


def _random_shapes(k=40, seed=0):
    rng = np.random.default_rng(seed)
    shapes = []
    for _ in range(k):
        w = int(rng.choice([rng.integers(1, 64), rng.integers(64, 1000), rng.integers(8000, 17000)]))
        h = int(rng.integers(1, max(2, min(300, 400000 // w))))
        shapes.append((h, w))
    return shapes


@pytest.mark.parametrize("shape", C.SHAPES + _random_shapes())
def test_kernel_bytes_equal_the_restatement(shape):
    h, w = shape
    kinds = C.KINDS
    maps = np.stack([C.content(kinds[i % len(kinds)], h, w, seed=i) for i in range(3)])
    want = [P.encode(m) for m in maps]
    assert _encode(maps) == want
    assert _encode(maps[:1], shift=1) == want[:1]


@pytest.mark.parametrize("batch", [1, 3, 12])
@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_batches_layouts_and_alignments(batch, shift):
    h, w = 97, 131
    maps = np.stack([C.content(C.KINDS[i % len(C.KINDS)], h, w, seed=40 + i) for i in range(batch)])
    want = [P.encode(m) for m in maps]
    assert _encode(maps, shift=shift) == want
    assert _encode(maps, shift=shift, four_d=True) == want


@pytest.mark.parametrize("shape", [(480, 854), (240, 427)])
def test_full_size_batch_of_12_and_the_long_code(shape):
    maps = np.stack([C.content(("bytescale", "mask")[i % 2], *shape, seed=i) for i in range(12)])
    want = [P.encode(m) for m in maps]
    assert _encode(maps) == want
    fib = C.fibonacci()[None]
    assert _encode(fib) == [P.encode(fib[0])]


def test_deterministic_and_independent_of_batch_mates():
    maps = np.stack([C.content(("bytescale", "mask", "noise")[i % 3], 240, 427, seed=60 + i) for i in range(12)])
    a = _encode(maps)
    assert _encode(maps) == a
    for i in (0, 5, 11):
        assert _encode(maps[i:i + 1]) == [a[i]]


def test_decoders_accept_the_kernel_files():
    cv2 = pytest.importorskip("cv2")
    from PIL import Image
    maps = np.stack([C.bytescale(480, 854, seed=1), C.mask(480, 854, seed=2), C.noise(480, 854, seed=3)])
    for m, data in zip(maps, _encode(maps)):
        assert np.array_equal(np.array(Image.open(io.BytesIO(data))), m)
        assert np.array_equal(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED), m)


def test_bad_inputs_are_refused():
    from osvos_pytorch_b200 import ops
    with pytest.raises(ValueError):
        ops.encode_png(torch.zeros(1, 2, 4, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.encode_png(torch.zeros(1, 4, 4, dtype=torch.float32, device="cuda"))
    with pytest.raises(ValueError):
        ops.encode_png(torch.zeros(1, 4, 32768, dtype=torch.uint8, device="cuda"))


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


@pytest.mark.parametrize("output", ["bytescale", "prob", "mask"])
@pytest.mark.parametrize("opts", [dict(), dict(input_res=(24, 32)), dict(input_res=(24, 32), output_res="stored"),
                                  dict(score=True, input_res=(24, 32), output_res="stored")])
def test_segmenter_png_equals_the_maps(output, opts):
    from PIL import Image
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    rng = np.random.default_rng(3)
    frames = [torch.from_numpy(rng.integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)).pin_memory() for _ in range(5)]
    score = opts.get("score", False)
    gts = [torch.from_numpy((rng.random((2, 40, 56)) > 0.5).astype(np.uint8) * 255).pin_memory() for _ in range(5)]
    items = list(zip(frames, gts)) if score else frames
    a = SequenceSegmenter(net, output=output, depth=2, frames="bgr8", **opts)
    want = [r.clone() for r in a(iter(items))]
    b = SequenceSegmenter(net, output=output, depth=2, frames="bgr8", encode="png", **opts)
    got = [[bytes(f) for f in r] for r in b(iter(items))]
    assert len(got) == len(want) == 5
    for files, maps in zip(got, want):
        assert len(files) == 2
        for f, m in zip(files, maps):
            assert np.array_equal(np.array(Image.open(io.BytesIO(f))), m[0].numpy())
            assert f == P.encode(m[0].numpy())
    cap = P.max_bytes(*want[0].shape[2:])
    assert b.d2h_bytes_per_frame == 2 * (cap + 8)
    if score:
        assert torch.equal(a.frame_counts(), b.frame_counts())


def test_segmenter_refuses_png_of_logits():
    from osvos_pytorch_b200.inference import SequenceSegmenter
    with pytest.raises(ValueError):
        SequenceSegmenter(_he_net(), output="logits", encode="png")


@pytest.mark.parametrize("extra", [[], ["--decode", "device", "--input-res", "24", "32", "--output-res", "stored"]])
def test_online_encode_device_writes_the_same_pngs_and_scores(tmp_path, tmp_path_factory, monkeypatch, extra):
    import davis_fixture
    import train_online
    from PIL import Image
    tree = davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))
    out = {}
    for encode in ("host", "device"):
        save = tmp_path / encode
        save.mkdir()
        torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
        monkeypatch.setenv("OSVOS_DB_ROOT", tree)
        monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
        try:
            train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                               "--parent-epoch", "1", "--loader", "native", "--evaluate", "--deterministic",
                               "--encode", encode] + extra)
        finally:
            torch.use_deterministic_algorithms(False)
        gc.collect()
        res = save / "Results"
        pngs = {p: np.array(Image.open(res / "cc" / p)) for p in sorted(os.listdir(res / "cc"))}
        out[encode] = (pngs, json.load(open(res / "cc_scores.json")))
    (hp, hs), (dp, ds) = out["host"], out["device"]
    assert len(hp) == 2 and sorted(hp) == sorted(dp) and all(p.endswith(".png") for p in dp)
    assert all(np.array_equal(hp[k], dp[k]) for k in hp)
    assert hs == ds

"""ops.decode_png (csrc/png_decode.cu) against cv2 and Pillow bit for bit, the device round trip with ops.encode_png,
the proven-cut machinery, the status words, png.decode_files, and the results scorer built on it."""
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import png_cases as C
import png_decode_cases as D

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cv(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_GRAYSCALE)


def _decode(datas, shift=0):
    """Files of one size -> (pixels [n,h,w] numpy, status list, path list)."""
    from osvos_pytorch_b200 import ops, png
    parsed = [png.parse(d) for d in datas]
    assert all(isinstance(p, png.Parsed) for p in parsed), parsed
    blob = png.pack(parsed)
    n, h, w = len(parsed), parsed[0].h, parsed[0].w
    buf = torch.empty(n * h * w + shift, dtype=torch.uint8, device="cuda")
    path = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    out, status = ops.decode_png(torch.from_numpy(blob).cuda(), n, h, w, png.segment_count(blob),
                                 out=buf[shift:].view(n, h, w), path=path)
    return out.cpu().numpy(), status.cpu().tolist(), path.cpu().tolist()


_FILES = D.subset_files()


@pytest.mark.parametrize("name,data", _FILES, ids=[n for n, _ in _FILES])
def test_equals_cv2_and_pillow(name, data):
    from PIL import Image
    got, status, path = _decode([data], shift=len(name) % 4)
    assert status == [0]
    assert np.array_equal(got[0], _cv(data))
    pil = np.array(Image.open(io.BytesIO(data)))
    assert np.array_equal(got[0], pil.astype(np.uint8) * 255 if pil.dtype == bool else pil)
    assert path == [1 if name.startswith("own-") else 2]


@pytest.mark.parametrize("batch", [1, 3, 12])
@pytest.mark.parametrize("shift", [1, 2, 3])
def test_mixed_batches_and_alignments(batch, shift):
    ws = D.writers()
    maps = [C.content(C.KINDS[i % len(C.KINDS)], 97, 131, seed=20 + i) for i in range(batch)]
    datas = [ws[(5 * i + shift) % len(ws)][1](m) for i, m in enumerate(maps)]
    got, status, _ = _decode(datas, shift=shift)
    assert status == [0] * batch
    for g, d in zip(got, datas):
        assert np.array_equal(g, _cv(d))
    for i in (0, batch - 1):                         # a file decodes the same alone as among batch mates
        assert np.array_equal(_decode([datas[i]])[0][0], got[i])


def _random_shapes(k=40, seed=1):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(k):
        w = int(rng.choice([rng.integers(1, 64), rng.integers(64, 1000), rng.integers(8000, 17000)]))
        out.append((int(rng.integers(1, max(2, min(300, 400000 // w)))), w))
    return out


@pytest.mark.parametrize("shape", C.SHAPES + _random_shapes())
def test_device_round_trip(shape):
    """decode_png(encode_png(x)) == x with no host codec: the file bytes go through png.parse and png.pack only."""
    from osvos_pytorch_b200 import ops
    h, w = shape
    maps = np.stack([C.content(k, h, w, seed=i) for i, k in enumerate(C.KINDS)])
    out, lengths = ops.encode_png(torch.from_numpy(maps).cuda())
    out, lengths = out.cpu().numpy(), lengths.cpu().tolist()
    got, status, path = _decode([out[i, :ln].tobytes() for i, ln in enumerate(lengths)], shift=1)
    assert status == [0] * len(maps) and path == [1] * len(maps)
    assert np.array_equal(got, maps)


def test_full_size_batch_of_12():
    from osvos_pytorch_b200 import ops
    maps = np.stack([C.content(("bytescale", "mask")[i % 2], 480, 854, seed=i) for i in range(12)])
    out, lengths = ops.encode_png(torch.from_numpy(maps).cuda())
    out, lengths = out.cpu().numpy(), lengths.cpu().tolist()
    own = [out[i, :ln].tobytes() for i, ln in enumerate(lengths)]
    got, status, path = _decode(own)
    assert status == [0] * 12 and path == [1] * 12 and np.array_equal(got, maps)
    foreign = [D.pillow(m) if i % 2 else D.opencv(m) for i, m in enumerate(maps)]
    got, status, path = _decode(foreign)
    assert status == [0] * 12 and path == [2] * 12 and np.array_equal(got, maps)


def test_proven_and_rejected_cuts():
    for make, want_path in ((D.full_flush_file, 1), (D.false_cut_file, 2), (D.sync_flush_file, 2)):
        data, m = make()
        got, status, path = _decode([data])
        assert status == [0] and path == [want_path], make.__name__
        assert np.array_equal(got[0], m)


@pytest.mark.parametrize("bit", [1, 2, 4, 8, 16])
def test_status_words(bit):
    """Contract tests of the bounds checks: the corrupt file reports its bit, the call returns, and a valid decode that
    follows on the same stream is right."""
    files, m = D.corrupt_files()
    good = D.pillow(m)
    _, status, _ = _decode([files[bit]])
    assert status[0] & bit
    got, status, _ = _decode([good, files[bit], good])
    assert status[0] == 0 and status[2] == 0 and status[1] & bit
    assert np.array_equal(got[0], m) and np.array_equal(got[2], m)


def test_header_status_and_argument_checks():
    from osvos_pytorch_b200 import ops, png
    parsed = [png.parse(D.pillow(C.mask(20, 30, 1)))]
    blob = png.pack(parsed)
    dev = torch.from_numpy(blob).cuda()
    _, status = ops.decode_png(dev, 1, 20, 31, 1)            # the blob says 20 x 30
    assert status.cpu().tolist() == [32]
    with pytest.raises(ValueError, match="nseg"):
        ops.decode_png(dev, 1, 20, 30, None)
    with pytest.raises(ValueError, match="aligned"):
        ops.decode_png(torch.cat([dev, dev])[8:8 + len(blob)], 1, 20, 30, 1)
    with pytest.raises(ValueError, match="out"):
        ops.decode_png(dev, 1, 20, 30, 1, out=torch.empty((1, 20, 31), dtype=torch.uint8, device="cuda"))
    with pytest.raises(RuntimeError):
        ops.decode_png(torch.from_numpy(blob), 1, 20, 30, 1)


def test_decode_files_mixes_device_fallback_and_corrupt():
    from osvos_pytorch_b200 import png
    m = C.bytescale(6, 10, 8)
    corrupt, _ = D.corrupt_files()                           # 6 x 10 as well
    rgb = cv2.imencode(".png", np.stack([m] * 3, -1))[1].tobytes()
    datas = [D.pillow(m), rgb, corrupt[16], D.pillow(m, "1"), D.opencv(m, 0)]
    # cv2 undoes filter type 7 leniently or refuses the file; only the first matters here
    want = [_cv(d) for d in datas]
    if want[2] is None:
        datas[2], want[2] = D.opencv(m, 9), m
    out, fallback, redecoded = png.decode_files(datas, "cuda")
    assert (fallback, redecoded) == (1, 1 if datas[2] is corrupt[16] else 0)
    for g, w_ in zip(out.cpu().numpy(), want):
        assert np.array_equal(g, w_)
    with pytest.raises(ValueError, match="size"):
        png.decode_files([D.pillow(m), D.pillow(m[:5])], "cuda")


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    import davis_fixture
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def _annotations(tree, seq):
    folder = os.path.join(tree, "Annotations", "480p", seq)
    return {f[:-4]: cv2.imread(os.path.join(folder, f), 0) for f in sorted(os.listdir(folder))}


def _write(folder, name, m):
    os.makedirs(folder, exist_ok=True)
    cv2.imwrite(os.path.join(folder, name + ".png"), m)


@pytest.mark.parametrize("decode", ["device", "host"])
def test_score_results_on_perfect_and_shifted_masks(tree, tmp_path, decode):
    import davis_measures_ref as M
    from osvos_pytorch_b200 import evaluation
    shifted = {}
    for seq in ("aa", "bb", "cc"):
        for stem, g in _annotations(tree, seq).items():
            _write(tmp_path / "perfect" / seq, stem, np.where(g > 0, 255, 0).astype(np.uint8))
            s = np.roll(np.where(g > 0, 200, 50).astype(np.uint8), 3, axis=1)
            shifted[(seq, stem)] = (s, g)
            _write(tmp_path / "shifted" / seq, stem, s)
    res = evaluation.score_results(str(tmp_path / "perfect"), tree, sequences=["aa", "bb", "cc"], decode=decode, batch=2)
    assert res["frames"] == 7 and res["redecoded_files"] == 0
    for seq, r in res["sequences"].items():
        assert r["J"] == [1.0] * len(r["J"]) and r["F"] == [1.0] * len(r["F"])
    res = evaluation.score_results(str(tmp_path / "shifted"), tree, decode=decode)     # val_seqs.txt: bb
    assert list(res["sequences"]) == ["bb"] and res["frames"] == 2
    for i, stem in enumerate(sorted(_annotations(tree, "bb"))):
        s, g = shifted[("bb", stem)]
        want = M.counts(np.where(s >= 128, 1.0, -1.0), g)
        assert res["sequences"]["bb"]["counts"][i] == [int(v) for v in want]
    low = evaluation.score_results(str(tmp_path / "shifted"), tree, sequences=["bb"], threshold=40, decode=decode)
    assert all(c[1] == 48 * 70 for c in low["sequences"]["bb"]["counts"])            # 50 and 200 are both foreground


def test_score_results_refuses_incomplete_input(tree, tmp_path):
    from osvos_pytorch_b200 import evaluation
    for stem, g in _annotations(tree, "aa").items():
        _write(tmp_path / "r" / "aa", stem, g)
    assert evaluation.score_results(str(tmp_path / "r"), tree, sequences=["aa"])["frames"] == 3
    with pytest.raises(ValueError, match="unknown sequence"):
        evaluation.score_results(str(tmp_path / "r"), tree, sequences=["zz"])
    with pytest.raises(ValueError, match="val_seqs"):
        evaluation.score_results(str(tmp_path / "r"), tree)
    os.remove(tmp_path / "r" / "aa" / "00001.png")
    with pytest.raises(ValueError, match="no result for frame"):
        evaluation.score_results(str(tmp_path / "r"), tree, sequences=["aa"])
    _write(tmp_path / "r" / "aa", "00001", np.zeros((30, 45), np.uint8))
    with pytest.raises(ValueError, match="size|results are"):
        evaluation.score_results(str(tmp_path / "r"), tree, sequences=["aa"])
    _write(tmp_path / "r" / "aa", "00001", np.zeros((33, 45), np.uint8))
    _write(tmp_path / "r" / "aa", "00009", np.zeros((33, 45), np.uint8))
    with pytest.raises(ValueError, match="no annotation"):
        evaluation.score_results(str(tmp_path / "r"), tree, sequences=["aa"])


@pytest.mark.parametrize("output", ["mask", "prob"])
def test_scoring_the_written_files_equals_scoring_in_the_pipeline(tree, tmp_path, output):
    from osvos_pytorch_b200 import evaluation
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net(seed=3).cuda().eval()
    ann = _annotations(tree, "cc")
    stems = sorted(ann)
    frames = [(torch.from_numpy(cv2.imread(os.path.join(tree, "JPEGImages", "480p", "cc", s + ".jpg"))[None]).pin_memory(),
               torch.from_numpy(ann[s][None]).pin_memory()) for s in stems]
    seg = SequenceSegmenter(net, output=output, frames="bgr8", encode="png", score=True)
    os.makedirs(tmp_path / "Results" / "cc")
    for s, files in zip(stems, seg(iter(frames))):
        with open(tmp_path / "Results" / "cc" / (s + ".png"), "wb") as f:
            f.write(files[0])
    want = seg.frame_counts().cpu().tolist()
    for decode in ("device", "host"):
        res = evaluation.score_results(str(tmp_path / "Results"), tree, sequences=["cc"], decode=decode)
        assert res["sequences"]["cc"]["counts"] == want
        assert res["fallback_files"] == 0 and res["redecoded_files"] == 0
    if output == "mask":
        env = dict(os.environ, OSVOS_DB_ROOT=tree, OSVOS_SAVE_ROOT=str(tmp_path), PYTHONPATH=ROOT)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "evaluate_results.py"), "--seq", "cc", "--json",
                            str(tmp_path / "scores.json")], env=env, capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stderr
        lines = r.stdout.strip().splitlines()
        assert lines[0].startswith("Scores of cc (frames 1 .. n-2): J M/O/D: ")
        assert lines[-1].startswith("Scores of the dataset, mean over 1 sequences (frames 1 .. n-2): J M/O/D: ")
        saved = json.load(open(tmp_path / "scores.json"))
        assert saved["sequences"]["cc"]["counts"] == want and saved["threshold"] == 128

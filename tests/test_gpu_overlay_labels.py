"""ops.overlay_labels (csrc/jpeg_encode.cu, DESIGN.md §25) against the numpy rule (tests/overlay_labels_ref.py) and
ops.overlay_mask, and the paths that use it: visualize.render_results (JPEG files equal to cv2.imencode of the
restated overlay, MJPEG videos of those files) and train_online.py --davis 2017 --overlay."""
import gc
import json
import os

import numpy as np
import pytest
import torch

import overlay_labels_ref as R
from png_palette_ref import davis_palette
from test_overlay_labels import label_maps

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")


def _at(arr, shift):
    """A device copy of ``arr`` that starts ``shift`` bytes past an allocation's start."""
    buf = torch.empty(arr.size + shift, dtype=torch.uint8, device="cuda")
    t = buf[shift:].view(*arr.shape)
    t.copy_(torch.from_numpy(np.ascontiguousarray(arr)))
    return t


@pytest.mark.parametrize("n,h,w", [(1, 1, 1), (1, 7, 5), (3, 37, 53), (12, 48, 85), (2, 480, 854)])
def test_overlay_labels_equals_the_rule(n, h, w):
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(n * 1000 + w)
    frames = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    lab = np.zeros((n, h, w), np.uint8)
    yy, xx = np.mgrid[:h, :w]
    for i in range(n):
        for k in range(1, 9):
            cy, cx = rng.integers(0, h), rng.integers(0, w)
            lab[i][((yy - cy) / max(1, h // 4)) ** 2 + ((xx - cx) / max(1, w // 5)) ** 2 <= 1] = k * 31 % 255
        lab[i, h // 2, :] = 3                                 # a 1-pixel line across the frame
        lab[i][rng.random((h, w)) < 0.02] = rng.integers(0, 256)
    for pal, name in [(None, "default"), (davis_palette(4), "short"), (bytes(rng.integers(0, 256, 768, np.uint8)),
                                                                       "file")]:
        want = R.overlay(frames, lab, davis_palette(256) if pal is None else pal)
        for fs, ls, os_ in [(0, 0, 0), (1, 3, 5)]:           # aligned, and every buffer off alignment
            x, y = _at(frames, fs), _at(lab, ls)
            out = torch.empty(frames.size + os_, dtype=torch.uint8, device="cuda")[os_:].view(n, h, w, 3)
            got = ops.overlay_labels(x, y, pal, out=out)
            assert got.data_ptr() == out.data_ptr()
            assert np.array_equal(got.cpu().numpy(), want), (name, fs)
            assert np.array_equal(x.cpu().numpy(), frames)   # the frames are only read
            # [N,1,H,W] labels, drawn in place
            got = ops.overlay_labels(x, y.view(n, 1, h, w), pal, out=x)
            assert got.data_ptr() == x.data_ptr() and np.array_equal(x.cpu().numpy(), want), (name, fs)


@pytest.mark.parametrize("name", list(label_maps()))
def test_overlay_labels_on_the_rule_cases(name):
    from osvos_pytorch_b200 import ops
    lab = label_maps()[name]
    frame = np.random.default_rng(len(name)).integers(0, 256, lab.shape + (3,), dtype=np.uint8)
    for pal in (davis_palette(6), davis_palette(256), b"\x10\x20\x30"):
        got = ops.overlay_labels(_at(frame[None], 1), _at(lab[None], 2), pal).cpu().numpy()
        assert np.array_equal(got, R.overlay(frame[None], lab[None], pal)), name


@pytest.mark.parametrize("n,h,w", [(1, 17, 23), (3, 40, 57), (12, 480, 854)])
def test_one_object_equals_overlay_mask(n, h, w):
    from osvos_pytorch_b200 import ops
    rng = np.random.default_rng(h)
    frames = torch.from_numpy(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)).cuda()
    logits = torch.from_numpy(rng.normal(0, 1, (n, 1, h, w)).astype(np.float32)).cuda()
    logits[:, :, h // 4:h // 2, w // 4:w // 2] = 2.0
    logits.view(-1)[::7] = 0.0
    want = ops.overlay_mask(frames, logits)
    got = ops.overlay_labels(frames, (logits > 0).to(torch.uint8), b"\0\0\0\xff\0\0")
    assert torch.equal(got, want)


def test_overlay_labels_refuses_bad_input():
    from osvos_pytorch_b200 import ops
    x = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device="cuda")
    lab = torch.zeros(1, 8, 8, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        ops.overlay_labels(x, torch.zeros(1, 8, 9, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.overlay_labels(x, lab.float())
    with pytest.raises(ValueError):
        ops.overlay_labels(x, lab.view(1, 8, 8, 1))
    with pytest.raises(ValueError):
        ops.overlay_labels(x[..., :2], lab)
    with pytest.raises(ValueError):
        ops.overlay_labels(x, lab, palette=b"\0\0")
    with pytest.raises(ValueError):
        ops.overlay_labels(x, lab, palette=b"\0" * 771)
    with pytest.raises(ValueError):
        ops.overlay_labels(x, lab, out=torch.zeros(1, 8, 8, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(RuntimeError):
        ops.overlay_labels(x.cpu(), lab)


# ---- render_results ---------------------------------------------------------------------------------------------------

SIZES = {"a": (45, 61), "b": (40, 56)}                        # a sequence per size; odd sizes on purpose
FRAMES = 5


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """One DAVIS layout serving both years: JPEG frames, DAVIS-2017 palette annotations with a void band, the 2016 and
    2017 sequence lists."""
    root = tmp_path_factory.mktemp("davis_vis")
    rng = np.random.default_rng(8)
    for s, (seq, (h, w)) in enumerate(SIZES.items()):
        os.makedirs(root / "JPEGImages" / "480p" / seq)
        os.makedirs(root / "Annotations" / "480p" / seq)
        yy, xx = np.mgrid[:h, :w]
        for f in range(FRAMES):
            img = np.stack([(xx * 4 + f * 9) % 256, (yy * 5) % 256, (xx + yy) * 2 % 256], -1).astype(np.uint8)
            img = np.clip(img.astype(np.int32) + rng.integers(-30, 31, img.shape), 0, 255).astype(np.uint8)
            cv2.imwrite(str(root / "JPEGImages" / "480p" / seq / f"{f:05d}.jpg"), img)
            gt = np.zeros((h, w), np.uint8)
            gt[h // 5:h // 2, w // 6:w // 2] = 1
            gt[h // 2:, w // 2:] = 2
            gt[0, 0] = 3
            if f:
                gt[:, w // 3:w // 3 + 2] = 255                # void band
            im = Image.fromarray(gt, "P")
            im.putpalette(davis_palette(256))
            im.save(str(root / "Annotations" / "480p" / seq / f"{f:05d}.png"))
    (root / "val_seqs.txt").write_text("\n".join(SIZES) + "\n")
    os.makedirs(root / "ImageSets" / "2017")
    (root / "ImageSets" / "2017" / "val.txt").write_text("\n".join(SIZES) + "\n")
    return str(root)


def _results(root, davis, scale=1):
    """Result PNGs: 2016 bytescaled probability maps; 2017 label maps, palette files (one without a PLTE chunk)."""
    rng = np.random.default_rng(3)
    os.makedirs(root)
    for seq, (h, w) in SIZES.items():
        os.makedirs(os.path.join(root, seq))
        h, w = h // scale, w // scale
        for f in range(FRAMES):
            path = os.path.join(root, seq, f"{f:05d}.png")
            if davis == "2016":
                m = rng.integers(0, 256, (h, w)).astype(np.uint8)
                m[h // 4:3 * h // 4, w // 4:3 * w // 4] = 255
                cv2.imwrite(path, m)
            else:
                lab = np.zeros((h, w), np.uint8)
                lab[h // 4:3 * h // 4, w // 5:w // 2] = 1
                lab[h // 3:, w // 2:] = 2
                lab[rng.random((h, w)) < 0.03] = 3
                lab[0, :] = 3                                 # past a 3-entry palette: black
                if f == 3:
                    Image.fromarray(lab, "L").save(path)       # no palette: the DAVIS palette
                else:
                    im = Image.fromarray(lab, "P")
                    im.putpalette(davis_palette(3) if f % 2 else bytes(range(48)))
                    im.save(path)


def _restated(results, root, davis, quality):
    """{relative path: bytes}: cv2.imencode of the restated overlay of each result over cv2.imread of its frame."""
    from osvos_pytorch_b200 import png
    out = {}
    for seq in SIZES:
        for f in range(FRAMES):
            frame = cv2.imread(os.path.join(root, "JPEGImages", "480p", seq, f"{f:05d}.jpg"))
            path = os.path.join(results, seq, f"{f:05d}.png")
            data = open(path, "rb").read()
            if davis == "2016":
                lab, pal = (cv2.imread(path, 0) >= 128).astype(np.uint8), b"\0\0\0\xff\0\0"
            else:
                lab, pal = np.array(Image.open(path)), png.palette_of(data) or davis_palette(256)
            if lab.shape != frame.shape[:2]:
                lab = np.array(Image.fromarray(lab).resize(frame.shape[1::-1], Image.NEAREST))
            ok, buf = cv2.imencode(".jpg", R.overlay(frame[None], lab[None], pal)[0], [cv2.IMWRITE_JPEG_QUALITY, quality])
            out[os.path.join(seq + "_overlay", f"{f:05d}.jpg")] = buf.tobytes()
    return out


def _written(out_dir):
    return {os.path.join(d, f): open(os.path.join(out_dir, d, f), "rb").read()
            for d in sorted(os.listdir(out_dir)) if d.endswith("_overlay") for f in sorted(os.listdir(os.path.join(out_dir, d)))}


@pytest.mark.parametrize("davis", ["2016", "2017"])
@pytest.mark.parametrize("scale", [1, 2])
def test_render_results_equals_cv2_of_the_rule(tmp_path, tree, davis, scale):
    from osvos_pytorch_b200 import video, visualize
    results = str(tmp_path / "res")
    _results(results, davis, scale)
    want = _restated(results, tree, davis, 90)
    got = {}
    for decode in ("device", "host"):
        out = str(tmp_path / decode)
        r = visualize.render_results(results, tree, davis=davis, quality=90, video=True, fps=12, out_dir=out,
                                     decode=decode, batch=3)
        assert r["sequences"] == {seq: FRAMES for seq in SIZES} and r["frames"] == FRAMES * len(SIZES)
        got[decode] = _written(out)
        assert got[decode] == want, (decode, sorted(k for k in want if got[decode].get(k) != want[k]))
        for seq in SIZES:
            avi = video.read_avi(open(os.path.join(out, seq + "_overlay.avi"), "rb").read())
            assert avi["frames"] == [want[os.path.join(seq + "_overlay", f"{f:05d}.jpg")] for f in range(FRAMES)]
    assert got["device"] == got["host"]


def test_render_results_cli_and_missing_frames(tmp_path, tree):
    import visualize_results
    results = str(tmp_path / "res")
    _results(results, "2017")
    visualize_results.main(["--results", results, "--db-root", tree, "--davis", "2017", "--seq", "b", "--video",
                            "--quality", "80"])
    assert sorted(os.listdir(results)) == ["a", "b", "b_overlay.avi"]     # --video alone writes no frame folder
    visualize_results.main(["--results", results, "--db-root", tree, "--davis", "2017", "--out", str(tmp_path / "o")])
    want = _restated(results, tree, "2017", 95)
    assert _written(str(tmp_path / "o")) == want
    open(os.path.join(results, "a", "00099.png"), "wb").write(open(os.path.join(results, "a", "00000.png"), "rb").read())
    with pytest.raises(ValueError, match="no frame for result"):
        visualize_results.main(["--results", results, "--db-root", tree, "--davis", "2017"])


# ---- train_online.py --davis 2017 --overlay ---------------------------------------------------------------------------

def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


@pytest.mark.parametrize("extra", [[], ["--encode", "device", "--decode", "device", "--overlay-quality", "80"]])
def test_online_2017_overlay(tmp_path, tree, monkeypatch, extra):
    import train_online
    from osvos_pytorch_b200 import png, visualize
    seq = "b"
    runs = {}
    for overlay in (False, True):
        save = tmp_path / str(overlay)
        save.mkdir()
        torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
        monkeypatch.setenv("OSVOS_DB_ROOT", tree)
        monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
        try:
            train_online.main(["--seq-name", seq, "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                               "--parent-epoch", "1", "--loader", "native", "--davis", "2017", "--evaluate",
                               "--deterministic"] + extra + (["--overlay"] if overlay else []))
        finally:
            torch.use_deterministic_algorithms(False)
        gc.collect()
        res = save / "Results"
        pngs = {p: (res / seq / p).read_bytes() for p in sorted(os.listdir(res / seq))}
        runs[overlay] = (pngs, (res / f"{seq}_scores.json").read_bytes(), res)
    (p0, s0, res0), (p1, s1, res) = runs[False], runs[True]
    assert p0 == p1 and s0 == s1 and len(p1) == FRAMES
    assert not os.path.exists(res0 / f"{seq}_overlay")
    assert json.loads(s1)["n_objects"] == 3
    first = open(os.path.join(tree, "Annotations", "480p", seq, "00000.png"), "rb").read()
    quality = 80 if "--overlay-quality" in extra else 95
    visualize.render_results(str(res), tree, sequences=[seq], davis="2017", quality=quality,
                             out_dir=str(tmp_path / "again"), palette=png.palette_of(first))
    written = _written(str(res))
    assert len(written) == FRAMES and written == _written(str(tmp_path / "again"))

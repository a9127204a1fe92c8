"""The K-object overlay rule (tests/overlay_labels_ref.py) against cv2's per-object contours, the DAVIS palette, the
MJPEG writer read back by its chunk walker and by cv2.VideoCapture, and visualize_results.py's argument checks."""
import os
import struct

import numpy as np
import pytest

import overlay_labels_ref as R
import overlay_ref
from png_palette_ref import davis_palette as davis_palette_ref

cv2 = pytest.importorskip("cv2")


def _drawn(mask):
    """The pixels cv2.drawContours(findContours(mask, RETR_TREE, CHAIN_APPROX_SIMPLE), -1, 0, 1) paints."""
    contours = cv2.findContours(mask.astype(np.uint8), cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)[-2]
    canvas = np.zeros(mask.shape, np.uint8)
    cv2.drawContours(canvas, contours, -1, 1, 1)
    return canvas.astype(bool)


def label_maps():
    """Label maps with many ids, holes, 1-pixel lines, objects touching each other and the frame's border."""
    rng = np.random.default_rng(11)
    out = {}
    m = np.zeros((24, 30), np.uint8)
    m[2:20, 3:15] = 1
    m[2:20, 15:27] = 2                                        # touching along a column
    m[8:12, 6:10] = 0                                         # a hole
    m[9:11, 18:22] = 3                                        # an object inside another
    m[0, :] = 4                                               # on the border
    m[:, 29] = 5
    m[22, 2:28] = 6                                           # a 1-pixel line
    out["touching"] = m
    m = np.zeros((17, 19), np.uint8)
    m[::2, :] = 7
    m[:, ::3] = 200
    out["grid"] = m
    out["checker"] = ((np.indices((13, 15)).sum(0) % 2) * 9).astype(np.uint8)
    out["full"] = np.full((9, 11), 254, np.uint8)
    out["single"] = np.pad(np.full((1, 1), 3, np.uint8), 4)
    for k in range(24):
        h, w = (int(v) for v in rng.integers(1, 70, 2))
        kmax = [2, 4, 16, 254][k % 4]
        if k % 3 == 0:
            out[f"noise{k}"] = rng.integers(0, kmax + 1, (h, w)).astype(np.uint8)
        else:                                                 # blobs of random ids painted over each other
            lab = np.zeros((h, w), np.uint8)
            yy, xx = np.mgrid[:h, :w]
            for _ in range(int(rng.integers(1, 12))):
                cy, cx = rng.integers(0, h), rng.integers(0, w)
                ry, rx = rng.integers(1, max(2, h // 2)), rng.integers(1, max(2, w // 2))
                lab[((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1] = rng.integers(1, kmax + 1)
            out[f"blobs{k}"] = lab
    return out


@pytest.mark.parametrize("name", list(label_maps()))
def test_each_objects_outline_is_what_draw_contours_paints(name):
    lab = label_maps()[name]
    e = R.edge(lab)
    for k in np.unique(lab):
        if k == 0:
            continue
        obj = lab == k
        assert np.array_equal(e & obj, _drawn(obj)), (name, k)
    assert not (e & (lab == 0)).any()


@pytest.mark.parametrize("name", list(label_maps()))
def test_rule_draws_each_object_in_its_colour(name):
    lab = label_maps()[name]
    rng = np.random.default_rng(len(name))
    frame = rng.integers(0, 256, lab.shape + (3,), dtype=np.uint8)
    pal = davis_palette_ref(6)                                # ids 6 and up lie past the palette: black
    got = R.overlay(frame[None], lab[None], pal)[0].astype(np.int64)
    e = R.edge(lab)
    assert np.array_equal(got[lab == 0], frame[lab == 0])
    assert (got[e] == 0).all()
    rgb = np.frombuffer(pal, np.uint8).reshape(-1, 3)
    for k in np.unique(lab[(lab != 0) & ~e]):
        c = rgb[k, ::-1].astype(np.int64) if k < 6 else np.zeros(3, np.int64)
        sel = (lab == k) & ~e
        assert np.array_equal(got[sel], (frame[sel].astype(np.int64) + c + 1) >> 1), (name, k)


def test_one_object_in_red_is_the_mask_overlay():
    rng = np.random.default_rng(2)
    frames = rng.integers(0, 256, (3, 21, 34, 3), dtype=np.uint8)
    logits = rng.normal(0, 1, (3, 21, 34)).astype(np.float32)
    logits[0, 5:15, 5:20] = 3.0
    want = overlay_ref.overlay(frames, logits)
    got = R.overlay(frames, (logits > 0).astype(np.uint8), b"\0\0\0\xff\0\0")
    assert np.array_equal(got, want)


def test_davis_palette_is_the_voc_colour_map():
    from osvos_pytorch_b200 import png
    voc = [(0, 0, 0), (128, 0, 0), (0, 128, 0), (128, 128, 0), (0, 0, 128), (128, 0, 128), (0, 128, 128),
           (128, 128, 128), (64, 0, 0), (192, 0, 0), (64, 128, 0), (192, 128, 0), (64, 0, 128), (192, 0, 128),
           (64, 128, 128), (192, 128, 128), (0, 64, 0), (128, 64, 0), (0, 192, 0), (128, 192, 0), (0, 64, 128)]
    pal = png.davis_palette()
    assert len(pal) == 768 and png.davis_palette(4) == pal[:12]
    assert [tuple(pal[3 * k:3 * k + 3]) for k in range(len(voc))] == voc
    assert tuple(pal[-3:]) == (224, 224, 192)                 # VOC's entry 255, the void colour
    assert pal == davis_palette_ref(256)


# ---- MJPEG ------------------------------------------------------------------------------------------------------------

def _jpegs(n, h, w, seed):
    rng = np.random.default_rng(seed)
    out = []
    yy, xx = np.mgrid[:h, :w]
    for i in range(n):
        img = np.stack([(xx * 3 + i * 20) % 256, (yy * 2) % 256, (xx + yy + 40 * i) % 256], -1).astype(np.uint8)
        img = cv2.GaussianBlur(img, (5, 5), 0)               # smooth content: decoders differ little there
        img[h // 4:h // 2, w // 4:w // 2] = rng.integers(0, 256, 3)   # and one flat block with sharp edges
        ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
        assert ok
        data = buf.tobytes()
        out.append(data + (b"\0" if i % 2 and len(data) % 2 == 0 else b""))   # odd sizes too
    return out


@pytest.mark.parametrize("n,h,w,fps", [(1, 16, 16, 24.0), (7, 48, 64, 30000 / 1001), (12, 120, 214, 10.0)])
def test_avi_holds_the_files_as_given(tmp_path, n, h, w, fps):
    from osvos_pytorch_b200 import video
    files = _jpegs(n, h, w, seed=n)
    assert any(len(f) % 2 for f in files) or n == 1
    path = str(tmp_path / "clip.avi")
    size = video.write_avi(path, files, fps)
    data = open(path, "rb").read()
    assert size == len(data) and data[:4] == b"RIFF" and struct.unpack("<I", data[4:8])[0] == len(data) - 8
    avi = video.read_avi(data)
    assert avi["frames"] == files
    assert len(avi["index"]) == n
    for (tag, flags, off, ln), f in zip(avi["index"], files):
        assert tag == b"00dc" and flags == video.AVIIF_KEYFRAME and ln == len(f)
        p = avi["movi"] + off                                 # offsets count from the 'movi' tag
        assert data[p:p + 4] == b"00dc" and struct.unpack("<I", data[p + 4:p + 8])[0] == len(f)
        assert data[p + 8:p + 8 + ln] == f
    usec, _, _, flags, frames, _, streams, _, aw, ah = struct.unpack("<10I", avi["avih"][:40])
    assert (frames, streams, aw, ah) == (n, 1, w, h) and flags & video.AVIF_HASINDEX
    assert usec == round(1e6 / fps)
    assert avi["strh"][:8] == b"vidsMJPG"
    scale, rate, _, length = struct.unpack("<4I", avi["strh"][20:36])
    assert length == n and abs(rate / scale - fps) < 1e-9
    assert struct.unpack("<Iii", avi["strf"][:12]) == (40, w, h) and avi["strf"][16:20] == b"MJPG"
    cap = cv2.VideoCapture(path)
    try:
        assert cap.isOpened()
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == n
        assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (w, h)
        for f in files:
            ok, img = cap.read()
            assert ok and img.shape == (h, w, 3)
            want = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR).astype(np.int32)
            # FFmpeg's IDCT and upsampling are not libjpeg-turbo's: a few levels apart at most
            # FFmpeg's IDCT, chroma upsampling and colour conversion are not libjpeg-turbo's: the luma stays within a
            # few levels, the colours differ more along sharp colour edges
            g = np.abs(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY).astype(np.int32)
                       - cv2.cvtColor(want.astype(np.uint8), cv2.COLOR_BGR2GRAY))
            assert g.max() <= 12 and g.mean() < 1.5
            assert np.abs(img.astype(np.int32) - want).mean() < 4
        assert not cap.read()[0]
    finally:
        cap.release()


def test_avi_refuses_bad_input(tmp_path):
    from osvos_pytorch_b200 import video
    path = str(tmp_path / "x.avi")
    with pytest.raises(ValueError):
        video.write_avi(path, [], 24)
    with pytest.raises(ValueError):
        video.write_avi(path, [b"not a jpeg"], 24)
    with pytest.raises(ValueError):
        video.write_avi(path, _jpegs(1, 16, 16, 0) + _jpegs(1, 16, 24, 0), 24)
    with pytest.raises(ValueError):
        video.write_avi(path, _jpegs(1, 16, 16, 0), 0)
    assert video.jpeg_size(_jpegs(1, 16, 24, 0)[0]) == (24, 16)


# ---- visualize_results.py ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("argv", [["--davis", "2017", "--threshold", "100"], ["--quality", "0"], ["--quality", "101"],
                                  ["--fps", "0"], ["--decode", "gpu"], ["--davis", "2018"]])
def test_cli_refuses_bad_arguments(argv, capsys):
    import visualize_results
    with pytest.raises(SystemExit) as e:
        visualize_results.main(argv)
    assert e.value.code == 2
    assert "error" in capsys.readouterr().err


def test_render_results_refuses_bad_arguments(tmp_path):
    from osvos_pytorch_b200 import visualize
    for kw in (dict(decode="gpu"), dict(davis="2018"), dict(quality=0), dict(frames=False, video=False),
               dict(fps=0), dict(palette=b"\0\0\0")):
        with pytest.raises(ValueError):
            visualize.render_results(str(tmp_path), str(tmp_path), **kw)
    os.makedirs(tmp_path / "db" / "JPEGImages" / "480p" / "s")
    os.makedirs(tmp_path / "res" / "s")
    (tmp_path / "res" / "s" / "00000.png").write_bytes(b"")
    with pytest.raises(ValueError, match="no frame for result"):
        visualize.render_results(str(tmp_path / "res"), str(tmp_path / "db"), sequences=["s"])
    with pytest.raises(ValueError, match="unknown sequence"):
        visualize.render_results(str(tmp_path / "res"), str(tmp_path / "db"), sequences=["t"])
    (tmp_path / "db" / "val_seqs.txt").write_text("t\n")
    with pytest.raises(ValueError, match="no sequence"):
        visualize.render_results(str(tmp_path / "res"), str(tmp_path / "db"))

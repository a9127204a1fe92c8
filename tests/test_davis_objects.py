"""DAVIS-2017 on the host (DESIGN.md §24): palette PNG parsing and its restatement against Pillow, the palette encoder's
restatement, the per-object count restatement against the DAVIS-2016 one, and the per-object statistics."""
import io
import math

import numpy as np
import pytest

import davis_measures_ref as M
import davis_objects_ref as O
import png_palette_ref as PP
import png_ref as P
from png_palette_ref import davis_palette, pillow_palette_png

Image = pytest.importorskip("PIL.Image")


def _labels(h, w, k, seed, void=False):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, k + 1, (h, w)).astype(np.uint8)
    a[: h // 3] = 0
    if void:
        a[:, w // 2:w // 2 + 2] = 255
    return a


# palette length -> the bit depth Pillow writes
DEPTHS = [(2, 1), (4, 2), (16, 4), (256, 8)]


@pytest.mark.parametrize("entries,depth", DEPTHS)
@pytest.mark.parametrize("w", [1, 7, 13, 33])
@pytest.mark.parametrize("trns", [None, 0])
def test_palette_restatement_equals_pillow(entries, depth, w, trns):
    from osvos_pytorch_b200 import png
    idx = _labels(11, w, min(entries, 256) - 1, seed=w + entries)
    data = pillow_palette_png(idx, entries, trns)
    got = png.parse(data, palette="index")
    assert isinstance(got, png.Parsed) and (got.depth, got.colour) == (depth, 3), got
    assert got.palette == davis_palette(entries)
    assert got.rowbytes == (w * depth + 7) // 8
    pil = np.array(Image.open(io.BytesIO(data)))
    ref, plte = PP.decode_index(data)
    assert np.array_equal(ref, pil) and np.array_equal(pil, idx)
    assert plte == got.palette == png.palette_of(data)
    assert np.array_equal(png.decode_host_index(data), pil)
    # the default mode keeps today's rule: a palette file is decoded by cv2 on the host
    assert isinstance(png.parse(data), png.Fallback)


def test_pack_records_the_colour_type():
    from osvos_pytorch_b200 import png
    a = pillow_palette_png(_labels(5, 9, 3, seed=1), 4)
    g = P.encode(_labels(5, 9, 3, seed=2))
    parsed = [png.parse(a, palette="index"), png.parse(g, palette="index")]
    blob = png.pack(parsed)
    hdr = png.HEADER.unpack_from(bytes(blob[:png.HEADER.size]))
    files = np.frombuffer(bytes(blob), png.FILE, 2, hdr[8])
    assert files["colour"].tolist() == [3, 0] and files["depth"].tolist() == [2, 8]


def test_palette_out_of_range_index_passes_through():
    """Indices beyond the palette are kept as they are, as Pillow keeps them."""
    from osvos_pytorch_b200 import png
    idx = np.array([[0, 1, 9, 3]], np.uint8)
    data = PP.encode(idx, davis_palette(4))
    assert np.array_equal(np.array(Image.open(io.BytesIO(data))), idx)
    assert np.array_equal(PP.decode_index(data)[0], idx)
    assert isinstance(png.parse(data, palette="index"), png.Parsed)


@pytest.mark.parametrize("shape", [(1, 1), (7, 13), (48, 640), (5, 17000)])
@pytest.mark.parametrize("entries", [1, 3, 256])
def test_palette_encoder_restatement(shape, entries):
    idx = _labels(*shape, k=min(entries, 255), seed=sum(shape))
    pal = davis_palette(entries)
    data = PP.encode(idx, pal)
    im = Image.open(io.BytesIO(data))
    assert im.mode == "P" and bytes(im.getpalette())[:3 * entries] == pal
    assert np.array_equal(np.array(im), idx)
    assert PP.strip_palette(data) == P.encode(idx)
    assert len(data) == len(P.encode(idx)) + 12 + 3 * entries


def test_single_object_without_void_equals_the_2016_counts():
    rng = np.random.default_rng(5)
    for h, w in [(30, 41), (64, 70)]:
        lab = (rng.random((h, w)) > 0.6).astype(np.uint8)
        gt = (rng.random((h, w)) > 0.55).astype(np.uint8)
        r = M.bound_pix(h, w)
        want = M.counts(np.where(lab == 1, 1.0, -1.0).astype(np.float32), gt, r)
        assert O.object_counts(lab, gt, 1, r) == [want]


def test_void_is_cleared_from_both_masks():
    lab = np.zeros((20, 20), np.uint8)
    gt = np.zeros((20, 20), np.uint8)
    lab[5:15, 5:15] = 1
    gt[5:15, 5:15] = 1
    gt[5:15, 10] = 255                                          # a void band through the object
    c, = O.object_counts(lab, gt, 1, 2)
    assert c[0] == c[1] == 90                                   # the band counts in neither mask
    lab2 = lab.copy()
    lab2[gt == 255] = 0
    assert c == M.counts(np.where(lab2 == 1, 1.0, -1.0).astype(np.float32), (gt == 1).astype(np.uint8), 2)


def test_absent_object_and_merge_rule():
    lab = np.zeros((8, 8), np.uint8)
    gt = np.zeros((8, 8), np.uint8)
    gt[2:4, 2:4] = 1
    c = O.object_counts(lab, gt, 2, 1)
    assert c[1] == [0, 0, 0, 0, 0, 0]                           # object 2: absent from both -> J = F = 1
    assert M.j_and_f(c[1]) == (1.0, 1.0)
    maps = np.array([[1.0, 2.0, 0.0, -0.0, np.nan, 3.0], [2.0, 2.0, -1.0, 0.0, 1.0, np.nan]], np.float32)
    assert O.merge(maps).tolist() == [2, 1, 0, 0, 2, 1]


def test_object_statistics_and_global_table():
    import torch

    from osvos_pytorch_b200 import evaluation
    rng = np.random.default_rng(11)
    per_seq, ref_stats = {}, []
    for seq, (frames, k) in {"a": (7, 2), "b": (5, 3)}.items():
        counts = np.zeros((frames, k, 6), np.int32)
        counts[..., 1] = rng.integers(1, 100, (frames, k))
        counts[..., 0] = (counts[..., 1] * rng.random((frames, k))).astype(np.int32)
        counts[..., 2:4] = rng.integers(0, 40, (frames, k, 2))
        counts[..., 4] = (counts[..., 2] * rng.random((frames, k))).astype(np.int32)
        counts[..., 5] = (counts[..., 3] * rng.random((frames, k))).astype(np.int32)
        sc = evaluation.ObjectScores(k)
        sc.add(torch.from_numpy(counts[:3]))
        sc.add(torch.from_numpy(counts[3:]))
        res = sc.result()
        assert sorted(res["objects"]) == list(range(1, k + 1))
        for j in range(k):
            jf = [M.j_and_f(counts[t, j]) for t in range(frames)]
            ob = res["objects"][j + 1]
            assert np.allclose(ob["J"], [x for x, _ in jf]) and np.allclose(ob["F"], [y for _, y in jf])
            sj, sf = M.statistics([x for x, _ in jf]), M.statistics([y for _, y in jf])
            assert np.allclose([ob["statistics"]["J"][m] for m in "MOD"], sj)
            assert np.allclose([ob["statistics"]["F"][m] for m in "MOD"], sf)
            ref_stats.append((sj, sf))
        per_seq[seq] = sc if seq == "a" else res
    d = evaluation.dataset_scores_objects(per_seq)
    assert d["objects"] == 5
    for i, m in enumerate("MOD"):
        assert math.isclose(d["J"][m], np.mean([s[0][i] for s in ref_stats]))
        assert math.isclose(d["F"][m], np.mean([s[1][i] for s in ref_stats]))
    assert math.isclose(d["J&F"], (d["J"]["M"] + d["F"]["M"]) / 2)
    assert evaluation.n_objects(np.array([[0, 3, 255], [1, 0, 2]], np.uint8)) == 3

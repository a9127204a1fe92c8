"""CPU checks of the online adaptation targets' restatement (tests/adaptation_ref.py) on hand-made cases, and of the
argument refusals of train_online.py --adapt."""
import numpy as np
import pytest
from scipy import ndimage

import adaptation_ref as ref


def disk(e):
    y, x = np.mgrid[-e:e + 1, -e:e + 1]
    return x * x + y * y <= e * e


def test_threshold_is_the_float32_logit_of_alpha():
    assert ref.threshold(0.5) == np.float32(0.0)
    assert ref.threshold(0.97) == np.float32(np.log(0.97 / 0.03))


def test_single_pixel():
    m = np.zeros((9, 11), np.uint8)
    m[4, 6] = 1
    assert ref.eroded(m, 0).sum() == 1
    assert ref.eroded(m, 1).sum() == 0                  # its background neighbours are at distance 1
    logits = np.zeros((9, 11), np.float32)
    labels, counts = ref.frame_labels(logits, m, 0.5, 0, 2)
    i, j = np.indices(m.shape)
    near = (i - 4) ** 2 + (j - 6) ** 2 <= 4
    assert np.array_equal(labels == 0, ~near)
    assert np.all(labels[near] == -1)                   # logit 0 equals the threshold of alpha 0.5: not positive
    assert counts.tolist() == [1, 0, int((~near).sum())]


def test_full_frame_is_not_eroded():
    m = np.full((6, 7), 255, np.uint8)
    for e in (0, 3, 100):
        assert ref.eroded(m, e).all()
    labels, counts = ref.frame_labels(np.ones((6, 7), np.float32), m, 0.5, 5, 0)
    assert (labels == 1).all() and counts.tolist() == [42, 42, 0]


def test_empty_mask_has_no_negatives():
    m = np.zeros((5, 8), np.uint8)
    logits = np.linspace(-3, 3, 40, dtype=np.float32).reshape(5, 8)
    labels, counts = ref.frame_labels(logits, m, 0.5, 0, 0)
    assert counts.tolist() == [0, int((logits > 0).sum()), 0]
    assert np.array_equal(labels, np.where(logits > 0, 1.0, -1.0).astype(np.float32))


@pytest.mark.parametrize("side", ["top", "bottom", "left", "right"])
def test_mask_touching_a_border_is_not_eroded_from_it(side):
    h, w, e = 20, 24, 3
    m = np.zeros((h, w), np.uint8)
    sl = {"top": (slice(0, 8), slice(6, 18)), "bottom": (slice(h - 8, h), slice(6, 18)),
          "left": (slice(6, 14), slice(0, 10)), "right": (slice(6, 14), slice(w - 10, w))}[side]
    m[sl] = 1
    e_set = ref.eroded(m, e)
    assert np.array_equal(e_set, ndimage.binary_erosion(m != 0, structure=disk(e), border_value=1))
    edge = {"top": e_set[0], "bottom": e_set[-1], "left": e_set[:, 0], "right": e_set[:, -1]}[side]
    assert edge.any()                                   # the frame's edge is not background


def test_erosion_zero_keeps_the_mask_and_distance_zero_negates_everything_outside_it():
    rng = np.random.default_rng(1)
    m = (rng.random((17, 23)) > 0.6).astype(np.uint8)
    assert np.array_equal(ref.eroded(m, 0), m != 0)
    labels, counts = ref.frame_labels(np.full((17, 23), 9.0, np.float32), m, 0.97, 0, 0)
    assert np.array_equal(labels, np.where(m != 0, 1.0, 0.0).astype(np.float32))
    assert counts.tolist() == [int(m.sum()), int(m.sum()), int((m == 0).sum())]


def test_distance_beyond_the_diagonal_has_no_negatives():
    m = np.zeros((30, 40), np.uint8)
    m[0, 0] = 1
    labels, counts = ref.frame_labels(np.zeros((30, 40), np.float32), m, 0.97, 0, 50)   # 50² = 29² + 39² + 58
    assert counts[2] == 0 and (labels == -1).all()
    _, counts = ref.frame_labels(np.zeros((30, 40), np.float32), m, 0.97, 0, 48)
    assert counts[2] == 2                                # (29, 39) and (28, 39): 2362 and 2305 > 48² = 2304


@pytest.mark.parametrize("seed", range(6))
def test_erosion_matches_binary_erosion_by_a_disk(seed):
    rng = np.random.default_rng(seed)
    h, w = rng.integers(5, 60, size=2)
    m = ndimage.gaussian_filter(rng.random((h, w)), 2.5) > 0.5
    for e in (0, 1, 2, 4, 7):
        want = m if e == 0 else ndimage.binary_erosion(m, structure=disk(e), border_value=1)
        assert np.array_equal(ref.eroded(m.astype(np.uint8), e), want)


def test_squared_distances_are_exact_integers():
    rng = np.random.default_rng(3)
    f = rng.random((13, 19)) > 0.9
    got = ref.squared_distance_to(f)
    qi, qj = np.nonzero(f)
    i, j = np.indices(f.shape)
    brute = ((i[..., None] - qi) ** 2 + (j[..., None] - qj) ** 2).min(-1)
    assert got.dtype == np.int64 and np.array_equal(got, brute)


# ---- train_online.py --adapt argument refusals ----------------------------------------------------------------------

def _parse(argv):
    import train_online
    return train_online.parse(argv)


def test_adapt_parses_with_native_loader():
    a = _parse(["--loader", "native", "--adapt", "--adapt-steps", "7", "--adapt-current-steps", "2", "--adapt-weight",
                "0.1", "--adapt-alpha", "0.9", "--adapt-distance", "100", "--adapt-erosion", "5", "--input-res", "240",
                "427", "--output-res", "stored", "--decode", "device", "--encode", "device", "--overlay", "--evaluate",
                "--deterministic"])
    assert a.adapt and (a.adapt_steps, a.adapt_current_steps, a.adapt_distance, a.adapt_erosion) == (7, 2, 100, 5)
    assert (a.adapt_weight, a.adapt_alpha) == (0.1, 0.9)
    d = _parse(["--loader", "native", "--adapt"])
    assert (d.adapt_steps, d.adapt_current_steps, d.adapt_weight, d.adapt_alpha, d.adapt_distance,
            d.adapt_erosion) == (15, 3, 0.05, 0.97, 220, 15)


@pytest.mark.parametrize("argv", [
    ["--adapt"],                                                   # --loader reference (the default)
    ["--loader", "reference", "--adapt"],
    ["--synthetic", "--adapt"],
    ["--loader", "native", "--davis", "2017", "--adapt"],
    ["--loader", "native", "--adapt", "--upsampling-lr", "1e-8"],
    ["--loader", "native", "--adapt", "--adapt-alpha", "1.0"],
    ["--loader", "native", "--adapt", "--adapt-alpha", "0"],
    ["--loader", "native", "--adapt", "--adapt-distance", "-1"],
    ["--loader", "native", "--adapt", "--adapt-erosion", "-2"],
    ["--loader", "native", "--adapt", "--adapt-steps", "-1"],
    ["--loader", "native", "--adapt", "--adapt-steps", "2", "--adapt-current-steps", "3"],
    ["--loader", "native", "--adapt-steps", "4"],                  # an --adapt-* option without --adapt
])
def test_adapt_refusals(argv, capsys):
    with pytest.raises(SystemExit) as ex:
        _parse(argv)
    assert ex.value.code == 2
    assert "--adapt" in capsys.readouterr().err

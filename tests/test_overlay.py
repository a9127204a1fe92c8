"""The overlay rule (tests/overlay_ref.py) against cv2's contours and against the reference's own overlay_mask."""
import os

import numpy as np
import pytest

import overlay_ref

cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_overlay.npz")


def _drawn(mask):
    """The pixels the reference's cv2.drawContours(findContours(m, RETR_TREE, CHAIN_APPROX_SIMPLE), -1, 0, 1) paints."""
    contours = cv2.findContours(mask.astype(np.uint8), cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)[-2]
    canvas = np.zeros(mask.shape, np.uint8)
    cv2.drawContours(canvas, contours, -1, 1, 1)
    return canvas.astype(bool)


def _masks():
    rng = np.random.default_rng(4)
    out = {}
    m = np.zeros((20, 24), bool)
    m[3:17, 4:20] = True
    m[8:12, 9:14] = False
    out["hole"] = m
    m = np.zeros((15, 15), bool)
    m[7, 2:13] = True
    m[2:13, 3] = True
    out["lines"] = m
    out["diagonal"] = np.eye(12, dtype=bool) | np.eye(12, k=3, dtype=bool)
    m = np.zeros((10, 13), bool)
    m[0:4, :] = True
    m[:, 10:] = True
    out["touching"] = m
    out["empty"] = np.zeros((9, 11), bool)
    out["full"] = np.ones((9, 11), bool)
    out["single"] = np.pad(np.ones((1, 1), bool), 3)
    for k in range(40):
        h, w = (int(v) for v in rng.integers(1, 60, 2))
        if k % 2:
            out[f"noise{k}"] = rng.random((h, w)) > 0.5
        else:
            yy, xx = np.mgrid[0:h, 0:w]
            out[f"blob{k}"] = np.sin(xx / (2 + k % 5)) * np.cos(yy / (3 + k % 7)) > 0.2
    return out


@pytest.mark.parametrize("name", list(_masks()))
def test_edge_is_what_draw_contours_paints(name):
    m = _masks()[name]
    assert np.array_equal(overlay_ref.edge(m), _drawn(m)), name


def test_overlay_is_within_half_a_level_of_the_reference():
    g = np.load(GOLDEN)
    ks = sorted(int(k.split(":")[1]) for k in g.files if k.startswith("frame:"))
    assert ks
    for k in ks:
        frame, mask, ref = g[f"frame:{k}"], g[f"mask:{k}"].astype(bool), g[f"out:{k}"].astype(np.float64) * 255
        logits = np.where(mask, 1.0, -1.0).astype(np.float32)
        got = overlay_ref.overlay(frame[None], logits[None])[0].astype(np.float64)
        e = overlay_ref.edge(mask)
        # the reference paints its contour black on the foreground only (its red blend is never 0 there)
        assert np.array_equal((ref == 0).all(-1) & mask, e)
        assert (got[e] == 0).all()
        blend = mask & ~e
        assert blend.any() and np.abs(got[blend] - ref[blend]).max() <= 0.5 + 1e-3
        assert np.array_equal(got[~mask], frame[~mask])
        assert np.all(np.abs(ref[~mask] - frame[~mask]) < 1e-3)


def test_zero_and_nan_logits_are_background():
    frame = np.full((1, 3, 4, 3), 100, np.uint8)
    logits = np.array([[[1.0, 0.0, -0.0, np.nan], [1.0, 1.0, 1.0, 1.0], [1.0, 1.0, 1.0, 1.0]]], np.float32)
    got = overlay_ref.overlay(frame, logits, color=(10, 20, 30))
    assert (got[0, 0, 1:] == 100).all()
    assert (got[0, 0, 0] == 0).all() and (got[0, 1, 3] == 0).all()
    assert (got[0, 1, 1] == 0).all()                                # its upper neighbour is 0.0
    g = overlay_ref.overlay(np.full((1, 5, 5, 3), 100, np.uint8), np.ones((1, 5, 5), np.float32), color=(10, 21, 255))
    assert tuple(g[0, 2, 2]) == (55, 61, 178)                       # (v + c + 1) >> 1

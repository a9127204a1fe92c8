"""The restatement of the component filter (tests/components_ref.py, DESIGN.md §30) on hand-made cases, scipy's
numbering, and train_online.py's --components options.  CPU only."""
import numpy as np
import pytest

import components_ref as ref


def _z(fg, value=1.0):
    return np.where(np.asarray(fg, bool), np.float32(value), np.float32(-1.0)).astype(np.float32)


@pytest.mark.parametrize("connectivity", [4, 8])
def test_scipy_numbers_components_in_raster_order_of_their_first_pixel(connectivity):
    rng = np.random.default_rng(0)
    for t in range(300):
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        mask = rng.random((h, w)) < rng.choice([0.2, 0.45, 0.6])
        lab, n = ref.label(mask, connectivity)
        firsts = [int(np.flatnonzero(lab.ravel() == i)[0]) for i in range(1, n + 1)]
        assert firsts == sorted(firsts), (t, connectivity)
        assert set(np.unique(lab)) <= set(range(n + 1)) and (lab > 0).sum() == mask.sum()


def test_diagonal_touch_joins_at_8_not_at_4():
    m = np.zeros((4, 4), np.uint8)
    m[1, 1] = m[2, 2] = 1
    assert ref.label(m, 8)[1] == 1 and ref.label(m, 4)[1] == 2
    z = _z(m)[None, None]
    _, kept8, st8 = ref.filter_components(z, "largest", connectivity=8)
    _, kept4, st4 = ref.filter_components(z, "largest", connectivity=4)
    assert st8[0, 0].tolist() == [1, 1, 2, 0] and kept8.sum() == 2
    assert st4[0, 0].tolist() == [2, 1, 2, 1] and kept4[0, 0, 1, 1] == 1 and kept4[0, 0, 2, 2] == 0


def test_tie_for_largest_goes_to_the_smallest_label():
    fg = np.zeros((5, 9), bool)
    fg[3, 0:3] = True          # label 2 (its first pixel comes later)
    fg[0, 6:9] = True          # label 1
    z = _z(fg, 2.5)
    out, kept, st = ref.filter_frame(z, None, "largest", 32, 8)
    assert kept[0, 6:9].all() and not kept[3].any()
    assert np.array_equal(out[3, 0:3], np.float32([-2.5] * 3)) and np.array_equal(out[0, 6:9], z[0, 6:9])
    assert st.tolist() == [2, 1, 6, 3]


# (radius, a pixel at squared distance exactly radius² from the prior pixel (10, 10), one at the next squared distance
# that a lattice point reaches: radius² + 1, or 2 when radius is 0); the two are never 4-neighbours
RADIUS_CASES = [(0, (10, 10), (11, 11)), (3, (13, 10), (11, 13)), (5, (13, 14), (11, 15))]


@pytest.mark.parametrize("radius,at,beyond", RADIUS_CASES)
def test_distance_exactly_radius_squared_is_kept_and_one_more_is_dropped(radius, at, beyond):
    h, w = 30, 40
    prior = np.zeros((h, w), bool)
    prior[10, 10] = True
    fg = np.zeros((h, w), bool)
    fg[0:3, 30:40] = True                          # the largest, far from the prior
    fg[at] = fg[beyond] = True
    d2 = lambda p: (p[0] - 10) ** 2 + (p[1] - 10) ** 2
    assert d2(at) == radius * radius and d2(beyond) == (radius * radius + 1 if radius else 2)
    out, kept, st = ref.filter_frame(_z(fg), prior, "near", radius, 4)
    assert kept[at] and not kept[beyond] and not kept[0:3].any()
    assert st.tolist() == [3, 1, int(fg.sum()), int(fg.sum()) - 1]
    assert out[beyond] == -1.0 and out[at] == 1.0


def test_empty_prior_and_no_near_component_keep_the_largest():
    fg = np.zeros((20, 20), bool)
    fg[0:4, 0:4] = True
    fg[15:17, 15:17] = True
    z = _z(fg)
    want = ref.filter_frame(z, None, "largest", 32, 8)
    for prior in (None, np.zeros((20, 20), bool)):
        got = ref.filter_frame(z, prior, "near", 32, 8)
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
    far = np.zeros((20, 20), bool)
    far[19, 0] = True                              # more than 2 pixels from both components
    got = ref.filter_frame(z, far, "near", 2, 8)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert got[1][0:4, 0:4].all() and not got[1][15:17, 15:17].any()


def test_near_keeps_every_component_in_reach_and_chains_frames():
    h, w = 16, 24
    maps = np.full((1, 3, h, w), -1.0, np.float32)
    maps[0, :, 2:6, 2:6] = 1.0                     # the object
    maps[0, :, 10:16, 16:24] = 1.0                 # a larger blob far away
    maps[0, 1, 2:4, 7:9] = 1.0                     # a fragment close to the object
    prior = np.zeros((1, h, w), np.uint8)
    prior[0, 3, 3] = 1
    out, kept, st = ref.filter_components(maps, "near", radius=3, connectivity=8, prior=prior)
    assert st[0, :, 1].tolist() == [1, 2, 1] and st[0, :, 0].tolist() == [2, 3, 2]
    assert kept[0, 1, 2:4, 7:9].all() and not kept[0, :, 10:].any()
    assert (out[0, :, 10:16, 16:24] == -1.0).all()
    # frame 2 is measured against frame 1's kept mask (object and fragment), so it keeps the object
    assert kept[0, 2, 2:6, 2:6].all()


def test_nan_and_signed_zero_are_background_and_keep_their_bits():
    z = np.full((3, 5), -2.0, np.float32)
    z[0, 0], z[0, 1], z[0, 2] = np.nan, 0.0, -0.0
    z[2, 2:5] = 3.0                                # the only component
    z[0, 4] = 1.0                                  # a dropped one
    out, kept, st = ref.filter_frame(z, None, "largest", 32, 8)
    assert np.isnan(out[0, 0]) and out[0, 1] == 0 and not np.signbit(out[0, 1]) and np.signbit(out[0, 2])
    assert out[0, 4] == -1.0 and (out[2, 2:5] == 3.0).all() and st.tolist() == [2, 1, 4, 1]
    assert kept.sum() == 3


def test_one_component_largest_returns_the_map():
    rng = np.random.default_rng(3)
    z = rng.standard_normal((9, 11)).astype(np.float32) - 8
    z[2:5, 3:8] = np.abs(z[2:5, 3:8]) + 0.5
    out, _, st = ref.filter_frame(z, None, "largest", 32, 8)
    assert st[0] == 1 and out.tobytes() == z.tobytes()


# ---- train_online.py --components ---------------------------------------------------------------------------------

def test_cli_parses_components():
    import train_online
    a = train_online.parse(["--components", "largest"])
    assert a.components_params.mode == "largest" and a.components_params.radius == 32
    assert a.components_params.connectivity == 8
    a = train_online.parse(["--components", "near", "--components-radius", "7", "--components-connectivity", "4",
                            "--loader", "native", "--davis", "2017"])
    assert (a.components_params.mode, a.components_params.radius, a.components_params.connectivity) == ("near", 7, 4)
    assert train_online.parse([]).components_params is None
    assert train_online.parse(["--components", "largest", "--synthetic"]).components_params is not None


@pytest.mark.parametrize("argv", [
    ["--components-radius", "5"],
    ["--components-connectivity", "4"],
    ["--components", "largest", "--components-radius", "5"],
    ["--components", "near", "--components-radius", "-1"],
    ["--components", "near", "--components-connectivity", "6"],
    ["--components", "biggest"],
])
def test_cli_refuses_bad_components_options(argv, capsys):
    import train_online
    with pytest.raises(SystemExit):
        train_online.parse(argv)
    assert "components" in capsys.readouterr().err


def test_components_parameters_are_validated():
    from osvos_pytorch_b200 import ops
    for kw in (dict(mode="big"), dict(mode="near", radius=-1), dict(mode="near", radius=1.5),
               dict(mode="near", radius=True), dict(mode="largest", connectivity=6),
               dict(mode="largest", connectivity=True)):
        with pytest.raises(ValueError):
            ops.Components(**kw)
    assert ops.Components("near") == ops.Components("near", radius=32, connectivity=8)

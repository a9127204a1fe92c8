"""CPU checks of the dense CRF's float64 restatement (tests/crf_ref.py, DESIGN.md §29) against its defining properties,
of ops.CRF's validation, and of train_online.py's --crf flags.  The device kernel is held to the restatement by
tests/test_gpu_crf.py."""
import numpy as np
import pytest
from scipy import ndimage

import crf_ref as ref


def _frames(seed, n, h, w):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("seed,shape,thetas", [(0, (1, 1, 1), (80.0, 13.0)), (1, (2, 7, 5), (80.0, 13.0)),
                                               (2, (1, 33, 45), (5.0, 3.0)), (3, (1, 12, 9), (0.7, 0.4))])
def test_barycentric_weights_are_a_partition_of_one(seed, shape, thetas):
    keys, wts = ref.elevate(_frames(seed, *shape), *thetas)
    assert np.all(wts >= 0)
    assert np.allclose(wts.sum(1), 1.0, rtol=0, atol=1e-12)
    # the 6 vertices of a simplex are distinct, one per remainder class
    assert all(len(set(row)) == 6 for row in keys.tolist())


def test_weights_interpolate_the_elevated_point():
    """Σ_r w_r · vertex_r is the elevated feature itself (the barycentric coordinates of the simplex)."""
    frames = _frames(4, 1, 6, 8)
    keys, wts = ref.elevate(frames, 7.0, 9.0)
    _, _, k = ref.decode(keys.ravel())
    k6 = np.vstack([k, -k.sum(0)]).reshape(6, -1, 6)           # coordinate, pixel, vertex
    point = np.einsum("cpr,pr->pc", k6, wts)
    s = ref.scales(7.0, 9.0)
    yy, xx = np.mgrid[0:6, 0:8]
    v = [xx.ravel(), yy.ravel(), frames[0, ..., 2].ravel(), frames[0, ..., 1].ravel(), frames[0, ..., 0].ravel()]
    cf = [v[j] * s[j] for j in range(5)]
    e = np.zeros((6, 48))
    for j in range(5, 0, -1):
        e[j] = sum(cf[j:]) - j * cf[j - 1]
    e[0] = sum(cf)
    assert np.allclose(point, e.T, rtol=0, atol=1e-9)


def test_filter_of_one_normalises_to_one():
    frames = _frames(5, 2, 9, 11)
    lat = ref.Lattice(frames, 4.0, 20.0)
    f1 = lat.filter(np.ones((lat.pixels, 1)))
    assert np.all(f1 > 0)
    assert np.allclose(f1 / f1, 1.0)


def _blur_matrix(lat, j):
    m = np.zeros((lat.m, lat.m))
    idx = np.arange(lat.m)
    m[idx, idx] = 0.5
    for nb in lat.nbr[j]:
        ok = nb >= 0
        m[idx[ok], nb[ok]] += 0.25
    return m


def test_each_directional_blur_is_symmetric_and_the_filter_adjoint_reverses_them():
    """Each direction's blur is a symmetric operator on the lattice's vertices (v is u's lower neighbour exactly when u
    is v's upper one).  On a sparse lattice the six blurs do not commute, so the unnormalised F = Sᵀ B₅⋯B₀ S is not
    itself symmetric; its adjoint is the same filter with the directions in reverse order: ⟨u, F v⟩ = ⟨F' u, v⟩."""
    frames = _frames(6, 1, 10, 13)
    lat = ref.Lattice(frames, 3.0, 30.0)
    for j in range(6):
        b = _blur_matrix(lat, j)
        assert np.array_equal(b, b.T)
    rng = np.random.default_rng(7)
    u, v = rng.standard_normal((lat.pixels, 1)), rng.standard_normal((lat.pixels, 1))
    lhs, rhs = float((u * lat.filter(v)).sum()), float((lat.filter(u, reverse=True) * v).sum())
    assert lhs == pytest.approx(rhs, rel=1e-12, abs=1e-12)


def test_filter_is_symmetric_where_every_neighbour_is_present():
    """Where the blurs commute (a lattice whose every vertex is one simplex: one pixel), F is symmetric."""
    frames = _frames(14, 3, 1, 1)
    lat = ref.Lattice(frames, 80.0, 13.0)
    f = np.stack([lat.filter(np.eye(lat.pixels)[:, i:i + 1])[:, 0] for i in range(lat.pixels)], 1)
    assert np.allclose(f, f.T, rtol=0, atol=1e-15)


def test_constant_image_averages_over_the_frame():
    """Every pixel at one feature point (1x1 frames, one colour) -> one simplex: B_l = the mean of Q_l."""
    n = 1
    frames = np.zeros((n, 1, 1, 3), dtype=np.uint8) + 77
    frames = np.repeat(frames, 5, axis=0)                       # 5 frames, each its own lattice
    lat = ref.Lattice(frames, 80.0, 13.0)
    assert lat.per_frame.tolist() == [6] * 5
    # one frame of many pixels at one feature: the position scale so large that every pixel rounds to one point
    frames = np.full((1, 4, 6, 3), 200, dtype=np.uint8)
    lat = ref.Lattice(frames, 1e9, 13.0)
    rng = np.random.default_rng(8)
    q = rng.random((lat.pixels, 3))
    b = lat.filter(q) / lat.filter(np.ones((lat.pixels, 1)))
    assert np.allclose(b, q.mean(0, keepdims=True), rtol=1e-12)


def _structured_frame(h, w):
    """A colour ramp in x, y and x + y with a flat blob: edges in colour as well as in position."""
    yy, xx = np.mgrid[0:h, 0:w]
    f = np.stack([xx * 255 // (w - 1), yy * 255 // (h - 1), (3 * xx + 5 * yy) % 256], -1)
    f[(xx - w / 3) ** 2 + (yy - h / 2) ** 2 < (h / 3) ** 2] = (200, 60, 90)
    return f.astype(np.uint8)[None]


@pytest.mark.parametrize("thetas", [(3.0, 13.0), (5.0, 20.0), (8.0, 30.0)])
def test_lattice_filter_has_the_width_the_parameters_name(thetas):
    """The normalised lattice filter F(Q)/F(1) approximates the dense Gaussian exp(-|Δf|² / 2) of
    f = (x/θα, y/θα, R/θβ, G/θβ, B/θβ) (DESIGN §29), and that Gaussian better than the same one at scale 0.7 or 1.4:
    the lattice's scale factors give the filter the width θα, θβ name, not one that is off by a constant factor.
    The approximation itself (one simplex per pixel, a 3-tap blur per direction) errs by a few hundredths here."""
    h, w = 24, 32
    frames = _structured_frame(h, w)
    u = np.random.default_rng(15).random(h * w)
    q = np.stack([u, 1 - u], 1)
    lat = ref.Lattice(frames, *thetas)
    b = lat.filter(q) / lat.filter(np.ones((lat.pixels, 1)))
    yy, xx = np.mgrid[0:h, 0:w]
    px = frames[0].reshape(-1, 3).astype(np.float64)
    ta, tb = thetas
    feat = np.stack([xx.ravel() / ta, yy.ravel() / ta, px[:, 2] / tb, px[:, 1] / tb, px[:, 0] / tb], 1)
    d2 = ((feat[:, None] - feat[None]) ** 2).sum(-1)
    err = {}
    for s in (0.7, 1.0, 1.4):
        k = np.exp(-d2 / (2 * s * s))
        diff = b - k @ q / k.sum(1, keepdims=True)
        err[s] = (float(np.abs(diff).max()), float(np.sqrt((diff ** 2).mean())))
    assert err[1.0][0] < 0.08 and err[1.0][1] < 0.015, err
    for s in (0.7, 1.4):
        assert err[1.0][0] < err[s][0] and 2 * err[1.0][1] < err[s][1], err


@pytest.mark.parametrize("theta,shape", [(3.0, (2, 20, 31)), (0.4, (1, 5, 6)), (1.7, (1, 3, 40)), (5.0, (1, 8, 8))])
def test_gaussian_message_is_the_truncated_correlation_renormalised(theta, shape):
    rng = np.random.default_rng(9)
    q = rng.random((2,) + shape)
    g = ref.gaussian_taps(theta)
    kern = np.outer(g, g)
    got = ref.smoothness(q, theta)
    for ql, sl in zip(q, got):
        for f in range(shape[0]):
            num = ndimage.correlate(ql[f], kern, mode="constant", cval=0.0)
            den = ndimage.correlate(np.ones(shape[1:]), kern, mode="constant", cval=0.0)
            assert np.allclose(sl[f], num / den, rtol=1e-12, atol=0)


def test_zero_iterations_return_the_maps():
    frames = _frames(10, 1, 4, 5)
    z = np.random.default_rng(11).standard_normal((3, 1, 4, 5)).astype(np.float32)
    assert np.array_equal(ref.dense_crf(frames, z, iterations=0), z.astype(np.float64))


def test_one_object_matches_the_sigmoid_form():
    """K = 1: Q⁰ = (1 - σ(z), σ(z)), and without messages the refined logit is z."""
    frames = _frames(12, 1, 6, 7)
    z = np.random.default_rng(13).standard_normal((1, 1, 6, 7))
    q0 = ref.softmax(np.concatenate([np.zeros_like(z), z]))
    assert np.allclose(q0[1], 1 / (1 + np.exp(-z)))
    r = ref.dense_crf(frames, z, iterations=3, w_a=0.0, w_g=0.0)
    assert np.allclose(r, z)


def test_messages_pull_an_outlier_towards_its_neighbours():
    """A uniform frame, confident foreground except one background pixel: the CRF raises that pixel's logit."""
    frames = np.full((1, 9, 9, 3), 90, dtype=np.uint8)
    z = np.full((1, 1, 9, 9), 4.0)
    z[0, 0, 4, 4] = -1.0
    r = ref.dense_crf(frames, z)
    assert r[0, 0, 4, 4] > 0
    assert np.all(r > 0)


# ---- ops.CRF validation (no GPU needed) ------------------------------------------------------------------------------

def test_crf_defaults_and_validation():
    from osvos_pytorch_b200 import ops
    c = ops.CRF()
    assert (c.iterations, c.bilateral_weight, c.bilateral_xy, c.bilateral_rgb, c.gaussian_weight, c.gaussian_xy) == \
        (5, 10.0, 80.0, 13.0, 3.0, 3.0)
    ops.CRF(iterations=0, bilateral_weight=0, gaussian_weight=0.0)
    for bad in (dict(iterations=-1), dict(iterations=2.0), dict(iterations=True), dict(bilateral_weight=-1.0),
                dict(gaussian_weight=float("nan")), dict(bilateral_xy=0.0), dict(bilateral_rgb=-3.0),
                dict(gaussian_xy=float("inf")), dict(bilateral_xy="80")):
        with pytest.raises(ValueError):
            ops.CRF(**bad)
    with pytest.raises(Exception):
        c.iterations = 3                                          # frozen


# ---- train_online.py --crf ------------------------------------------------------------------------------------------

def _parse(argv):
    import train_online
    return train_online.parse(argv)


def test_crf_parses_with_native_loader():
    from osvos_pytorch_b200 import ops
    a = _parse(["--loader", "native", "--crf", "--crf-iterations", "3", "--crf-bilateral", "5", "60", "10",
                "--crf-gaussian", "2", "1.5", "--evaluate"])
    assert a.crf_params == ops.CRF(3, 5.0, 60.0, 10.0, 2.0, 1.5)
    assert _parse(["--loader", "native", "--crf"]).crf_params == ops.CRF()
    d = _parse(["--loader", "native", "--davis", "2017", "--crf", "--input-res", "240", "427", "--output-res", "stored"])
    assert d.crf_params == ops.CRF()
    assert _parse(["--loader", "native"]).crf_params is None


@pytest.mark.parametrize("argv", [
    ["--crf"],                                                     # --loader reference (the default)
    ["--loader", "reference", "--crf"],
    ["--synthetic", "--crf"],
    ["--loader", "native", "--crf-iterations", "3"],               # a --crf-* option without --crf
    ["--loader", "native", "--crf-bilateral", "1", "2", "3"],
    ["--loader", "native", "--crf-gaussian", "1", "2"],
    ["--loader", "native", "--crf", "--crf-iterations", "-1"],
    ["--loader", "native", "--crf", "--crf-bilateral", "-1", "80", "13"],
    ["--loader", "native", "--crf", "--crf-bilateral", "10", "0", "13"],
    ["--loader", "native", "--crf", "--crf-gaussian", "3", "nan"],
])
def test_crf_refusals(argv, capsys):
    with pytest.raises(SystemExit) as ex:
        _parse(argv)
    assert ex.value.code == 2
    assert "--crf" in capsys.readouterr().err

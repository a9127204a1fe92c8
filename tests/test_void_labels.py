"""Void labels on the CPU: the fp64 restatement of the void-aware class-balanced BCE (void_loss_ref) against the oracle's
loss and analytic cases, the id-mode warp's host restatement against cv2, the compiled void kernels, and the argument
refusals of train_parent.py --davis 2017 and train_online.py --ignore-void."""
import subprocess

import numpy as np
import pytest
import torch

from oracle import osvos_oracle as oc
import void_loss_ref as V


def _case(seed, shape=(2, 1, 13, 17), p_void=0.0, p_pos=0.3):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 3, shape)
    u = rng.random(shape)
    y = np.where(u < p_void, -1.0, np.where(u < p_void + p_pos, 1.0, 0.0))
    return x, y


@pytest.mark.parametrize("divisor", [1.0, 2.0])
def test_without_void_equals_the_oracle(divisor):
    x, y = _case(1)
    loss, g = V.void_loss(x, y, divisor)
    xt, yt = torch.from_numpy(x), torch.from_numpy(y)
    ref = oc.class_balanced_cross_entropy_loss(xt, yt, size_average=False, batch_average=divisor == 2.0)
    gref = oc.class_balanced_cross_entropy_grad(xt, yt, size_average=False, batch_average=divisor == 2.0)
    assert abs(loss - float(ref)) <= 1e-12 * abs(float(ref))
    assert np.abs(g - gref.numpy()).max() <= 1e-15
    assert abs(float(V.void_loss_torch(xt, yt, divisor)) - loss) <= 1e-12 * abs(loss)


def test_void_pixels_get_zero_gradient_and_do_not_count():
    x, y = _case(2, p_void=0.3)
    loss, g = V.void_loss(x, y)
    assert np.all(g[y < 0] == 0) and np.all(g[y >= 0] != 0)
    keep = y >= 0                          # the loss of the non-void pixels alone, as one flat tensor
    ref = oc.class_balanced_cross_entropy_loss(torch.from_numpy(x[keep]), torch.from_numpy(y[keep]),
                                               size_average=False, batch_average=False)
    assert abs(loss - float(ref)) <= 1e-12 * abs(float(ref))
    # the gradient is the derivative of the loss (central differences at a few pixels)
    for i in np.flatnonzero(keep)[:5]:
        e = np.zeros(x.size)
        e[i] = 1e-6
        lp, _ = V.void_loss(x + e.reshape(x.shape), y)
        lm, _ = V.void_loss(x - e.reshape(x.shape), y)
        assert abs((lp - lm) / 2e-6 - g.flat[i]) <= 1e-6 * max(1.0, abs(g.flat[i]))


def test_all_void_all_positive_all_negative():
    x, _ = _case(3)
    loss, g = V.void_loss(x, -np.ones_like(x))
    assert loss == 0.0 and np.all(g == 0)
    assert float(V.void_loss_torch(torch.from_numpy(x), -torch.ones(x.shape, dtype=torch.float64))) == 0.0
    # all positive: Nn = 0, so the positive term has weight 0 and the (empty) negative term weight 1
    loss, g = V.void_loss(x, np.ones_like(x))
    assert loss == 0.0 and np.all(g == 0)
    loss, g = V.void_loss(x, np.zeros_like(x))
    assert loss == 0.0 and np.all(g == 0)
    # positives and void only: the same
    y = np.where(np.arange(x.size).reshape(x.shape) % 2 == 0, 1.0, -1.0)
    loss, g = V.void_loss(x, y)
    assert loss == 0.0 and np.all(g == 0)


def test_labels_of_ids():
    ids = np.array([[0, 1, 2, 254, 255, 7]], np.uint8)
    assert V.labels_of_ids(ids).tolist() == [[0, 1, 1, 1, -1, 1]]
    assert V.labels_of_ids(ids, 2).tolist() == [[0, 0, 1, 0, -1, 0]]


@pytest.mark.parametrize("seed", range(6))
def test_id_warp_restatement_equals_cv2_nearest(seed):
    """The host id-mode warp (the oracle's nearest scale_n_rotate of the ids, then the id rule) equals cv2.warpAffine
    (INTER_NEAREST) of the flipped ids with the reference's matrix, then the id rule."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(seed)
    h, w = [(40, 56), (37, 61), (480, 854)][seed % 3]
    ids = rng.integers(0, 5, (h, w)).astype(np.uint8)
    ids[rng.random((h, w)) < 0.1] = 255
    rot, sc, flip = float(rng.uniform(-30, 30)), float(rng.uniform(0.75, 1.25)), bool(seed % 2)
    src = cv2.flip(ids, 1) if flip else ids
    m = cv2.getRotationMatrix2D((w / 2, h / 2), rot, sc)
    want_ids = cv2.warpAffine(src, m, (w, h), flags=cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    for obj in (None, 3):
        assert np.array_equal(V.warp_ids(ids, rot, sc, flip, obj), V.labels_of_ids(want_ids, obj))


def test_compiled_void_kernels():
    """The void forms are their own kernels: cbce_fwd_void_kernel<false|true>, cbce_bwd_void_kernel,
    tail_fwd_void_kernel<false|true>, tail_bwd2_void_kernel<false|true>, and the id ingest's two kernels."""
    import os
    import re
    from osvos_pytorch_b200 import build
    nvcc_dir = os.path.dirname(build._nvcc())
    cuobjdump, cufilt = os.path.join(nvcc_dir, "cuobjdump"), os.path.join(nvcc_dir, "cu++filt")
    if not (os.path.exists(cuobjdump) and os.path.exists(cufilt)):
        pytest.skip("cuobjdump / cu++filt not found next to nvcc")
    build.build()
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = subprocess.run([cufilt], input=syms, capture_output=True, text=True, check=True).stdout
    found = set()
    for line in names.splitlines():
        m = re.search(r"\b((?:cbce_fwd_void|cbce_bwd_void|tail_fwd_void|tail_bwd2_void|labels_from_ids)_kernel"
                      r"(?:<[^<>]*>)?)\(", line)
        if m:
            found.add(re.sub(r"\(bool\)1", "true", re.sub(r"\(bool\)0", "false", m.group(1))))
        if "affine_warp_kernel<osvos::WarpSrcIds8>" in line:
            found.add("affine_warp_kernel<WarpSrcIds8>")
    assert found == {"cbce_fwd_void_kernel<false>", "cbce_fwd_void_kernel<true>", "cbce_bwd_void_kernel",
                     "tail_fwd_void_kernel<false>", "tail_fwd_void_kernel<true>", "tail_bwd2_void_kernel<false>",
                     "tail_bwd2_void_kernel<true>", "labels_from_ids_kernel", "affine_warp_kernel<WarpSrcIds8>"}, found


def test_void_size_queries():
    from osvos_pytorch_b200 import _native as nat
    lib = nat.load()
    det, void = nat.FLAG_DETERMINISTIC, nat.FLAG_VOID_LABELS
    for n, h, w in [(1, 8, 8), (12, 480, 854)]:
        assert lib.osvos_tail_fwd_sums(n, h, w, 0) == lib.osvos_tail_fwd_sums(n, h, w, void) == nat.TAIL_SUMS
        assert lib.osvos_tail_fwd_sums(n, h, w, det) == lib.osvos_tail_fwd_deterministic_sums(n, h, w)
        rows = (lib.osvos_tail_fwd_sums(n, h, w, det) - nat.TAIL_SUMS) // 13
        assert lib.osvos_tail_fwd_sums(n, h, w, det | void) == nat.TAIL_SUMS + 14 * rows
    assert lib.osvos_tail_fwd_sums(1, 8, 8, 128) == 0 and lib.osvos_tail_fwd_sums(0, 8, 8, void) == 0
    for numel in (7, 1 << 22):
        rows = (lib.osvos_cbce_fwd_sums(numel, det) - 5) // 3
        assert lib.osvos_cbce_fwd_sums(numel, void) == 5
        assert lib.osvos_cbce_fwd_sums(numel, det | void) == 5 + 4 * rows
    assert lib.osvos_cbce_fwd_sums(7, 128) == 0
    # refusals before any CUDA call
    assert lib.osvos_labels_from_ids(None, None, 1, 8, 8, 0, None) == 1
    assert lib.osvos_labels_from_ids(1 << 20, 1 << 20, 1, 8, 8, 255, None) == 1
    assert lib.osvos_affine_warp_ids(1 << 20, 1 << 20, None, None, None, 1, 1, 8, 8, 0, None) == 1


def test_python_refusals():
    from osvos_pytorch_b200 import ops
    from osvos_pytorch_b200.layers.osvos_layers import class_balanced_cross_entropy_loss
    with pytest.raises(ValueError, match="size_average"):
        class_balanced_cross_entropy_loss(torch.zeros(1, 1, 4, 4), torch.zeros(1, 1, 4, 4), size_average=True, void=True)
    for bad in (0, 255, -1, True, "some"):
        with pytest.raises(ValueError, match="object"):
            ops._id_object(bad)
    assert ops._id_object(None) == ops._id_object("all") == 0 and ops._id_object(7) == 7


@pytest.mark.parametrize("argv,msg", [
    (["--davis", "2017", "--synthetic"], "--synthetic"),
    (["--davis", "2017"], "--loader reference"),
    (["--davis", "2017", "--loader", "native", "--upsampling-lr", "1e-3"], "--upsampling-lr"),
])
def test_train_parent_refuses(argv, msg, capsys):
    import train_parent
    with pytest.raises(SystemExit):
        train_parent.parse(argv)
    assert msg in capsys.readouterr().err


@pytest.mark.parametrize("argv,msg", [
    (["--ignore-void"], "--davis 2017"),
    (["--ignore-void", "--davis", "2017", "--loader", "native", "--upsampling-lr", "1e-3"], "--upsampling-lr"),
])
def test_train_online_refuses(argv, msg, capsys):
    import train_online
    with pytest.raises(SystemExit):
        train_online.parse(argv)
    assert msg in capsys.readouterr().err


def test_train_parent_accepts_2017_native():
    import train_parent
    a = train_parent.parse(["--davis", "2017", "--loader", "native", "--cache", "device", "--deterministic",
                            "--val-measures", "--input-res", "240", "427", "--output-res", "stored"])
    assert a.davis == "2017"
    assert train_parent.parse([]).davis == "2016"

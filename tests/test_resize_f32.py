"""CPU checks of the fp32 resize that brings fused logits back to the annotations' stored size (csrc/resize.cu
osvos_resize_f32, ops.resize_f32, DESIGN.md §18): the numpy restatement the GPU tests compare against
(tests/resize_f32_ref.py) is Pillow's BILINEAR resize of an 'F' image bit for bit, the entry points check their
arguments before any CUDA call, and both scripts take ``--output-res``."""
import numpy as np
import pytest

import resize_f32_ref

# (H, W) -> (H', W'): network resolutions back to DAVIS' 480x854, a downscale, small and large factors, one axis only,
# 1-pixel outputs, identity, and up in one axis with down in the other
SHAPES = [((240, 427), (480, 854)), ((120, 214), (480, 854)), ((360, 640), (480, 854)), ((480, 854), (240, 427)),
          ((7, 9), (30, 41)), ((30, 54), (1080, 1920)), ((240, 427), (480, 427)), ((240, 427), (240, 854)),
          ((33, 45), (1, 1)), ((33, 45), (1, 45)), ((33, 45), (33, 1)), ((1, 1), (5, 7)), ((31, 29), (31, 29)),
          ((5, 70), (64, 3)), ((97, 131), (40, 300))]


def _pil_resize(arr, size):
    Image = pytest.importorskip("PIL.Image")
    im = Image.fromarray(np.ascontiguousarray(arr, dtype=np.float32))
    assert im.mode == "F"
    return np.asarray(im.resize((size[1], size[0]), Image.Resampling.BILINEAR))


def _logits(rng, shape, span=30.0):
    """Logit-like maps: smooth structure of both signs plus noise."""
    h, w = shape
    yy, xx = np.meshgrid(np.linspace(-1, 1, h), np.linspace(-1, 1, w), indexing="ij")
    smooth = span * np.sin(3 * xx + rng.uniform(0, 6)) * np.cos(2 * yy + rng.uniform(0, 6))
    return (smooth + rng.normal(0, span / 10, shape)).astype(np.float32)


@pytest.mark.parametrize("src,dst", SHAPES)
def test_restatement_is_pillow(src, dst):
    rng = np.random.default_rng(list(src + dst))
    arr = _logits(rng, src)
    got = resize_f32_ref.resize(arr, dst)
    assert got.dtype == np.float32 and got.shape == dst
    assert np.array_equal(got.view(np.uint32), _pil_resize(arr, dst).view(np.uint32))


def test_restatement_is_pillow_on_random_shapes():
    rng = np.random.default_rng(17)
    for _ in range(40):
        src = tuple(int(v) for v in rng.integers(1, 200, 2))
        dst = tuple(int(v) for v in rng.integers(1, 200, 2))
        arr = _logits(rng, src)
        got = resize_f32_ref.resize(arr, dst)
        assert np.array_equal(got.view(np.uint32), _pil_resize(arr, dst).view(np.uint32)), (src, dst)


@pytest.mark.parametrize("src,dst", [((240, 427), (480, 854)), ((50, 30), (17, 77))])
def test_restatement_is_pillow_on_large_values_of_both_signs(src, dst):
    rng = np.random.default_rng(3)
    arr = (rng.uniform(-1e4, 1e4, src) * 10.0 ** rng.integers(-6, 1, src)).astype(np.float32)
    arr[::7] *= -1
    got = resize_f32_ref.resize(arr, dst)
    assert (got < 0).any() and (got > 0).any()
    assert np.array_equal(got.view(np.uint32), _pil_resize(arr, dst).view(np.uint32))


def test_restatement_takes_batches():
    rng = np.random.default_rng(4)
    maps = np.stack([_logits(rng, (24, 40)) for _ in range(3)])[:, None]
    got = resize_f32_ref.resize(maps, (50, 33))
    assert got.shape == (3, 1, 50, 33)
    for i in range(3):
        assert np.array_equal(got[i, 0], resize_f32_ref.resize(maps[i, 0], (50, 33)))


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


ADDR = 1 << 20                                           # placeholder device address, never dereferenced


@pytest.mark.parametrize("args,rejected_by", [
    ((None, ADDR, ADDR, 1, 8, 8, 4, 4), "src != nullptr"),
    ((ADDR, None, ADDR, 1, 8, 8, 4, 4), "dst != nullptr"),
    ((ADDR, ADDR, ADDR, 0, 8, 8, 4, 4), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 65536, 8, 8, 4, 4), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 32768, 4, 4), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 8, 0, 4), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 8, 4, 32768), "resize_dims_ok"),
    ((ADDR, ADDR, None, 1, 8, 8, 4, 4), "workspace != nullptr"),
    ((ADDR, ADDR, ADDR + 4, 1, 8, 8, 4, 4), "workspace != nullptr"),
])
def test_resize_f32_checks_arguments_first(lib, args, rejected_by):
    assert lib.osvos_resize_f32(*args, None) == 1
    msg = lib.osvos_last_error()
    assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


def test_resize_f32_workspace_bytes(lib):
    q = lib.osvos_resize_f32_workspace_bytes
    assert q(1, 8, 8, 8, 8) == 0                                                # identity: a copy
    for bad in ((0, 8, 8, 4, 4), (65536, 8, 8, 4, 4), (1, 0, 8, 4, 4), (1, 8, 32768, 4, 4), (1, 8, 8, -1, 4),
                (1, 8, 8, 4, 32768)):
        assert q(*bad) == 0, bad
    a16 = lambda v: (v + 15) // 16 * 16
    bounds = lambda out: a16(8 * out)                                           # {xmin, count} per output
    weights = lambda out, k: a16(8 * out * k)                                   # ksize doubles per output
    # 2x upscale in both axes (ksize 3): both tables, then the horizontal pass's fp32 intermediate
    assert q(12, 240, 427, 480, 854) == (bounds(854) + bounds(480) + weights(854, 3) + weights(480, 3)
                                         + 4 * 12 * 240 * 854)
    assert q(2, 240, 427, 480, 427) == bounds(480) + weights(480, 3)           # vertical only: no intermediate
    assert q(2, 480, 854, 480, 427) == bounds(427) + weights(427, 5)           # horizontal 2x downscale: ksize 5


def test_resize_f32_refuses_cpu_tensors():
    import torch
    from osvos_pytorch_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.resize_f32(torch.zeros(1, 1, 8, 8), (16, 16))


@pytest.mark.parametrize("script", ["train_online", "train_parent"])
def test_output_res_option(script):
    import importlib
    mod = importlib.import_module(script)
    assert mod.parse(["--loader", "native", "--input-res", "240", "427"]).output_res == "network"
    assert mod.parse(["--loader", "native", "--input-res", "240", "427", "--output-res", "stored"]).output_res == "stored"
    assert mod.parse(["--loader", "native", "--output-res", "network"]).output_res == "network"
    for bad in ("native", "full", "480"):
        with pytest.raises(SystemExit):
            mod.parse(["--loader", "native", "--input-res", "240", "427", "--output-res", bad])

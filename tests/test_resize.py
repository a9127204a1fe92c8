"""CPU checks of the frame resize (csrc/resize.cu, ops.resize_u8, davis.imresize_size): the numpy restatement the GPU
tests compare against (tests/resize_ref.py) is Pillow's Image.resize, the size argument follows scipy 1.0's imresize,
and the entry points check their arguments before any CUDA call."""
import numpy as np
import pytest

import resize_ref

# (H, W) -> (H', W'): down, up, one axis only, up in one axis and down in the other, 1-pixel outputs, identity
SHAPES = [((480, 854), (240, 427)), ((480, 854), (360, 640)), ((480, 854), (720, 1280)), ((480, 854), (480, 427)),
          ((1080, 1920), (480, 854)), ((48, 70), (33, 45)), ((37, 53), (100, 21)), ((31, 29), (31, 29)),
          ((33, 45), (1, 1)), ((33, 45), (1, 45)), ((33, 45), (33, 1)), ((5, 7), (64, 3)), ((97, 131), (48, 131)),
          ((2, 3), (3, 2))]


def _pil_resize(arr, size, mode):
    Image = pytest.importorskip("PIL.Image")
    resample = Image.Resampling.BILINEAR if mode == "bilinear" else Image.Resampling.NEAREST
    return np.asarray(Image.fromarray(arr).resize((size[1], size[0]), resample))


@pytest.mark.parametrize("src,dst", SHAPES)
@pytest.mark.parametrize("mode,c", [("bilinear", 3), ("bilinear", 1), ("nearest", 1), ("nearest", 3)])
def test_restatement_is_pillow(src, dst, mode, c):
    rng = np.random.default_rng(list(src + dst) + [c, len(mode)])
    arr = rng.integers(0, 256, src + ((c,) if c == 3 else ()), dtype=np.uint8)
    if mode == "nearest" and c == 1:
        arr = np.where(arr > 128, 255, 0).astype(np.uint8)          # a mask
    assert np.array_equal(resize_ref.resize(arr, dst, mode), _pil_resize(arr, dst, mode))


def test_restatement_is_pillow_on_random_shapes():
    rng = np.random.default_rng(5)
    for _ in range(40):
        src = tuple(int(v) for v in rng.integers(1, 160, 2))
        dst = tuple(int(v) for v in rng.integers(1, 160, 2))
        arr = rng.integers(0, 256, src + (3,), dtype=np.uint8)
        for mode in ("bilinear", "nearest"):
            assert np.array_equal(resize_ref.resize(arr, dst, mode), _pil_resize(arr, dst, mode)), (src, dst, mode)


def test_imresize_size_follows_scipy():
    from osvos_pytorch_b200.davis import imresize_size
    assert imresize_size((240, 427), 480, 854) == (240, 427)
    assert imresize_size([100, 21], 37, 53) == (100, 21)
    assert imresize_size(50, 480, 854) == (240, 427)                 # int: a percentage
    assert imresize_size(np.int64(33), 480, 854) == (158, 281)       # int(480 * 0.33), int(854 * 0.33)
    assert imresize_size(0.5, 480, 854) == (240, 427)                # float: a fraction
    assert imresize_size(0.3, 97, 131) == (29, 39)
    assert imresize_size(np.float32(1.5), 33, 45) == (49, 67)
    assert imresize_size(150, 33, 45) == (49, 67)
    for bad, exc in [((1,), ValueError), (0, ValueError), (0.001, ValueError), (True, TypeError)]:
        with pytest.raises(exc):
            imresize_size(bad, 480, 854)


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


ADDR = 1 << 20                                           # placeholder device address, never dereferenced


@pytest.mark.parametrize("args,rejected_by", [
    ((None, ADDR, ADDR, 1, 8, 8, 3, 4, 4, 0), "src != nullptr"),
    ((ADDR, None, ADDR, 1, 8, 8, 3, 4, 4, 0), "dst != nullptr"),
    ((ADDR, ADDR, ADDR, 0, 8, 8, 3, 4, 4, 0), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 70000, 8, 8, 3, 4, 4, 0), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 40000, 3, 4, 4, 0), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 8, 3, 0, 4, 0), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 8, 3, 4, 32768, 0), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 8, 2, 4, 4, 0), "resize_dims_ok"),
    ((ADDR, ADDR, ADDR, 1, 8, 8, 3, 4, 4, 2), "resize_dims_ok"),
    ((ADDR, ADDR, None, 1, 8, 8, 3, 4, 4, 0), "workspace != nullptr"),
    ((ADDR, ADDR, ADDR + 2, 1, 8, 8, 1, 4, 4, 1), "workspace != nullptr"),
])
def test_resize_u8_checks_arguments_first(lib, args, rejected_by):
    assert lib.osvos_resize_u8(*args, None) == 1
    msg = lib.osvos_last_error()
    assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


def test_resize_u8_workspace_bytes(lib):
    q = lib.osvos_resize_u8_workspace_bytes
    assert q(1, 8, 8, 3, 8, 8, 0) == 0 and q(1, 8, 8, 1, 8, 8, 1) == 0         # identity: a copy
    assert q(0, 8, 8, 3, 4, 4, 0) == 0 and q(1, 8, 8, 2, 4, 4, 0) == 0         # invalid arguments
    a16 = lambda v: (v + 15) // 16 * 16
    # nearest: the two index tables, 16-byte aligned
    assert q(12, 480, 854, 1, 240, 427, 1) == a16(427 * 4) + a16(240 * 4)
    # bilinear, both axes: {xmin, count, ksize weights} per output and axis (ksize 5 for a 2x downscale), then the
    # horizontal pass's intermediate at the full source height
    tab = lambda out, k: a16(4 * out * (k + 2))
    assert q(12, 480, 854, 3, 240, 427, 0) == tab(427, 5) + tab(240, 5) + 12 * 480 * 427 * 3
    assert q(2, 480, 854, 3, 480, 427, 0) == tab(427, 5)                        # horizontal only: no intermediate
    assert q(2, 37, 53, 1, 100, 53, 0) == tab(100, 3)                           # vertical only, upscale: ksize 3


def test_resize_u8_refuses_cpu_tensors():
    import torch
    from osvos_pytorch_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.resize_u8(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), (4, 4))


@pytest.mark.parametrize("script", ["train_online", "train_parent"])
def test_input_res_option_needs_the_native_loader(script):
    import importlib
    mod = importlib.import_module(script)
    assert mod.parse(["--loader", "native", "--input-res", "240", "427"]).input_res == [240, 427]
    assert mod.parse(["--loader", "native"]).input_res is None
    for argv in (["--input-res", "240", "427"], ["--synthetic", "--input-res", "240", "427"]):
        with pytest.raises(SystemExit):
            mod.parse(argv)

"""CPU checks of the per-object upsample fused with the merge (csrc/resize.cu osvos_upsample_merge_objects,
ops.upsample_merge_objects, DESIGN.md §27): the numpy restatement the GPU tests compare against
(tests/upsample_merge_ref.py) is Pillow's 'F' resize of each map followed by an argmax with a background plane, the
entry points check their arguments before any CUDA call, and train_online.py takes --davis 2017 --input-res only with
--output-res stored."""
import ctypes

import numpy as np
import pytest

import upsample_merge_ref

SHAPES = [((24, 40), (48, 80)), ((7, 9), (30, 41)), ((30, 54), (60, 108)), ((48, 80), (24, 40)), ((24, 40), (48, 40)),
          ((24, 40), (24, 80)), ((13, 17), (13, 17)), ((13, 17), (1, 1)), ((5, 70), (64, 3))]


def _pillow_argmax(maps, size):
    """Each map through Pillow's 'F' BILINEAR resize, then the label rule as an argmax over a background plane of +0
    in front of the objects (the first maximum wins, so ties go to the background or the lowest object; NaN is -inf)."""
    Image = pytest.importorskip("PIL.Image")
    up = [np.asarray(Image.fromarray(np.ascontiguousarray(m, np.float32)).resize((size[1], size[0]),
                                                                                 Image.Resampling.BILINEAR))
          for m in maps]
    vals = np.stack([np.zeros_like(up[0])] + up)
    vals = np.where(np.isnan(vals), -np.inf, vals)
    return np.argmax(vals, axis=0).astype(np.uint8)


def _maps(rng, k, shape):
    """K logit-like maps with exact ties across objects, ±0, NaN and all-negative maps."""
    m = np.round(rng.normal(0, 2, (k,) + shape) * 2) / 2
    sel = rng.random(shape)
    m[:, sel < 0.05] = np.nan
    m[:, (sel >= 0.05) & (sel < 0.1)] = 0.0
    m[:, (sel >= 0.1) & (sel < 0.15)] = -0.0
    if k > 1:
        m[1] = -np.abs(m[1]) - 1.0                               # one map negative everywhere
        m[k - 1, sel > 0.9] = m[0, sel > 0.9]                    # ties between the first and the last object
    return m.astype(np.float32)


@pytest.mark.parametrize("src,dst", SHAPES)
@pytest.mark.parametrize("k", [1, 2, 4])
def test_restatement_is_pillow_and_argmax(src, dst, k):
    rng = np.random.default_rng(list(src + dst) + [k])
    maps = _maps(rng, k, src)
    assert np.array_equal(upsample_merge_ref.upsample_merge(maps, dst), _pillow_argmax(maps, dst))


def test_restatement_on_random_shapes():
    rng = np.random.default_rng(27)
    for _ in range(20):
        src = tuple(int(v) for v in rng.integers(1, 60, 2))
        dst = tuple(int(v) for v in rng.integers(1, 120, 2))
        k = int(rng.integers(1, 6))
        maps = _maps(rng, k, src) * np.float32(10.0) ** rng.integers(-6, 5)
        assert np.array_equal(upsample_merge_ref.upsample_merge(maps, dst), _pillow_argmax(maps, dst)), (src, dst, k)


def test_restatement_takes_batches():
    rng = np.random.default_rng(5)
    maps = _maps(rng, 3, (2, 1, 12, 20))
    got = upsample_merge_ref.upsample_merge(maps, (25, 41))
    assert got.shape == (2, 1, 25, 41)
    for i in range(2):
        assert np.array_equal(got[i, 0], upsample_merge_ref.upsample_merge(maps[:, i, 0], (25, 41)))


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


ADDR = 1 << 20                                           # placeholder device address, never dereferenced


def _ptrs(k, bad=None):
    """A host array of max(k, 1) map pointers; ``bad`` = (index, value) replaces one."""
    vals = [ADDR] * max(k, 1)
    if bad is not None:
        vals[bad[0]] = bad[1]
    return (ctypes.c_void_p * len(vals))(*vals)


@pytest.mark.parametrize("maps,k,out,dims,rejected_by", [
    (None, 2, ADDR, (1, 8, 8, 16, 16), "maps != nullptr"),
    ("ok", 2, None, (1, 8, 8, 16, 16), "out != nullptr"),
    ("ok", 0, ADDR, (1, 8, 8, 16, 16), "k >= 1"),
    ("ok", 255, ADDR, (1, 8, 8, 16, 16), "k >= 1"),
    ("ok", 2, ADDR, (0, 8, 8, 16, 16), "resize_dims_ok"),
    ("ok", 2, ADDR, (65536, 8, 8, 16, 16), "resize_dims_ok"),
    ("ok", 2, ADDR, (1, 32768, 8, 16, 16), "resize_dims_ok"),
    ("ok", 2, ADDR, (1, 8, 32768, 16, 16), "resize_dims_ok"),
    ("ok", 2, ADDR, (1, 8, 8, 32768, 16), "resize_dims_ok"),
    ("ok", 2, ADDR, (1, 8, 8, 16, 32768), "resize_dims_ok"),
    ("ok", 2, ADDR, (1, 8, 8, 0, 16), "resize_dims_ok"),
    ((1, None), 2, ADDR, (1, 8, 8, 16, 16), "maps[i] != nullptr"),
    ((0, ADDR + 2), 2, ADDR, (1, 8, 8, 16, 16), "maps[i] != nullptr"),
    ("ok", 2, ADDR, (1, 30000, 8, 1, 8), "p.tile_h > 0"),       # a 30000 -> 1 downscale: one row cannot be staged
    ("ok", 2, ADDR, (1, 1200, 8, 50, 8), "p.tile_h > 0"),       # factor 24
])
def test_entry_point_checks_arguments_first(lib, maps, k, out, dims, rejected_by):
    arr = None if maps is None else _ptrs(k, None if maps == "ok" else maps)
    assert lib.osvos_upsample_merge_objects(arr, k, out, ADDR, *dims, None) == 1
    msg = lib.osvos_last_error()
    assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


@pytest.mark.parametrize("ws", [None, ADDR + 4])
def test_entry_point_checks_the_workspace(lib, ws):
    assert lib.osvos_upsample_merge_objects(_ptrs(2), 2, ADDR, ws, 1, 8, 8, 16, 16, None) == 1
    assert b"workspace != nullptr" in lib.osvos_last_error()


def test_workspace_bytes(lib):
    q = lib.osvos_upsample_merge_objects_workspace_bytes
    assert q(1, 2, 8, 8, 8, 8) == 0                                             # identity: a plain merge
    for bad in ((0, 1, 8, 8, 4, 4), (65536, 1, 8, 8, 4, 4), (1, 0, 8, 8, 4, 4), (1, 255, 8, 8, 4, 4),
                (1, 1, 0, 8, 4, 4), (1, 1, 8, 32768, 4, 4), (1, 1, 8, 8, -1, 4), (1, 1, 8, 8, 4, 32768),
                (1, 1, 30000, 8, 1, 8), (1, 1, 1200, 8, 50, 8)):
        assert q(*bad) == 0, bad
    a16 = lambda v: (v + 15) // 16 * 16
    bounds = lambda out: a16(8 * out)                                           # {xmin, count} per output
    weights = lambda out, k: a16(8 * out * k)                                   # double weights, ksize per output
    # the fp32 resize's tables only, never its intermediate: the same for every n and k
    both = bounds(854) + bounds(480) + weights(854, 3) + weights(480, 3)
    assert q(1, 1, 240, 427, 480, 854) == q(12, 254, 240, 427, 480, 854) == both
    assert q(2, 3, 240, 427, 480, 427) == bounds(480) + weights(480, 3)        # vertical only
    assert q(2, 3, 480, 854, 480, 427) == bounds(427) + weights(427, 5)        # horizontal 2x downscale: ksize 5
    assert q(1, 1, 1100, 8, 50, 8) > 0                                          # factor 22 is still staged


def test_refuses_cpu_tensors():
    import torch
    from osvos_pytorch_b200 import ops
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.upsample_merge_objects([torch.zeros(1, 1, 8, 8)], (16, 16))


def test_train_online_davis_2017_input_res_rules():
    import train_online
    base = ["--loader", "native", "--davis", "2017"]
    a = train_online.parse(base + ["--input-res", "240", "427", "--output-res", "stored"])
    assert a.input_res == [240, 427] and a.output_res == "stored"
    a = train_online.parse(base + ["--input-res", "240", "427", "--output-res", "stored", "--ignore-void"])
    assert a.ignore_void
    assert train_online.parse(base + ["--output-res", "stored"]).input_res is None     # a no-op, as for 2016
    for extra in (["--input-res", "240", "427"], ["--input-res", "240", "427", "--output-res", "network"]):
        with pytest.raises(SystemExit):
            train_online.parse(base + extra)
    with pytest.raises(SystemExit):
        train_online.parse(["--davis", "2017", "--input-res", "240", "427", "--output-res", "stored"])   # reference


def test_train_online_refusal_names_output_res_stored(capsys):
    import train_online
    with pytest.raises(SystemExit):
        train_online.parse(["--loader", "native", "--davis", "2017", "--input-res", "240", "427"])
    assert "--output-res stored" in capsys.readouterr().err

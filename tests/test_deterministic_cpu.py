"""CPU-side checks of the deterministic forms: argument validation before any CUDA call, shape queries, and the
--deterministic switch of the two training scripts."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


def test_flag_value_matches_header():
    import os
    import re
    from osvos_pytorch_b200 import _native as nat
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "osvos_b200.h")).read()
    assert int(re.search(r"OSVOS_FLAG_DETERMINISTIC\s*=\s*(\d+)", hdr).group(1)) == nat.FLAG_DETERMINISTIC


def test_flagged_entry_points_refuse_bad_arguments(lib):
    from osvos_pytorch_b200 import _native as nat
    det = nat.FLAG_DETERMINISTIC
    addr = 1 << 20                                  # placeholder device address, never dereferenced
    assert lib.osvos_reduce_rows(None, 4, 4, addr, addr, 0, None) == 1
    assert lib.osvos_reduce_rows(addr, 0, 4, addr, addr, 0, None) == 1
    assert lib.osvos_wgrad_finish(None, None, 1, det, None) == 1

    def unpool(dpool, dside, dpq, wfold, x=addr, flags=det, c=64):
        return lib.osvos_unpool_mask(dpool, None, x, None, dside, dpq, wfold, addr, None, None, 1, 8, 8, c, flags, None)
    assert unpool(None, None, None, None, x=None) == 1
    # dpq without wfold or the reverse, the add form without dpool (no consumer), dside with dpq, unknown flag bits
    assert unpool(None, None, addr, None) == 1
    assert unpool(None, None, None, addr) == 1
    assert unpool(None, None, None, None) == 1
    assert unpool(None, None, None, None, flags=0) == 1
    assert unpool(addr, addr, addr, addr) == 1
    assert unpool(addr, None, None, None, flags=det | nat.FLAG_FAST) == 1
    # misaligned dside / wfold, and channel counts the block layout cannot take
    assert unpool(None, addr + 4, None, None) == 1
    assert unpool(None, None, addr, addr + 4) == 1
    assert unpool(addr, None, None, None, c=60) == 1
    assert unpool(addr, None, None, None, c=0) == 1
    assert lib.osvos_side_folded_wgrad_multi(None, 1, addr, det, None) == 1
    assert lib.osvos_side_folded_wgrad_multi(None, 1, None, 0, None) == 1
    assert lib.osvos_conv_first_bwd(None, addr, None, None, addr, None, addr, 1, 8, 8, det, None) == 1
    assert lib.osvos_conv_first_bwd(None, addr, None, None, addr, None, addr, 1, 8, 8, 0, None) == 1
    assert lib.osvos_sum_f32(addr, 16, None, addr, det, None) == 1
    assert lib.osvos_sum_f32(addr, 16, addr, addr, nat.FLAG_RELU, None) == 1
    assert lib.osvos_cbce_fwd(addr, addr, 16, 1.0, addr, addr, nat.FLAG_RELU, None) == 1
    assert b"invalid argument" in lib.osvos_last_error()


def test_wgrad_finish_takes_splits_with_the_flag_only(lib):
    from osvos_pytorch_b200 import _native as nat
    addr = 1 << 20
    item = nat.WgradFinishItem(addr, addr, 64, 64, 64, 0, 1.0)
    splits = (ctypes.c_int * 1)(2)
    assert lib.osvos_wgrad_finish(ctypes.byref(item), None, 1, nat.FLAG_DETERMINISTIC, None) == 1
    assert lib.osvos_wgrad_finish(ctypes.byref(item), splits, 1, 0, None) == 1
    assert lib.osvos_wgrad_finish(ctypes.byref(item), None, 1, nat.FLAG_FAST, None) == 1
    assert b"invalid argument" in lib.osvos_last_error()


def test_flagged_shape_queries(lib):
    from osvos_pytorch_b200 import _native as nat
    det = nat.FLAG_DETERMINISTIC
    assert lib.osvos_reduce_rows_scratch_floats(10, 3) == 30
    assert lib.osvos_reduce_rows_scratch_floats(1000, 3) == 64 * 3
    assert lib.osvos_reduce_rows_scratch_floats(0, 3) == 0
    assert lib.osvos_conv3x3_colsum_rows(1, 16, 8) == 8
    assert lib.osvos_conv3x3_colsum_rows(2, 17, 9) == 2 * 2 * 2 * 8
    assert lib.osvos_conv3x3_colsum_rows(0, 16, 8) == 0
    # the split count comes from a nominal device: a pure function of the shape
    s = lib.osvos_wgrad_deterministic_splits(1, 480, 854, 64, 64)
    assert s > 1
    assert lib.osvos_wgrad_workspace_bytes(1, 480, 854, 64, 64, det) == \
        s * lib.osvos_wgrad_workspace_bytes(1, 480, 854, 64, 64, 0)
    assert lib.osvos_wgrad_deterministic_splits(1, 8, 8, 96, 64) == 0        # cin neither 64 nor a multiple of 128
    assert lib.osvos_wgrad_workspace_bytes(0, 8, 8, 64, 64, det) == 0
    assert lib.osvos_unpool_colsum_rows(1, 8, 8, 60, 1, 0) == 0               # 256 % (c / 8) != 0
    assert lib.osvos_conv_first_bwd_workspace_bytes(0, 8, 8, det) == 0
    assert lib.osvos_tail_fwd_deterministic_sums(0, 8, 8) == 0
    assert lib.osvos_sum_f32_scratch_bytes(det) == (256 + 1) * 4
    assert lib.osvos_sum_f32_scratch_bytes(0) == 2 * 8
    assert lib.osvos_cbce_fwd_sums(0, det) == 0
    assert lib.osvos_side_folded_wgrad_workspace_bytes(None, 1, det) == 0
    # unknown flag bits: no size
    for bad in (nat.FLAG_FAST, det | nat.FLAG_RELU):
        assert lib.osvos_wgrad_workspace_bytes(1, 8, 8, 64, 64, bad) == 0
        assert lib.osvos_conv_first_bwd_workspace_bytes(1, 8, 8, bad) == 0
        assert lib.osvos_sum_f32_scratch_bytes(bad) == 0
        assert lib.osvos_cbce_fwd_sums(16, bad) == 0


def test_default_workspace_queries_are_unchanged(lib):
    assert lib.osvos_wgrad_workspace_bytes(1, 8, 8, 64, 128, 0) == 9 * 128 * 64 * 4
    assert lib.osvos_conv_first_bwd_workspace_bytes(1, 8, 8, 0) == (16 * 64 * 27 + 4) * 4
    assert lib.osvos_cbce_fwd_sums(1, 0) == lib.osvos_cbce_fwd_sums(1 << 24, 0) == 5


@pytest.mark.parametrize("script", ["train_online", "train_parent"])
def test_scripts_parse_deterministic(script):
    mod = __import__(script)
    assert mod.parse([]).deterministic is False
    assert mod.parse(["--deterministic"]).deterministic is True

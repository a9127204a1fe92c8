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


def test_entry_points_refuse_null_arguments(lib):
    addr = 1 << 20                                  # placeholder device address, never dereferenced
    assert lib.osvos_reduce_rows(None, 4, 4, addr, addr, 0, None) == 1
    assert lib.osvos_reduce_rows(addr, 0, 4, addr, addr, 0, None) == 1
    assert lib.osvos_wgrad_finish_deterministic(None, None, 1, None) == 1
    assert lib.osvos_unpool_mask_deterministic(None, None, None, None, None, None, None, None, None, 1, 8, 8, 64,
                                               None) == 1
    # dpq without wfold, and the add form without dpool, are refused
    assert lib.osvos_unpool_mask_deterministic(None, None, addr, None, addr, None, addr, None, None, 1, 8, 8, 64,
                                               None) == 1
    assert lib.osvos_unpool_mask_deterministic(None, None, addr, None, None, None, addr, None, None, 1, 8, 8, 64,
                                               None) == 1
    assert lib.osvos_side_folded_wgrad_multi_deterministic(None, 1, addr, None) == 1
    assert lib.osvos_conv_first_bwd_deterministic(None, addr, None, None, addr, None, addr, 1, 8, 8, None) == 1
    assert b"invalid argument" in lib.osvos_last_error()


def test_shape_queries(lib):
    assert lib.osvos_reduce_rows_scratch_floats(10, 3) == 30
    assert lib.osvos_reduce_rows_scratch_floats(1000, 3) == 64 * 3
    assert lib.osvos_reduce_rows_scratch_floats(0, 3) == 0
    assert lib.osvos_conv3x3_colsum_rows(1, 16, 8) == 8
    assert lib.osvos_conv3x3_colsum_rows(2, 17, 9) == 2 * 2 * 2 * 8
    assert lib.osvos_conv3x3_colsum_rows(0, 16, 8) == 0
    # the split count comes from a nominal device: a pure function of the shape
    s = lib.osvos_wgrad_deterministic_splits(1, 480, 854, 64, 64)
    assert s > 1
    assert lib.osvos_wgrad_deterministic_workspace_bytes(1, 480, 854, 64, 64) == s * lib.osvos_wgrad_workspace_bytes(64, 64)
    assert lib.osvos_wgrad_deterministic_splits(1, 8, 8, 96, 64) == 0        # cin neither 64 nor a multiple of 128
    assert lib.osvos_wgrad_deterministic_workspace_bytes(0, 8, 8, 64, 64) == 0
    assert lib.osvos_unpool_colsum_rows(1, 8, 8, 60, 1, 0) == 0               # 256 % (c / 8) != 0
    assert lib.osvos_conv_first_bwd_deterministic_workspace_bytes(0, 8, 8) == 0
    assert lib.osvos_tail_fwd_deterministic_sums(0, 8, 8) == 0


def test_default_workspace_query_is_unchanged(lib):
    assert lib.osvos_wgrad_workspace_bytes(128, 64) == 9 * 128 * 64 * 4


@pytest.mark.parametrize("script", ["train_online", "train_parent"])
def test_scripts_parse_deterministic(script):
    mod = __import__(script)
    assert mod.parse([]).deterministic is False
    assert mod.parse(["--deterministic"]).deterministic is True

"""CPU checks of the host restatement of the conv1_1, tail-backward, general-tail and loss launch plans
(tests/train_dispatch_ref.py): it agrees with the library's own planning queries, it reaches every regime at any
plausible SM count, and the kernels compiled into the library are exactly the instantiations planned there.  No GPU
needed: the library loads on a CPU box, where its SM count is the H100's 132."""
import itertools
import subprocess

import pytest

import train_dispatch_ref as ref
from conv_dispatch_ref import parse_kernel_name
from test_conv_dispatch import _cuda_tool

HOST_SMS = 132      # device_sm_count() without a device


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat, build
    build.build()
    return nat.load()


SIZES = [(1, 1), (3, 5), (8, 8), (9, 17), (16, 24), (31, 45), (60, 107), (97, 131), (120, 214), (240, 427), (480, 854),
         (7, 64), (5, 65), (3, 129), (2, 1000)]


def test_first_bwd_workspace_query_matches(lib):
    from osvos_pytorch_b200._native import FLAG_DETERMINISTIC as DET
    assert lib.osvos_conv_first_bwd_workspace_bytes(1, 8, 8, 0) == ref.first_bwd_workspace_bytes() == (16 * 1728 + 4) * 4
    for n, (h, w) in itertools.product((1, 2, 3, 12), SIZES):
        p = ref.first_wgrad_plan(n, h, w, HOST_SMS)
        assert lib.osvos_conv_first_bwd_workspace_bytes(n, h, w, 0) == ref.first_bwd_workspace_bytes(), (n, h, w)
        assert lib.osvos_conv_first_bwd_workspace_bytes(n, h, w, DET) == 4 * p.det_workspace_floats, (n, h, w)
        assert sum(len(t) for t in p.block_tiles) == p.tiles and 1 <= p.last_valid <= ref.FW_PIX
    assert lib.osvos_conv_first_bwd_workspace_bytes(0, 8, 8, DET) == 0


def test_reduce_rows_scratch_matches(lib):
    for nrows, ncols in itertools.product((1, 2, 63, 64, 65, 127, 4100), (1, 31, 1728, 5000)):
        assert lib.osvos_reduce_rows_scratch_floats(nrows, ncols) == ref.reduce_rows_scratch_floats(nrows, ncols)
    assert lib.osvos_reduce_rows_scratch_floats(0, 5) == 0 and lib.osvos_reduce_rows_scratch_floats(5, 0) == 0


def test_general_tail_plans_match(lib):
    for n, (h, w) in itertools.product((1, 2, 3, 12), SIZES):
        assert lib.osvos_tail_general_fwd_sums(n, h, w) == ref.gen_fwd_sums(n, h, HOST_SMS), (n, h, w)
        p = ref.gen_bwd_plan(n, h, w)
        assert lib.osvos_tail_general_bwd_workspace_bytes(n, h, w) == 4 * p.workspace_floats, (n, h, w)
        assert p.row_len == tuple(17 * 4 * s * s + 33 for s in (2, 4, 8, 16))
    assert lib.osvos_tail_general_fwd_sums(1, 0, 4) == 0 and lib.osvos_tail_general_bwd_workspace_bytes(1, 4, 0) == 0


def test_cbce_sums_query_matches(lib):
    from osvos_pytorch_b200._native import FLAG_DETERMINISTIC as DET
    for numel in (1, 2, 3, 4, 5, 1023, 1024, 1025, 4096, 4097, 270336, 1081344, 1081345, 5 * 10 ** 6, 854 * 480 * 12):
        assert lib.osvos_cbce_fwd_sums(numel, DET) == ref.cbce_det_sums(numel, HOST_SMS), numel
        assert lib.osvos_cbce_fwd_sums(numel, 0) == 5, numel
    assert lib.osvos_cbce_fwd_sums(0, DET) == 0


def test_tail_bwd_items_cover_the_plan():
    """The per-row items of tail_bwd_row_items are the plan's segments: n hk segs items per scale, in scale order."""
    for n, (h, w) in itertools.product((1, 3), SIZES):
        scales, total = ref.tail_bwd_scales(n, h, w)
        row = ref.tail_bwd_row_items(w)
        assert total == sum(n * sc.hk * sum(1 for it in row if it.scale == k) for k, sc in enumerate(scales))
        for it in row:
            sc = scales[it.scale]
            assert it.width <= 512 + 32 and (it.rgroups == 1 or it.width <= it.wpad)
            assert sum(i.nout for i in row if i.scale == it.scale) == sc.wk
    assert ref.tail_bwd_reachable() == {(0, 1), (0, 2), (0, 4), (0, 8), (1, 1), (1, 2), (1, 4), (1, 8),
                                        (2, 2), (2, 4), (2, 8), (3, 2), (3, 4), (3, 8)}


@pytest.mark.parametrize("sms", range(60, 145))
def test_every_regime_is_found_at_sms(sms):
    """The searches the GPU file runs reach every regime at any SM count from 60 to 144, with the promised shapes."""
    for regime in ref.FIRST_REGIMES:
        n, h, w = ref.find_first_shape(regime, sms)
        assert h % ref.FIRST_TILE_H != 0 and w % ref.FIRST_TILE_W != 0
        p = ref.conv_first_plan(n, h, w, False, True, sms)
        counts = {len(t) for t in p.cta_tiles}
        if regime == "one_wave":
            assert p.tiles <= sms and counts == {1}
        else:
            assert n >= 2 and p.tiles > 3 * sms and p.tiles % sms != 0 and p.tiles_per_image < p.grid
            assert counts == {p.tiles // sms, p.tiles // sms + 1} and min(counts) >= ref.FIRST_STAGES
    for regime, width in ref.fw_cases():
        n, h, w = ref.find_fw_shape(regime, width, sms)
        p = ref.first_wgrad_plan(n, h, w, sms)
        assert w == ref.FW_WIDTHS[width] and n >= 2
        assert p.last_valid == {"narrow": 37, "64k": 64, "64k+1": 1}[width]
        counts = {len(t) for t in p.block_tiles}
        if regime == "few":
            assert p.tiles < ref.FW_COPIES and p.grid < ref.RED_SEGS and counts == {1}
        elif regime == "one_wave":
            assert ref.RED_SEGS < p.grid == p.tiles <= 4 * sms and counts == {1}
        else:
            assert p.grid == 4 * sms > ref.RED_SEGS and min(counts) >= 2 and len(counts) == 2
    for regime in ref.GEN_FWD_REGIMES:
        n, h, w = ref.find_gen_fwd_shape(regime, sms)
        blocks = ref.gen_fwd_blocks(n, h, sms)
        if regime == "wide_rows":
            assert blocks == n * h and w > 256
        else:
            assert blocks == 8 * sms and n * h // blocks >= 2 and n * h % blocks != 0 and w % 2 == 1
    widths = ref.find_tail_bwd_widths()
    items = [it for w in widths for it in ref.tail_bwd_row_items(w)]
    assert {(it.scale, it.rgroups) for it in items} == ref.tail_bwd_reachable()
    assert {it.wpad for it in items} & set(ref.IDLE_WPADS)
    assert any(ref._full_and_short(w) for w in widths) and len(widths) <= 12
    for regime in ref.CBCE_REGIMES:
        numels = ref.find_cbce_numels(regime, sms)
        assert {m % 4 for m in numels} >= {1, 2, 3}
        grids = {ref.loss_grid(m, sms) for m in numels}
        if regime == "tiny":
            assert grids == {1} and max(numels) < 4
        elif regime == "one_block":
            assert grids == {1} and all(m // 4 < ref.LOSS_THREADS for m in numels)
        else:
            assert grids == {8 * sms} and {ref.loss_vectors_per_thread(m, sms) for m in numels} == {3}


def test_plans_by_hand():
    p = ref.conv_first_plan(2, 21, 37, True, False, 132)
    assert p.inst == (1, False) and p.tiles == 20 and p.grid == 20
    q = ref.first_wgrad_plan(2, 600, 193, 132)
    assert q.chunks_x == 4 and q.tiles == 4800 and q.grid == 528 and q.last_valid == 1
    assert q.block_tiles[0][:3] == (0, 528, 1056) and q.dgrad_grid == (2, 600, 2)
    assert q.det_workspace_floats == 528 * 1728 + 64 * 1728
    assert ref.tail_bwd_row_items(513)[0] == ref.TailBwdItem(0, 2, 0, 255, 512, 256, 1)
    assert ref.tail_bwd_row_items(513)[1] == ref.TailBwdItem(0, 2, 1, 2, 6, 32, 8)
    assert ref.tail_bwd_depth(ref.TailBwdItem(3, 16, 0, 7, 128, 128, 2)) == 16 + 2 + 1 + 5 + 1
    g = ref.gen_bwd_plan(1, 17, 40)
    assert g.segs == (2, 1, 1, 1) and g.nrows == (18, 5, 3, 2)


def test_parse_train_kernel_names():
    parse = ref.parse_train_kernel_name
    assert parse("void osvos::conv_first_tc_kernel<2, true>(float const*, float const*, osvos::OutMaps, "
                 "osvos::ConvParams)") == ("conv_first_tc_kernel", (2, True))
    assert parse("void osvos::conv_first_tc_kernel<(int)1, (bool)0>(x)") == ("conv_first_tc_kernel", (1, False))
    assert parse("void osvos::conv_first_wgrad_kernel<true>(float const*, x)") == ("conv_first_wgrad_kernel", (True,))
    assert parse("void osvos::tail_bwd2_kernel<true, false>(osvos::TailBwdParams)") == \
        ("tail_bwd2_kernel", (True, False))
    assert parse("void osvos::tail_general_bwd_kernel<(bool)1>(x)") == ("tail_general_bwd_kernel", (True,))
    assert parse("void osvos::cbce_fwd_kernel<false>(float const*, float const*, unsigned long, double*, double, "
                 "float*)") == ("cbce_fwd_kernel", (False,))
    assert parse("osvos::conv_first_dgrad_kernel(__nv_bfloat16 const*, __nv_bfloat16 const*, float const*, float*, "
                 "int, int, int)") == ("conv_first_dgrad_kernel", ())
    for name in ref.PLAIN_KERNELS:
        assert parse(f"void osvos::{name}(int)") == (name, ())
    assert parse("void osvos::sum_f32_det_kernel(float const*)") == ("sum_f32_det_kernel", ())
    assert parse("void osvos::tail_fwd_kernel<true>(osvos::TailParams)") is None
    assert parse("void osvos::my_sum_f32_kernel(int)") is None
    assert parse("void osvos::side_conv_kernel<2, 16>(x)") is None
    assert parse_kernel_name("void osvos::conv_first_tc_kernel<2, true>(x)") is None    # the default set is unchanged


def test_compiled_train_instantiations(lib):
    """conv_first_tc_kernel {1, 2} x {false, true}, conv_first_wgrad_kernel {false, true}, tail_bwd2_kernel
    {false, true}^2, tail_general_bwd_kernel {false, true} and cbce_fwd_kernel {false, true} - no more, no fewer; and
    each plain kernel named here exists."""
    from osvos_pytorch_b200 import build
    cuobjdump, cufilt = _cuda_tool("cuobjdump"), _cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt not found next to nvcc")
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = subprocess.run([cufilt], input=syms, capture_output=True, text=True, check=True).stdout
    found = {}
    for p in map(ref.parse_train_kernel_name, names.splitlines()):
        if p:
            found.setdefault(p[0], []).append(p[1])
    assert set(found) == set(ref.COMPILED) | set(ref.PLAIN_KERNELS)
    for kernel, want in ref.COMPILED.items():
        assert len(found[kernel]) == len(set(found[kernel])) and set(found[kernel]) == want, (kernel, found[kernel])
    assert sum(len(v) for v in ref.COMPILED.values()) == 14
    for kernel in ref.PLAIN_KERNELS:
        assert found[kernel] == [()], (kernel, found[kernel])

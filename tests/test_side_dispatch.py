"""CPU checks of the host restatement of the side-branch, unpool and tail launch plans (tests/side_dispatch_ref.py): it
agrees with the library's own planning queries, it reaches every regime at any plausible SM count, and the kernels
compiled into the library are exactly the instantiations planned there.  No GPU needed: the library loads on a CPU box,
where its SM count is the H100's 132."""
import itertools
import subprocess

import pytest

import side_dispatch_ref as ref
from conv_dispatch_ref import parse_kernel_name
from test_conv_dispatch import _cuda_tool

HOST_SMS = 132      # device_sm_count() without a device


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat, build
    build.build()
    return nat.load()


SIZES = [(1, 1), (3, 5), (8, 8), (9, 17), (16, 24), (31, 45), (60, 107), (97, 131), (120, 214), (240, 427), (480, 854)]


def test_unpool_colsum_rows_is_the_grid(lib):
    for n, (h, w), c, pool, side in itertools.product((1, 2, 3, 12), SIZES, ref.UNPOOL_CHANNELS + (8, 16, 32),
                                                      (False, True), (False, True)):
        plan = ref.unpool_plan(n, h, w, c, pool, side, True, HOST_SMS)
        assert lib.osvos_unpool_colsum_rows(n, h, w, c, int(pool), int(side)) == plan.grid, (n, h, w, c, pool, side)
    assert lib.osvos_unpool_colsum_rows(1, 8, 8, 48, 1, 0) == 0          # 256 % (c / 8) != 0: refused


def _sw_items(shapes):
    from osvos_pytorch_b200 import _native as nat
    arr = (nat.SideWgradItem * len(shapes))()
    for k, (it, (n, h, w, c)) in enumerate(zip(arr, shapes)):
        # the plan encodes no tensor maps for the workspace query: any non-null 16-byte-aligned pointers
        it.x_hi, it.x_lo, it.dpq, it.g = 0x10000 * (k + 1), 0x20000 * (k + 1), 0x30000 * (k + 1), 0x40000 * (k + 1)
        it.n, it.h, it.w, it.c = n, h, w, c
    return arr


SW_SHAPES = [(n, h, w, c) for n in (1, 2, 12) for h, w in SIZES for c in (128, 256, 512)]


@pytest.mark.parametrize("count", [1, 2, 3, 4])
def test_side_wgrad_workspace_query_matches(lib, count):
    """osvos_side_folded_wgrad_workspace_bytes of the deterministic form is the restated partial rows plus the row
    reduction's scratch, over 1 - 4 scales; the default form needs none."""
    from osvos_pytorch_b200._native import FLAG_DETERMINISTIC as DET
    for k in range(0, len(SW_SHAPES), 7):
        shapes = [SW_SHAPES[(k + 13 * j) % len(SW_SHAPES)] for j in range(count)]
        plan = ref.side_wgrad_plan(shapes, HOST_SMS)
        got = lib.osvos_side_folded_wgrad_workspace_bytes(_sw_items(shapes), count, DET)
        assert got == 4 * plan.workspace_floats, (shapes, got, plan)
        assert lib.osvos_side_folded_wgrad_workspace_bytes(_sw_items(shapes), count, 0) == 0
        assert plan.total_blocks <= 2 * HOST_SMS + 4 * count * 4
        for sc in plan.scales:
            assert 1 <= sc.blocks_per_slab <= sc.chunks and sum(sc.chunks_per_block) == sc.chunks
    assert lib.osvos_side_folded_wgrad_workspace_bytes(_sw_items([(1, 8, 8, 64)]), 1, DET) == 0


def test_tail_det_sums_match(lib):
    for n, (h, w) in itertools.product((1, 2, 3, 12), SIZES):
        want = ref.TAIL_SUMS + ref.TAIL_VALS * ref.tail_fwd_blocks(n, h, HOST_SMS)
        assert ref.tail_det_sums(n, h, HOST_SMS) == want
        assert lib.osvos_tail_fwd_deterministic_sums(n, h, w) == want, (n, h, w)


def test_side_conv_plan_deals_round_robin():
    p = ref.side_conv_plan([(2, 45, 65, 128, 2), (2, 12, 17, 512, 2), (2, 23, 33, 256, 2), (2, 6, 9, 512, 2)], True, 132)
    assert p.inst == (1, 2)
    assert [s[3] for s in p.scales] == [512, 512, 256, 128] and p.scales[0][1] == 12     # deepest first, ties in order
    assert p.tile_begin == (0, 12, 16, 46) and p.total_tiles == 136 and p.grid == 132
    assert p.cta_tiles[0] == (0, 132) and p.cta_tiles[131] == (131,)
    assert ref.crossing_ctas(p) == [0, 1, 2, 3]
    assert ref.side_conv_plan([(1, 21, 19, 64, 16)], False, 132).grid == 9


@pytest.mark.parametrize("sms", range(60, 145))
def test_every_regime_is_found_at_sms(sms):
    """The searches the GPU file runs reach every regime at any SM count from 60 to 144, with the promised shapes."""
    for regime in ref.SIDE_REGIMES:
        n, h, w = ref.find_side_shape(regime, sms)
        assert n >= 2 and h % 10 != 0 and w % 8 != 0
        for nco in (2, 16):
            p = ref.side_conv_plan([(n, h, w, 128, nco)], False, sms)
            counts = {len(t) for t in p.cta_tiles}
            if regime == "one_wave":
                assert p.total_tiles <= sms and counts == {1}
            else:
                assert p.grid == sms and counts == {p.total_tiles // sms, p.total_tiles // sms + 1}
                assert min(counts) >= 2 and {c % 2 for c in counts} == {0, 1}
    for count in (2, 3, 4):
        n, h, w = ref.find_side_multi_shape(count, sms)
        shapes = ref.multi_scale_shapes(h, w, count)
        assert n >= 2 and all(hh % 10 != 0 and ww % 8 != 0 for hh, ww, _ in shapes)
        assert [c for _, _, c in shapes] == list(ref.SIDE_MULTI_CINS[count])
        p = ref.side_conv_plan([(n, hh, ww, c, 2) for hh, ww, c in shapes], False, sms)
        cross = ref.crossing_ctas(p)
        assert cross and p.total_tiles > sms and p.total_tiles % sms != 0
        # a crossing CTA's tiles have different chunk counts
        assert any(len({p.scales[p.scale_of(t)][3] for t in p.cta_tiles[b]}) > 1 for b in cross)
    for regime in ref.SW_REGIMES:
        items = ref.find_sw_items(regime, sms)
        assert items is not None, (regime, sms)
        assert all(it[0] >= 2 and it[2] % 2 == 1 for it in items)
        p = ref.side_wgrad_plan(items, sms)
        s0 = p.scales[0]
        if regime == "one_chunk":
            assert set(s0.chunks_per_block) == {1} and s0.blocks_per_slab > 1
        elif regime == "ring_wraps":
            assert s0.chunks_per_block[0] > 2 * ref.SW_STAGES and len(set(s0.chunks_per_block)) == 2
        elif regime == "clamped":
            assert len(items) == 3 and {sc.blocks_per_slab == 1 for sc in p.scales} == {True, False}
        else:
            assert items[0][2] < ref.SW_CHUNK and s0.chunks_per_block[0] > 1
    for pool, side, det, wf in ref.unpool_targets():
        for c in ref.UNPOOL_CHANNELS:
            n, h, w = ref.find_unpool_shape(pool, side, det, wf, c, sms)
            p = ref.unpool_plan(n, h, w, c, pool, side, det, sms)
            assert n >= 2 and h % 2 == 1 and w % 2 == 1
            assert p.tiles > p.grid and p.wf_in_smem == wf and p.inst == (pool, side, det)
    n, h, w = ref.find_tail_shape(sms)
    blocks = ref.tail_fwd_blocks(n, h, sms)
    assert n * h > 8 * sms and blocks == 8 * sms and w % 2 == 1 and n * h // blocks >= 2


def test_parse_side_kernel_names():
    assert ref.parse_side_kernel_name("void osvos::side_conv_kernel<2, 16>(osvos::SideMaps, osvos::SideParams)") == \
        ("side_conv_kernel", (2, 16))
    assert ref.parse_side_kernel_name("void osvos::side_conv_kernel<(int)1, (int)2>(x)") == ("side_conv_kernel", (1, 2))
    assert ref.parse_side_kernel_name("void osvos::unpool_add_mask_kernel<true, false, (bool)1>(x)") == \
        ("unpool_add_mask_kernel", (True, False, True))
    assert ref.parse_side_kernel_name("void osvos::side_folded_wgrad_kernel<false>(SwMaps)") == \
        ("side_folded_wgrad_kernel", (False,))
    assert ref.parse_side_kernel_name("void osvos::tail_fwd_kernel<(bool)1>(osvos::TailParams)") == \
        ("tail_fwd_kernel", (True,))
    assert ref.parse_side_kernel_name("void osvos::tail_bwd2_kernel<true, false>(x)") is None
    assert ref.parse_side_kernel_name("void osvos::conv3x3_halo_kernel<128, 2, true, false, false, false>(x)") is None
    assert parse_kernel_name("void osvos::side_conv_kernel<16, 2>(int)") is None     # the default set is unchanged


def test_compiled_instantiations(lib):
    """side_conv_kernel {1, 2} x {2, 16}, all eight unpool_add_mask_kernel<POOL, SIDE, DET>, and both forms of the
    folded G and tail forward kernels - no more, no fewer."""
    from osvos_pytorch_b200 import build
    cuobjdump, cufilt = _cuda_tool("cuobjdump"), _cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt not found next to nvcc")
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = subprocess.run([cufilt], input=syms, capture_output=True, text=True, check=True).stdout
    found = {}
    for p in map(ref.parse_side_kernel_name, names.splitlines()):
        if p:
            found.setdefault(p[0], []).append(p[1])
    assert set(found) == set(ref.COMPILED)
    for kernel, want in ref.COMPILED.items():
        assert len(found[kernel]) == len(set(found[kernel])) and set(found[kernel]) == want, (kernel, found[kernel])

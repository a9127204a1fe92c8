"""CPU checks of the host restatement of the convolution dispatchers (tests/conv_dispatch_ref.py): it agrees with the
library's own planning entry points, it reaches every schedule at any plausible SM count, and the halo kernels compiled
into the library are exactly the ones the dispatcher can pick.  No GPU needed: the library loads on a CPU box."""
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

import conv_dispatch_ref as ref


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat, build
    build.build()
    return nat.load()


SIZES = [(5, 3), (8, 8), (9, 17), (16, 24), (31, 45), (60, 107), (97, 131), (120, 214), (240, 427), (480, 854)]
CHANNELS = [(64, 64), (64, 128), (64, 512), (128, 128), (128, 64), (256, 256), (512, 512), (128, 512), (512, 256)]


@pytest.mark.parametrize("cin,dz", CHANNELS)
def test_wgrad_plan_matches_deterministic_splits(lib, cin, dz):
    """plan_wgrad at the nominal 132 SMs is what osvos_wgrad_deterministic_splits reports, over every item mode, batches
    1 - 3 and 5x3 .. 480x854."""
    for n, (h, w) in itertools.product((1, 2, 3), SIZES):
        plan = ref.wgrad_plan(n, h, w, dz, cin, ref.WGRAD_NOMINAL_SMS)
        assert plan.splits == lib.osvos_wgrad_deterministic_splits(n, h, w, cin, dz), (n, h, w, cin, dz, plan)
        assert plan.patches_per_split * (plan.splits - 1) < plan.patches_total <= plan.patches_per_split * plan.splits
        assert plan.total_items == plan.m_blocks * plan.n_blocks * plan.tap_items * plan.splits
        want = "tap_rows" if (cin, dz) == (64, 64) else "tap_pairs" if cin == 64 else "nine_taps"
        assert plan.mode == want


def test_wgrad_plan_refuses_dz_channels_192(lib):
    with pytest.raises(ValueError):
        ref.wgrad_plan(1, 16, 16, 192, 128, 132)
    assert lib.osvos_wgrad_deterministic_splits(1, 16, 16, 128, 192) == 0


def test_colsum_rows_matches_tile_count(lib):
    for n, (h, w) in itertools.product((1, 2, 3), SIZES):
        tiles = -(-h // ref.TILE_H) * -(-w // ref.TILE_W) * n
        assert lib.osvos_conv3x3_colsum_rows(n, h, w) == 8 * tiles


def test_reachable_halo_set():
    assert len(ref.REACHABLE_HALO) == 22
    for block_n, planes, split, lean, pingpong, det in ref.REACHABLE_HALO:
        assert not (lean and det) and not (lean and planes == 1)
        assert block_n != 256 or (planes == 1 and not pingpong)


def test_halo_plan_stays_inside_reachable_set():
    """Over a grid of shapes, flags and SM counts every plan is one of REACHABLE_HALO, and each of them occurs."""
    seen = set()
    for sms in (78, 114, 132):
        for m, cout in itertools.product(range(1, 3 * sms + 2, 7), (64, 128, 256, 384, 512)):
            for fast, lean, det in itertools.product((False, True), repeat=3):
                if lean and det:
                    continue
                target, total = ref.halo_plan(m, 16, 8, 64, cout, fast, lean, det, sms)
                assert target in ref.REACHABLE_HALO, (m, cout, fast, lean, det, sms, target)
                assert total == m * cout // target[0]
                seen.add(target)
    assert seen == ref.REACHABLE_HALO


def test_exact_mode_never_prefers_256_wide_tiles():
    """Exact mode's former N = 256 rule, waves256 * 2200 < waves128 * 1000, never holds: for T tiles of 256 on S SMs
    waves128 = ceil(2T / S) <= 2 ceil(T / S) = 2 waves256.  Checked for every S <= 300 and T <= 3000."""
    s = np.arange(1, 301, dtype=np.int64)[:, None]
    t = np.arange(1, 3001, dtype=np.int64)[None, :]
    waves256 = -(-t // s)
    waves128 = -(-(2 * t) // s)
    assert not np.any(waves256 * 2200 < waves128 * 1000)
    # the fast-mode rule does select N = 256 somewhere, and the restated dispatcher follows it
    assert np.any(waves256 * 1100 < waves128 * 700)
    for sms in (60, 132, 300):
        for m in range(1, 3001, 13):
            assert ref.halo_plan(m, 16, 8, 64, 512, False, False, False, sms)[0][0] != 256


@pytest.mark.parametrize("sms", range(60, 145))
def test_every_schedule_is_found_at_sms(sms):
    """halo_cases / wgrad_cases (what the GPU file runs) reach every target at any SM count from 60 to 144, with the
    shape constraints the search promises."""
    cases = ref.halo_cases(sms)
    assert sorted(t for t, _ in cases) == sorted(ref.REACHABLE_HALO)
    for target, s in cases:
        assert s is not None, (sms, target)
        assert ref.halo_plan(s.n, s.h, s.w, s.cin, s.cout, s.fast, s.lean, s.det, sms) == (target, s.total_tiles)
        assert s.w % 8 != 0 and s.h % 16 != 0 and s.n >= 2
        # more tiles than CTAs (grid = sms), unevenly dealt: some CTAs run a second tile, cooperative or ping-pong
        assert s.total_tiles > sms and s.total_tiles % sms != 0
        # fewer tiles per image than CTAs: CTA b's tiles b and b + sms lie in different images
        assert s.total_tiles // s.n < sms
    assert any(s.cin == 192 for _, s in cases) and any(s.cout == 384 for _, s in cases)
    seen = set()
    for cid, mode, regime, fast, det, n, h, w, cin, dz, plan in ref.wgrad_cases(sms):
        assert plan == ref.wgrad_plan(n, h, w, dz, cin, ref.WGRAD_NOMINAL_SMS if det else sms)
        assert plan.mode == mode and h % 8 != 0 and w % 8 != 0
        if regime == "splits":
            assert plan.splits > 1 and plan.patches_total % plan.patches_per_split != 0
        elif regime == "one_split":
            assert plan.splits == 1
        else:
            assert plan.total_items > sms and plan.patches_per_split > 6
        seen.add(cid)
    assert len(seen) == 28


def test_find_halo_shape_example_at_132():
    """Ping-pong at N = 64 from 3x29x357 (270 tiles: 2 or 3 per CTA), at N = 128 with three N blocks from 3x29x117
    (90 pixel tiles x 3 N blocks), and the cooperative N = 128 exact form from 3x29x61 (144 tiles: 1 or 2 per CTA)."""
    s = ref.find_halo_shape((64, 2, True, False, True, False), 132)
    assert (s.n, s.h, s.w, s.cout, s.total_tiles) == (3, 29, 357, 64, 270)
    s = ref.find_halo_shape((128, 2, False, False, True, False), 132, cin=192, couts=(384,))
    assert (s.n, s.h, s.w, s.cout, s.total_tiles) == (3, 29, 117, 384, 270)
    s = ref.find_halo_shape((128, 2, True, False, False, False), 132, cin=192, couts=(384,))
    assert (s.n, s.h, s.w, s.cout, s.total_tiles) == (3, 29, 61, 384, 144)


def test_parse_kernel_name_both_spellings():
    a = "void osvos::conv3x3_halo_kernel<128, 2, true, false, false, false>(CUtensorMap_st, CUtensorMap_st, " \
        "CUtensorMap_st, CUtensorMap_st, osvos::ConvParams)"
    b = "void osvos::conv3x3_halo_kernel<(int)128, (int)2, (bool)1, (bool)0, (bool)0, (bool)0>(CUtensorMap_st, " \
        "CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, osvos::ConvParams)"
    want = ("conv3x3_halo_kernel", (128, 2, True, False, False, False))
    assert ref.parse_kernel_name(a) == want and ref.parse_kernel_name(b) == want
    for t, v in zip(ref.parse_kernel_name(a)[1], want[1]):
        assert type(t) is type(v)
    assert ref.parse_kernel_name("osvos::wgrad_tc_kernel<(int)128, (int)1, (bool)1>(x)") == \
        ("wgrad_tc_kernel", (128, 1, True))
    assert ref.parse_kernel_name("void osvos::wgrad_tc_kernel<128, 2, false>(CUtensorMap_st)") == \
        ("wgrad_tc_kernel", (128, 2, False))
    assert ref.parse_kernel_name("void osvos::wgrad_finish_kernel<true>(float const*)") is None
    assert ref.parse_kernel_name("void osvos::side_conv_kernel<16, 2>(int)") is None


def _cuda_tool(name):
    from osvos_pytorch_b200 import build
    try:
        path = os.path.join(os.path.dirname(build._nvcc()), name)
    except RuntimeError:
        path = None
    if path is None or not os.path.exists(path):
        path = shutil.which(name)
    return path


def test_compiled_halo_kernels_are_the_reachable_set(lib):
    """The conv3x3_halo_kernel instantiations in libosvos_b200.so are exactly REACHABLE_HALO (22): every compiled
    schedule is one the dispatcher can pick, and tests/test_gpu_conv_schedules.py runs each of them."""
    from osvos_pytorch_b200 import build
    cuobjdump, cufilt = _cuda_tool("cuobjdump"), _cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt not found next to nvcc")
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = subprocess.run([cufilt], input=syms, capture_output=True, text=True, check=True).stdout
    halo = [p[1] for p in map(ref.parse_kernel_name, names.splitlines()) if p and p[0] == "conv3x3_halo_kernel"]
    assert len(halo) == len(set(halo)) == 22, sorted(halo)
    assert set(halo) == ref.REACHABLE_HALO
    wgrad = {p[1] for p in map(ref.parse_kernel_name, names.splitlines()) if p and p[0] == "wgrad_tc_kernel"}
    assert wgrad == {(128, planes, det) for planes in (1, 2) for det in (False, True)}

"""CPU checks of tests/general_tail_dispatch_ref.py: the general tail backward's item walk is the library's plan, the
shape search reaches every segment regime and the other cases the GPU file relies on, the side finish's launch plan,
and the kernel names it parses.  No GPU needed."""
import subprocess

import pytest

import general_tail_dispatch_ref as gtr
import train_dispatch_ref as tdr
from test_conv_dispatch import _cuda_tool


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat, build
    build.build()
    return nat.load()


GEN_SHAPES = gtr.find_gen_bwd_shapes()


def test_general_tail_bwd_regimes_are_reached():
    """The shapes tests/test_gpu_general_tail_schedules.py runs reach, at every scale: one short segment, only full
    segments, a one-pixel last segment after full ones and several segments with a ragged last one, each with odd and
    even w; hk = 1 (h = 1 and 2) and w = 1; top and left from odd and from even (hk + 1) s - h and (wk + 1) s - w;
    n = 1 and 3; the 480 x 854 frame; row reductions of 1, fewer than 64 and more than 4096 rows."""
    assert GEN_SHAPES is not None and GEN_SHAPES[-1] == gtr.GEN_FRAME == (1, 480, 854)
    assert len(GEN_SHAPES) <= 10 and all(h * w <= 13 * 400 for _, h, w in GEN_SHAPES[:-1])
    reached = set()
    for n, h, w in GEN_SHAPES:
        for k, (hk, wk, s, top, left) in enumerate(tdr.tail_scales(h, w)):
            segs = -(-wk // tdr.GEN_SEG)
            nouts = [it.nout for it in gtr.gen_bwd_items(1, 1, w) if it.scale == k]
            assert len(nouts) == segs and all(x == tdr.GEN_SEG for x in nouts[:-1])
            last = nouts[-1]
            if segs == 1 and wk < tdr.GEN_SEG:
                reached.add((k, "short", w % 2))
            elif segs >= 2 and last == 1:
                reached.add((k, "one_px", w % 2))
            elif segs >= 2 and 1 < last < tdr.GEN_SEG:
                reached.add((k, "ragged", w % 2))
            elif last == tdr.GEN_SEG:
                reached.add((k, "full", w % 2))
            reached |= {(k, "hk1")} if hk == 1 else set()
            reached |= {(k, "top", ((hk + 1) * s - h) % 2), (k, "left", ((wk + 1) * s - w) % 2)}
            nrows = tdr.gen_bwd_plan(n, h, w).nrows[k]
            reached.add("rows=1" if nrows == 1 else "rows<64" if nrows < 64 else "rows>4096" if nrows > 4096 else "")
            if k == 0 and segs > 1 and nrows > 4096 and -(-nrows // tdr.RED_SEGS) > 8:
                reached.add("frame: several segments, several row lanes")
        reached |= {("n", n), ("w=1", w == 1)}
    want = {(k, r, p) for k in range(4) for r in gtr.GEN_SEG_REGIMES for p in (0, 1)}
    want |= {(k, "hk1") for k in range(4)} | {(k, e, p) for k in range(4) for e in ("top", "left") for p in (0, 1)}
    want |= {"rows=1", "rows<64", "rows>4096", "frame: several segments, several row lanes", ("n", 1), ("n", 3),
             ("w=1", True)}
    assert want <= reached, want - reached
    assert {(n, h) for n, h, _ in GEN_SHAPES} >= {(1, 1), (3, 2)}     # hk = 1 at every scale with h = 1 and h = 2


@pytest.mark.parametrize("shape", GEN_SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in GEN_SHAPES])
def test_general_tail_bwd_items_cover_the_plan(lib, shape):
    """The items of gen_bwd_items are gen_bwd_plan's blocks, in launch order: per scale their nout add up to n hk wk,
    they visit every source pixel (img, iy, ix) exactly once, and each window starts where its first source's 2s x 2s
    taps land in the cropped map; the library's workspace query agrees with the plan."""
    n, h, w = shape
    plan = tdr.gen_bwd_plan(n, h, w)
    items = gtr.gen_bwd_items(n, h, w)
    assert len(items) == plan.items and lib.osvos_tail_general_bwd_workspace_bytes(n, h, w) == 4 * plan.workspace_floats
    first = 0
    for k, (hk, wk, s, top, left) in enumerate(tdr.tail_scales(h, w)):
        mine = items[first:first + plan.nrows[k]]
        first += plan.nrows[k]
        assert {it.scale for it in mine} == {k} and sum(it.nout for it in mine) == n * hk * wk
        pix = [(it.img, it.iy, tdr.GEN_SEG * it.seg + j) for it in mine for j in range(it.nout)]
        assert len(pix) == len(set(pix)) and all(0 <= i < n and 0 <= y < hk and 0 <= x < wk for i, y, x in pix)
        for it in mine:
            assert 1 <= it.nout <= tdr.GEN_SEG and it.seg < plan.segs[k]
            assert it.y0 + top == it.iy * s and it.x0 + left == tdr.GEN_SEG * it.seg * s
    assert first == len(items)


def test_general_tail_bwd_items_by_hand():
    items = gtr.gen_bwd_items(2, 1, 257)
    s0 = [it for it in items if it.scale == 0]                            # wk = 129: 9 segments, the last of 1
    assert len(s0) == 18 and s0[8] == gtr.GenBwdItem(0, 0, 0, 8, 1, -1, 256 - 1) and s0[9].img == 1
    s3 = [it for it in items if it.scale == 3]                            # wk = 17, top = (32 - 1) // 2
    assert [it.nout for it in s3] == [16, 1, 16, 1] and s3[1] == gtr.GenBwdItem(3, 0, 0, 1, 1, -15, 256 - 15)
    assert gtr.gen_seg_regime(15) == "short" and gtr.gen_seg_regime(32) == "full"
    assert gtr.gen_seg_regime(33) == "one_px" and gtr.gen_seg_regime(18) == "ragged"


def test_side_finish_plan():
    """osvos_side_grads_finish: 16 blocks per table entry, 18 (cmax + 1) + 2 floats of shared memory, and the opt-in
    above 48 KB, first needed at cmax = 682."""
    assert gtr.side_finish_plan((128, 256, 512, 512)) == gtr.SideFinishPlan(64, (18 * 513 + 2) * 4, False)
    assert gtr.side_finish_plan((512, 128)) == gtr.side_finish_plan((128, 512)) == (32, (18 * 513 + 2) * 4, False)
    assert gtr.side_finish_plan((1024,)) == gtr.SideFinishPlan(16, (18 * 1025 + 2) * 4, True)
    assert not gtr.side_finish_plan((681,)).opt_in and gtr.side_finish_plan((64, 682)).opt_in


def test_parse_general_tail_kernel_names():
    parse = gtr.parse_general_tail_kernel_name
    assert parse("void osvos::side_grads_finish_kernel(osvos::SideGradTable)") == ("side_grads_finish_kernel", ())
    assert parse("void osvos::tail_general_bwd_kernel<(bool)1>(x)") == ("tail_general_bwd_kernel", (True,))
    assert parse("void osvos::reduce_rows_final_kernel(float const*)") == ("reduce_rows_final_kernel", ())
    assert parse("void osvos::my_side_grads_finish_kernel(int)") is None


def test_side_grads_finish_kernel_is_compiled_once(lib):
    from osvos_pytorch_b200 import build
    cuobjdump, cufilt = _cuda_tool("cuobjdump"), _cuda_tool("cu++filt")
    if cuobjdump is None or cufilt is None:
        pytest.skip("cuobjdump / cu++filt not found next to nvcc")
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = subprocess.run([cufilt], input=syms, capture_output=True, text=True, check=True).stdout
    found = [p for p in map(gtr.parse_general_tail_kernel_name, names.splitlines()) if p and p[0] in gtr.FINISH_KERNELS]
    assert found == [("side_grads_finish_kernel", ())], found

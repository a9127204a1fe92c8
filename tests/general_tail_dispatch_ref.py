"""Host restatement of the general tail's backward grid and of the folded tail's parameter-gradient finish, and a
search for small shapes that reach every segment regime of the backward.  Built on tests/train_dispatch_ref.py
(tail_scales, gen_bwd_plan, the kernel names of the training step), which it leaves as it is.

- `gen_bwd_items` walks `tail_general_bwd_kernel`'s grid item by item (csrc/tail_general.cu): scale, image, source row,
  segment, its source columns and its window origin.
- `find_gen_bwd_shapes` finds small shapes whose segments reach every regime at each scale, then adds the DAVIS frame.
- `side_finish_plan` restates the launch of `side_grads_finish_kernel` (csrc/side_bwd_folded.cu).
- `parse_general_tail_kernel_name` is train_dispatch_ref's kernel-name parser plus `side_grads_finish_kernel`.

tests/test_general_tail_dispatch.py checks the restatements against the library, and
tests/test_gpu_general_tail_schedules.py runs the shapes found here against fp64 and checks which kernels ran."""
import re
from typing import NamedTuple

from train_dispatch_ref import GEN_SEG, parse_train_kernel_name, tail_scales

# plain kernels of this file's calls that train_dispatch_ref does not name: matched by exact name
FINISH_KERNELS = ("side_grads_finish_kernel",)
_FINISH_RE = re.compile(r"\b(" + "|".join(FINISH_KERNELS) + r")\(")


def _cdiv(a, b):
    return -(-a // b)


def parse_general_tail_kernel_name(name):
    """train_dispatch_ref.parse_train_kernel_name, and (kernel, ()) of FINISH_KERNELS; else None."""
    p = parse_train_kernel_name(name)
    if p is not None:
        return p
    m = _FINISH_RE.search(name)
    return (m.group(1), ()) if m else None


class GenBwdItem(NamedTuple):
    scale: int
    img: int
    iy: int                     # source row
    seg: int                    # segment of GEN_SEG source columns within the row
    nout: int                   # source columns of the segment: min(GEN_SEG, wk - GEN_SEG seg)
    y0: int                     # window origin in the cropped map: iy s - top
    x0: int                     # GEN_SEG seg s - left


def gen_bwd_items(n, h, w):
    """The grid of tail_general_bwd_kernel block by block: the blocks of scale k start at gen_bwd_plan's first item of
    k, and block `local` of a scale is (img, iy, seg) with seg fastest, then iy, then img."""
    out = []
    for k, (hk, wk, s, top, left) in enumerate(tail_scales(h, w)):
        segs = _cdiv(wk, GEN_SEG)
        for local in range(n * hk * segs):
            seg, rowi = local % segs, local // segs
            iy, img = rowi % hk, rowi // hk
            out.append(GenBwdItem(k, img, iy, seg, min(GEN_SEG, wk - GEN_SEG * seg), iy * s - top,
                                  GEN_SEG * seg * s - left))
    return out


# the segment regimes of one scale, from its width wk: a single segment shorter than GEN_SEG; only full segments;
# a last segment of one source column after at least one full one; several segments, the last of 2 .. GEN_SEG - 1
GEN_SEG_REGIMES = ("short", "full", "one_px", "ragged")
GEN_FRAME = (1, 480, 854)                # the DAVIS frame: scale 0 reduces n hk segs = 6480 partial rows
GEN_BWD_NH = ((1, 1), (3, 2), (1, 13), (3, 6))   # (n, h) of the found widths, in turn


def gen_seg_regime(wk):
    last = wk - GEN_SEG * (_cdiv(wk, GEN_SEG) - 1)
    if wk < GEN_SEG:
        return "short"
    if last == GEN_SEG:
        return "full"
    return "one_px" if last == 1 else "ragged"


def gen_bwd_regimes(w):
    """{(scale, segment regime, w % 2)} of a width: the segments depend on w only, and since s is even, the parity
    of (wk + 1) s - w (whether `left` halves it exactly or floors) is the parity of w at every scale."""
    return {(k, gen_seg_regime(wk), w % 2) for k, (_, wk, _, _, _) in enumerate(tail_scales(1, w))}


def find_gen_bwd_shapes(limit=1024):
    """(n, h, w) shapes of the general tail's backward that together reach every segment regime at each of the four
    scales with odd and with even w, then the DAVIS frame (GEN_FRAME).  Greedy and deterministic: take the width
    1 <= w < limit that adds the most (scale, regime, parity) triples not yet reached, the narrowest on ties, until all
    32 are reached.  The found widths get (n, h) from GEN_BWD_NH in turn: h = 1 and 2 give hk = 1 at every scale,
    h = 13 and 6 several source rows, and odd and even h give odd and even (hk + 1) s - h, as for w."""
    want = {(k, r, p) for k in range(4) for r in GEN_SEG_REGIMES for p in (0, 1)}
    have, widths = set(), []
    while have != want:
        gain, w = max((len(gen_bwd_regimes(w) - have), -w) for w in range(1, limit))
        if gain == 0:
            return None
        widths.append(-w)
        have |= gen_bwd_regimes(-w)
    shapes = [GEN_BWD_NH[i % len(GEN_BWD_NH)] + (w,) for i, w in enumerate(widths)]
    return shapes + [GEN_FRAME]


class SideFinishPlan(NamedTuple):
    grid: int                   # 16 blocks (one per side feature f) per table entry
    smem_bytes: int             # G of the widest entry at pitch c + 1, and S
    opt_in: bool                # above the 48 KB default: the kernel's attribute is raised first


def side_finish_plan(cs):
    """osvos_side_grads_finish's launch for a table of entries with channels cs (csrc/side_bwd_folded.cu)."""
    assert 1 <= len(cs) <= 4 and max(cs) <= 2048
    smem = (18 * (max(cs) + 1) + 2) * 4
    return SideFinishPlan(16 * len(cs), smem, smem > 48 * 1024)



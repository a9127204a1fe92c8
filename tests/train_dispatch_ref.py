"""Host restatement of the launch plans of the kernels at both ends of a training step - conv1_1 forward and backward,
the tail backward, the general-weights tail, the class-balanced loss and the reductions - and a search for small shapes
that reach each of their regimes at a given SM count.

- `conv_first_plan` restates `conv_first_tc_launch` (csrc/conv_first_tc.cu): `conv_first_tc_kernel<PLANES, STAGED>`,
  8 x 16 pixel tiles, grid = min(tiles, SMs), the tiles each CTA walks.
- `first_wgrad_plan` restates the conv1_1 backward (csrc/bwd_kernels.cu): `conv_first_wgrad_kernel<DET>`'s 64-pixel
  row chunks, grid = clamp(tiles, 1, 4 SMs), the last chunk's valid pixels, each block's tile list, the deterministic
  workspace (grid slots of 1728 floats + the row reduction's scratch) and `conv_first_dgrad_kernel`'s grid.
- `tail_bwd_scales` and `tail_bwd_row_items` restate `fill_tail_bwd_scales` (csrc/tail.cu) and, per work item of `tail_bwd2_kernel<LOSS, DET>`,
  the segment's low-res columns, its source width, the padded width and the row groups of phase 1.
- `gen_fwd_blocks` / `gen_fwd_sums` and `gen_bwd_plan` restate the general-weights tail's plans (csrc/tail_general.cu);
  `find_gen_fwd_shape` finds shapes for the forward's two regimes (one row per block, rows strided over blocks).
- `loss_grid` and `cbce_det_sums` restate csrc/loss.cu; `sum_grid` the `grid_cap(., 4)` grid of osvos_sum_f32.

tests/test_train_dispatch.py checks the restatements against the library's own queries and the compiled kernel set, and
tests/test_gpu_train_schedules.py runs the regimes found here against fp64 and checks which kernels actually ran."""
import re
from typing import NamedTuple

from conv_dispatch_ref import parse_kernel_name
from side_dispatch_ref import RED_SEGS, reduce_rows_scratch_floats, reduce_rows_depth   # noqa: F401 (re-exported)

FIRST_TILE_W, FIRST_TILE_H = 8, 16     # conv_first_tc_kernel output tile (kTileW x kTileH)
FIRST_STAGES = 3                       # conv_first_tc_kernel: A-tile ring stages (kFirstStages)
FW_PIX = 64                            # conv_first_wgrad_kernel: pixels per chunk (kFwPix)
FW_COPIES = 16                         # conv_first_wgrad_kernel: replicas of the atomic partial result (kFwCopies)
FW_SLOT = 64 * 27                      # floats of one partial dW
DGRAD_X = 128                          # conv_first_dgrad_kernel: pixels per block along x
TAIL_SEG_LO = (255, 63, 15, 7)         # tail_bwd2_kernel: low-res columns per segment, per scale (kSegLo)
TAIL_SUMS, TAIL_VALS = 15, 13          # OSVOS_TAIL_SUMS, and block partials per block (kTailVals)
GEN_SEG = 16                           # tail_general_bwd_kernel: low-res columns per segment (kGenSeg)
GEN_TAPS = 16 + 64 + 256 + 1024        # OSVOS_UPSAMPLING_TAPS
LOSS_THREADS = 256                     # kLossThreads
SUM_BLOCKS = 256                       # sum_f32_det_kernel's fixed grid (kSumBlocks)

# kernel name -> number of leading integer template arguments (parse_kernel_name)
TRAIN_KERNELS = {"conv_first_tc_kernel": 1, "conv_first_wgrad_kernel": 0, "tail_bwd2_kernel": 0,
                 "tail_general_bwd_kernel": 0, "cbce_fwd_kernel": 0}
# kernels that are not templates: matched by exact name
PLAIN_KERNELS = ("conv_first_dgrad_kernel", "tail_general_fwd_kernel", "upsampling_fold_kernel",
                 "upsampling_grads_finish_kernel", "cbce_bwd_kernel", "reduce_rows_segments_kernel",
                 "reduce_rows_final_kernel", "sum_f32_kernel", "sum_f32_det_kernel")
_PLAIN_RE = re.compile(r"\b(" + "|".join(PLAIN_KERNELS) + r")\(")

# every instantiation the library compiles (and the entry points below can reach)
COMPILED = {
    "conv_first_tc_kernel": {(planes, staged) for planes in (1, 2) for staged in (False, True)},
    "conv_first_wgrad_kernel": {(False,), (True,)},
    "tail_bwd2_kernel": {(loss, det) for loss in (False, True) for det in (False, True)},
    "tail_general_bwd_kernel": {(False,), (True,)},
    "cbce_fwd_kernel": {(False,), (True,)},
}


def _cdiv(a, b):
    return -(-a // b)


def parse_train_kernel_name(name):
    """(kernel, template arguments) of the template kernels above, (kernel, ()) of the plain ones, or None."""
    p = parse_kernel_name(name, TRAIN_KERNELS)
    if p is not None:
        return p
    m = _PLAIN_RE.search(name)
    return (m.group(1), ()) if m else None


def _ctas(total, grid):
    return tuple(tuple(range(b, total, grid)) for b in range(grid))


# ------------------------------------------------------------------------------------------------ conv1_1 forward
class FirstPlan(NamedTuple):
    inst: tuple                 # (PLANES, STAGED)
    tiles: int
    tiles_per_image: int
    grid: int
    cta_tiles: tuple


def conv_first_plan(n, h, w, fast, staged, sms):
    per_image = _cdiv(w, FIRST_TILE_W) * _cdiv(h, FIRST_TILE_H)
    tiles = n * per_image
    grid = min(tiles, sms)
    return FirstPlan((1 if fast else 2, staged), tiles, per_image, grid, _ctas(tiles, grid))


FIRST_REGIMES = ("one_wave", "waves")


def find_first_shape(regime, sms):
    """(n, h, w), h = 21 (two tile rows, the second of 5) and w % 8 == 5:
    - "one_wave": n = 2, the widest with tiles <= sms (one tile per CTA);
    - "waves": n = 5, the narrowest with tiles > 3 sms and tiles % sms != 0: CTAs run three or four tiles, so the
      3-stage ring wraps and its phase flips, and an image holds fewer tiles than there are CTAs, so each next-tile
      prefetch reads another image."""
    assert regime in FIRST_REGIMES
    n, h = (2, 21) if regime == "one_wave" else (5, 21)
    found = None
    for tx in range(1, 8 * sms):
        w = FIRST_TILE_W * tx - 3
        p = conv_first_plan(n, h, w, False, True, sms)
        if regime == "one_wave":
            if p.tiles > sms:
                return found
            found = (n, h, w)
        elif p.tiles > 3 * sms and p.tiles % sms != 0:
            return (n, h, w)
    return None


# ------------------------------------------------------------------------------------------------ conv1_1 backward
class FirstWgradPlan(NamedTuple):
    chunks_x: int
    tiles: int
    grid: int
    last_valid: int             # valid pixels of a row's last chunk
    block_tiles: tuple          # per block: its tiles, in order
    det_workspace_floats: int
    dgrad_grid: tuple           # (x blocks, h, n)


def first_wgrad_plan(n, h, w, sms):
    chunks_x = _cdiv(w, FW_PIX)
    tiles = n * h * chunks_x
    grid = min(max(tiles, 1), 4 * sms)
    ws = grid * FW_SLOT + reduce_rows_scratch_floats(grid, FW_SLOT)
    return FirstWgradPlan(chunks_x, tiles, grid, w - (chunks_x - 1) * FW_PIX, _ctas(tiles, grid), ws,
                          (_cdiv(w, DGRAD_X), h, n))


def first_bwd_workspace_bytes():
    """osvos_conv_first_bwd_workspace_bytes: the kFwCopies replicas and the arrival counter (padded to 4 floats)."""
    return (FW_COPIES * FW_SLOT + 4) * 4


FW_REGIMES = ("few", "one_wave", "waves")
FW_WIDTHS = {"narrow": 37, "64k": 256, "64k+1": 193}      # w < 64, a multiple of 64, 64 k + 1 (a last chunk of 1)


def find_fw_shape(regime, width, sms, n=2):
    """(n, h, w) of a conv1_1 backward with w = FW_WIDTHS[width]:
    - "few": the tallest with tiles < 16, so some of the kFwCopies replicas stay zero (and the grid is below the 64
      segments of the deterministic form's row reduction);
    - "one_wave": the tallest with tiles <= 4 sms: one tile per block, more blocks than 64 reduction segments;
    - "waves": the shortest with tiles > 8 sms and tiles % (4 sms) != 0: blocks walk two or three tiles, so the
      register prefetch of the next tile runs, and not every block the same number of times."""
    assert regime in FW_REGIMES
    w = FW_WIDTHS[width]
    found = None
    for h in range(1, 1 << 16):
        p = first_wgrad_plan(n, h, w, sms)
        if regime == "few":
            if p.tiles >= 16:
                return found
            found = (n, h, w)
        elif regime == "one_wave":
            if p.tiles > 4 * sms:
                return found
            found = (n, h, w)
        elif p.tiles > 8 * sms and p.tiles % (4 * sms) != 0:
            return (n, h, w)
    return None


def fw_cases():
    return [(r, wd) for r in FW_REGIMES for wd in FW_WIDTHS]


# ------------------------------------------------------------------------------------------------ tail backward
class TailBwdItem(NamedTuple):
    scale: int
    s: int
    seg: int                    # segment index within its row
    nout: int                   # low-res columns of the segment
    width: int                  # source columns the segment reads: nout s + s
    wpad: int
    rgroups: int


class TailBwdScale(NamedTuple):
    hk: int
    wk: int
    s: int
    top: int
    left: int
    seg_lo: int
    segs: int
    first_item: int


def tail_scales(h, w):
    """(hk, wk, s, top, left) of the four scales (fill_tail_scales / fill_tail_bwd_scales / fill_gen_scales)."""
    out, hk, wk = [], h, w
    for k in range(4):
        hk, wk = _cdiv(hk, 2), _cdiv(wk, 2)
        s = 2 << k
        out.append((hk, wk, s, ((hk + 1) * s - h) // 2, ((wk + 1) * s - w) // 2))
    return out


def tail_bwd_scales(n, h, w):
    res, items = [], 0
    for k, (hk, wk, s, top, left) in enumerate(tail_scales(h, w)):
        segs = _cdiv(wk, TAIL_SEG_LO[k])
        res.append(TailBwdScale(hk, wk, s, top, left, TAIL_SEG_LO[k], segs, items))
        items += n * hk * segs
    return res, items


def tail_bwd_row_items(w):
    """The items of one low-res row of every scale (the plan repeats them for every image and row)."""
    out = []
    for k, (_, wk, s, _, _) in enumerate(tail_scales(1, w)):
        seg_lo = TAIL_SEG_LO[k]
        for j in range(_cdiv(wk, seg_lo)):
            nout = min(seg_lo, wk - j * seg_lo)
            width = nout * s + s
            wpad = min(256, _cdiv(width, 32) * 32)
            out.append(TailBwdItem(k, s, j, nout, width, wpad, 256 // wpad))
    return out


def tail_bwd_depth(item):
    """fp32 roundings on the longest path of one dpq value: phase 1's FMAs per thread (ceil(2s / rgroups)), the
    row groups' adds into shared memory, phase 2's taps per lane, the shuffle levels and the final scaling."""
    fs = 2 * item.s
    lw = min(32, fs)
    return _cdiv(fs, item.rgroups) + item.rgroups + _cdiv(fs, lw) + (lw.bit_length() - 1) + 1


def tail_bwd_reachable():
    """Every (scale, rgroups) pair some segment width can give."""
    pairs = set()
    for k in range(4):
        s = 2 << k
        for nout in range(1, TAIL_SEG_LO[k] + 1):
            wpad = min(256, _cdiv(nout * s + s, 32) * 32)
            pairs.add((k, 256 // wpad))
    return pairs


IDLE_WPADS = (96, 160, 192, 224)       # 256 % wpad != 0: 256 - rgroups wpad threads sit out phase 1


def find_tail_bwd_widths(limit=4096):
    """A small set of widths whose rows together reach every reachable (scale, rgroups) pair, an idle-thread wpad, and
    full and short segments at scales 0 and 1: the narrowest width with two segments at scale 0, the last one short,
    then, narrowest first, every width that adds a pair not yet reached."""
    want = tail_bwd_reachable()
    first = next(w for w in range(1, limit) if _full_and_short(w))
    chosen, have = [first], {(it.scale, it.rgroups) for it in tail_bwd_row_items(first)}
    for w in range(1, limit):
        if have >= want:
            break
        new = {(it.scale, it.rgroups) for it in tail_bwd_row_items(w)} - have
        if new:
            chosen.append(w)
            have |= new
    return sorted(chosen) if have >= want else None


def _full_and_short(w):
    items = tail_bwd_row_items(w)
    for k in (0, 1):
        nouts = [it.nout for it in items if it.scale == k]
        if not (TAIL_SEG_LO[k] in nouts and min(nouts) < TAIL_SEG_LO[k]):
            return False
    return True


# ------------------------------------------------------------------------------------------------ general tail
def gen_fwd_blocks(n, h, sms):
    return min(n * h, 8 * sms)


def gen_fwd_sums(n, h, sms):
    """Doubles of osvos_tail_general_fwd_sums: the tail forward's layout, one row of partials per block."""
    return TAIL_SUMS + TAIL_VALS * gen_fwd_blocks(n, h, sms)


GEN_FWD_REGIMES = ("wide_rows", "strided")


def find_gen_fwd_shape(regime, sms):
    """(n, h, w) of a general-weights tail forward:
    - "wide_rows": n h <= 8 sms (one row per block) and w = 301 > 256, so each thread walks two pixels of its row;
    - "strided": n h > 8 sms with about 2.5 rows per block (blocks walk two or three rows), w = 37 odd."""
    assert regime in GEN_FWD_REGIMES
    if regime == "wide_rows":
        return 2, 19, 301
    n = 3
    return n, 5 * 8 * sms // (2 * n) + 1, 37


def gen_row_len(taps):
    return 17 * taps + 33


class GenBwdPlan(NamedTuple):
    segs: tuple                 # per scale
    nrows: tuple                # per scale: n hk segs partial rows
    row_len: tuple              # per scale
    row_offset: tuple           # per scale, floats; then the end of the rows
    items: int
    workspace_floats: int       # rows + the largest row reduction scratch


def gen_bwd_plan(n, h, w):
    segs, nrows, lens, offs, rows = [], [], [], [], 0
    for hk, wk, s, _, _ in tail_scales(h, w):
        sg = _cdiv(wk, GEN_SEG)
        nk = n * hk * sg
        segs.append(sg)
        nrows.append(nk)
        lens.append(gen_row_len(4 * s * s))
        offs.append(rows)
        rows += nk * lens[-1]
    scratch = max(reduce_rows_scratch_floats(r, c) for r, c in zip(nrows, lens))
    return GenBwdPlan(tuple(segs), tuple(nrows), tuple(lens), tuple(offs) + (rows,), sum(nrows), rows + scratch)


# ------------------------------------------------------------------------------------------------ loss and sums
def loss_grid(numel, sms):
    return min(max(_cdiv(numel // 4, LOSS_THREADS), 1), 8 * sms)


def cbce_det_sums(numel, sms):
    """Doubles of osvos_cbce_fwd_sums with OSVOS_FLAG_DETERMINISTIC: five leading values, then three per block."""
    return 5 + 3 * loss_grid(numel, sms) if numel > 0 else 0


def loss_vectors_per_thread(numel, sms):
    return _cdiv(numel // 4, loss_grid(numel, sms) * LOSS_THREADS) if numel >= 4 else 0


def grid_cap4(blocks, sms):
    return min(max(blocks, 1), 4 * sms)


def sum_grid(numel, sms):
    return grid_cap4(_cdiv(numel, 256), sms)


CBCE_REGIMES = ("tiny", "one_block", "capped")


def find_cbce_numels(regime, sms):
    """numel values of a regime:
    - "tiny": 1, 2, 3 (no vector at all: only the scalar tail);
    - "one_block": 4 k + {0, 1, 2, 3} with a single block of fewer than 256 vectors;
    - "capped": the grid capped at 8 sms with 2 - 3 vectors per thread, and numel % 4 = 1, 2, 3 and 0."""
    assert regime in CBCE_REGIMES
    if regime == "tiny":
        return [1, 2, 3]
    if regime == "one_block":
        return [4 * 97 + r for r in (1, 2, 3, 0)]
    base = 4 * (8 * sms * LOSS_THREADS * 2 + 8 * sms * LOSS_THREADS // 3)
    return [base + r for r in (1, 2, 3, 0)]

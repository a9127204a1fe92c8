"""Host restatement of the launch plans of the side-branch, unpool and tail kernels, and a search for small shapes that
reach each of their regimes at a given SM count.

- `side_conv_plan` restates `launch_side` (csrc/side_conv.cu) and the scale order of `osvos_side_folded_multi`: which
  `side_conv_kernel<PLANES, NCO>` runs, each scale's first tile, the grid and the tiles each CTA walks.
- `side_wgrad_plan` restates `side_wgrad_plan` (csrc/side_bwd_folded.cu): the blocks per scale of
  `side_folded_wgrad_kernel<DET>`, the chunks each block walks and the deterministic workspace.
- `unpool_plan` restates `launch_unpool` (csrc/bwd_kernels.cu): `unpool_add_mask_kernel<POOL, SIDE, DET>`'s grid,
  whether the folded weights go to shared memory, and the dynamic shared memory.
- `tail_fwd_blocks` restates the grid of `tail_fwd_kernel<DET>` (csrc/tail.cu).

tests/test_side_dispatch.py checks the restatements against the library's own queries and the compiled kernel set, and
tests/test_gpu_side_schedules.py runs every regime found here against fp64 and checks which kernel actually ran."""
from typing import NamedTuple

from conv_dispatch_ref import parse_kernel_name

SIDE_TILE_W, SIDE_TILE_H = 8, 10   # side_conv_kernel output tile (kSideTileW x kSideTileH)
SIDE_MAX_SCALES = 4
SW_SLAB, SW_CHUNK, SW_STAGES = 128, 28, 4    # side_folded_wgrad_kernel: channel slab, pixels per chunk, ring stages
RED_SEGS = 64                                # osvos_reduce_rows: row segments (kRedSegs)
TAIL_SUMS, TAIL_VALS = 15, 13                # tail_fwd_kernel: sums, and block partials per block under DET

# kernel name -> number of leading integer template arguments (parse_kernel_name)
SIDE_KERNELS = {"side_conv_kernel": 2, "unpool_add_mask_kernel": 0, "side_folded_wgrad_kernel": 0,
                "tail_fwd_kernel": 0}


def _cdiv(a, b):
    return -(-a // b)


def parse_side_kernel_name(name):
    """(kernel, template arguments) of the four kernel templates planned here, or None."""
    return parse_kernel_name(name, SIDE_KERNELS)


# every instantiation the library compiles (and the entry points below can reach)
COMPILED = {
    "side_conv_kernel": {(planes, nco) for planes in (1, 2) for nco in (2, 16)},
    "unpool_add_mask_kernel": {(pool, side, det) for pool in (False, True) for side in (False, True)
                               for det in (False, True)},
    "side_folded_wgrad_kernel": {(False,), (True,)},
    "tail_fwd_kernel": {(False,), (True,)},
}


# ------------------------------------------------------------------------------------------------ side convolution
class SidePlan(NamedTuple):
    inst: tuple                 # (PLANES, NCO)
    scales: tuple               # the scales in launch order: (n, h, w, cin, cout)
    tile_begin: tuple           # first tile of each scale (launch order)
    total_tiles: int
    grid: int
    cta_tiles: tuple            # per CTA: the tiles it runs, in order

    def scale_of(self, tile):
        k = 0
        while k + 1 < len(self.tile_begin) and tile >= self.tile_begin[k + 1]:
            k += 1
        return k


def side_tiles(h, w, n):
    return _cdiv(w, SIDE_TILE_W) * _cdiv(h, SIDE_TILE_H) * n


def side_conv_plan(scales, fast, sms):
    """``scales``: [(n, h, w, cin, cout)]: one entry for an osvos_conv3x3 call with cout 2 or 16, several (cout 2) for
    osvos_side_folded_multi, which launches them deepest (largest cin) first, ties in the given order."""
    assert 1 <= len(scales) <= SIDE_MAX_SCALES
    nco = scales[0][4]
    assert nco in (2, 16) and all(s[4] == nco for s in scales) and (nco == 2 or len(scales) == 1)
    order = sorted(scales, key=lambda s: -s[3]) if len(scales) > 1 else list(scales)   # stable: ties keep their order
    begin, total = [], 0
    for n, h, w, cin, _ in order:
        assert cin % 64 == 0
        begin.append(total)
        total += side_tiles(h, w, n)
    grid = min(total, sms)
    ctas = tuple(tuple(range(b, total, grid)) for b in range(grid))
    return SidePlan((1 if fast else 2, nco), tuple(order), tuple(begin), total, grid, ctas)


SIDE_REGIMES = ("one_wave", "waves")
SIDE_MULTI_CINS = {2: (256, 128), 3: (512, 256, 128), 4: (512, 512, 256, 128)}


def _ragged(h, w):
    return h % SIDE_TILE_H != 0 and w % SIDE_TILE_W != 0


def find_side_shape(regime, sms, n=2, h=17):
    """(n, h, w) of one side convolution, tiles ragged in both directions (h = 17: two tile rows, the second of 7):
    - "one_wave": the widest with tiles <= sms (one tile per CTA, every CTA busy at once);
    - "waves": the narrowest with tiles > 2 sms and tiles % sms != 0, so every CTA runs two or three tiles and CTAs
      run both odd and even tile counts (the NCO = 2 exchange buffer of parity 0 is used twice by some CTAs)."""
    assert regime in SIDE_REGIMES
    found = None
    for tx in range(1, 4 * sms):
        w = SIDE_TILE_W * tx - 3
        tiles = side_tiles(h, w, n)
        if regime == "one_wave":
            if tiles > sms:
                return found
            found = (n, h, w)
        elif tiles > 2 * sms and tiles % sms != 0:
            return (n, h, w)
    return None


def multi_scale_shapes(h, w, count):
    """The scales of a network-like multi-scale launch: deepest first, each half the size of the next."""
    cins = SIDE_MULTI_CINS[count]
    return [(-(-h // 2 ** (count - 1 - k)), -(-w // 2 ** (count - 1 - k)), cin) for k, cin in enumerate(cins)]


def find_side_multi_shape(count, sms, n=2, h=45):
    """(n, h, w) of the shallowest scale of a ``count``-scale launch (multi_scale_shapes) with every scale ragged, more
    tiles than CTAs with total % sms != 0, and fewer tiles in the first (deepest) scale than CTAs, so that CTA 0's walk
    goes from the first scale into a later one: the chunk count changes between consecutive tiles of one ring."""
    for w in range(9, 4096):
        shapes = multi_scale_shapes(h, w, count)
        if not all(_ragged(hh, ww) for hh, ww, _ in shapes):
            continue
        plan = side_conv_plan([(n, hh, ww, cin, 2) for hh, ww, cin in shapes], False, sms)
        first = plan.tile_begin[1]
        if plan.total_tiles > sms and plan.total_tiles % sms != 0 and first < sms:
            return n, h, w
    return None


def crossing_ctas(plan):
    """CTAs whose tiles lie in more than one scale."""
    return [b for b, ts in enumerate(plan.cta_tiles) if len({plan.scale_of(t) for t in ts}) > 1]


# ------------------------------------------------------------------------------------------------ folded side G
class SwScalePlan(NamedTuple):
    chunks: int                 # n * h * ceil(w / 28)
    slabs: int                  # c / 128
    blocks_per_slab: int        # blocks of one slab: block k walks chunks k, k + blocks_per_slab, ...
    block_begin: int
    chunks_per_block: tuple     # per block of a slab (max first)


class SwPlan(NamedTuple):
    scales: tuple
    total_blocks: int
    rows_floats: int            # DET: partial rows of every scale
    workspace_floats: int       # DET: + the row reduction's scratch


def sw_row_pitch(c):
    return (18 * c + 2 + 3) // 4 * 4


def reduce_rows_scratch_floats(nrows, ncols):
    return min(RED_SEGS, nrows) * ncols


def reduce_rows_depth(nrows):
    """Additions on the longest path of osvos_reduce_rows over ``nrows`` rows into an accumulator: eight row lanes per
    segment, the lanes in order, the segments in order, then the add into the output."""
    seg = _cdiv(nrows, RED_SEGS)
    segs = _cdiv(nrows, seg)
    return _cdiv(seg, 8) + 7 + segs


def side_wgrad_plan(items, sms):
    """``items``: [(n, h, w, c)] in launch order (osvos_side_folded_wgrad_multi keeps the caller's order)."""
    assert 1 <= len(items) <= 4
    work = []
    for n, h, w, c in items:
        assert c >= SW_SLAB and c % SW_SLAB == 0
        work.append(n * h * _cdiv(w, SW_CHUNK) * (c // SW_SLAB))
    total_work = sum(work)
    budget = 2 * sms
    scales, begin, rows, scratch = [], 0, 0, 0
    for (n, h, w, c), wk in zip(items, work):
        slabs = c // SW_SLAB
        chunks = wk // slabs
        b = (budget * wk + total_work // 2) // total_work // slabs
        b = min(max(b, 1), chunks)
        cpb = tuple(_cdiv(chunks - k, b) for k in range(b))
        scales.append(SwScalePlan(chunks, slabs, b, begin, cpb))
        begin += b * slabs
        rows += b * sw_row_pitch(c)
        scratch = max(scratch, reduce_rows_scratch_floats(b, 18 * c + 2))
    return SwPlan(tuple(scales), begin, rows, rows + scratch)


SW_REGIMES = ("one_chunk", "ring_wraps", "clamped", "narrow")


def _sw_ok(regime, items, plan):
    s = plan.scales
    if regime == "one_chunk":
        return s[0].chunks_per_block[0] == 1 and s[0].blocks_per_slab > 1
    if regime == "ring_wraps":
        return s[0].chunks_per_block[0] > 2 * SW_STAGES and s[0].chunks % s[0].blocks_per_slab != 0
    if regime == "clamped":
        return any(sc.blocks_per_slab == 1 for sc in s) and any(sc.blocks_per_slab > 1 for sc in s)
    n, h, w, _ = items[0]
    return w < SW_CHUNK and s[0].chunks_per_block[0] > 1


def sw_items(regime, k):
    """The item list of ``regime`` for search index k (k = 1, 2, ...); n >= 2 and odd widths throughout."""
    if regime == "one_chunk":        # one 128-channel slab of 2 x 9 x (28 k + 23): 18 (k + 1) chunks
        return [(2, 9, SW_CHUNK * k + 23, 128)]
    if regime == "ring_wraps":       # 2 x (2 k + 1) x 201 at 256 channels: 8 chunks per image row
        return [(2, 2 * k + 1, 201, 256)]
    if regime == "clamped":          # a large 128-channel scale and two small 512-channel ones: 1 block per slab
        return [(2, 3 * k, 139, 128), (2, 3, 5, 512), (2, 1, 3, 512)]
    return [(3, 2 * k + 1, 19, 128)]  # narrow: w = 19, each chunk's box runs 9 pixels into the next row / image


def find_sw_items(regime, sms):
    """The smallest item list of ``regime`` that reaches it on ``sms`` SMs:
    - "one_chunk": every block of the slab gets exactly one chunk, and there are several blocks;
    - "ring_wraps": more than 2 SW_STAGES chunks per block (the four-stage ring wraps twice: its phase flips and flips
      back), and the block count
      does not divide the chunk count (blocks of one slab walk different numbers of chunks);
    - "clamped": a multi-scale launch in which one scale gets one block per slab (its share of the budget rounds to 0);
    - "narrow": w < 28 with n = 3: each chunk is a partial row whose 28-pixel TMA box runs into the next row, the next
      image, or (for the last chunk) past the end of the tensor; several chunks per block."""
    assert regime in SW_REGIMES
    for k in range(1, 4096):
        items = sw_items(regime, k)
        if _sw_ok(regime, items, side_wgrad_plan(items, sms)):
            return items
    return None


# ------------------------------------------------------------------------------------------------ unpool
class UnpoolPlan(NamedTuple):
    inst: tuple                 # (POOL, SIDE, DET)
    tiles: int
    grid: int
    wf_in_smem: bool
    smem: int                   # dynamic shared memory, bytes
    ppb: int                    # (pooled) pixels per block iteration


def unpool_plan(n, h, w, c, pool, side, det, sms):
    assert c % 8 == 0 and 256 % (c // 8) == 0
    oh, ow = (_cdiv(h, 2), _cdiv(w, 2)) if pool else (h, w)
    ppb = 256 // (c // 8)
    tiles = n * oh * _cdiv(ow, ppb)
    grid = max(1, min(tiles, sms * (2 if side else 4)))
    wf = bool(side and tiles >= 4 * grid)
    smem = c * 4 * (19 if wf else 1) + (256 * 8 * 4 if det else 0)
    return UnpoolPlan((pool, side, det), tiles, grid, wf, smem, ppb)


UNPOOL_CHANNELS = (64, 128, 256, 512)


def unpool_targets():
    """(POOL, SIDE, DET, wf_in_smem) of every test target: all eight instantiations, the SIDE ones with the folded
    weights in global and in shared memory."""
    return [(pool, side, det, wf) for pool in (False, True) for side in (False, True) for det in (False, True)
            for wf in ((False, True) if side else (False,))]


def find_unpool_shape(pool, side, det, wf, c, sms, n=2):
    """(n, h, w) with odd h and w and more tiles than CTAs, the folded weights in shared memory iff ``wf``: the smallest
    such h.  w gives two tile columns, a full block iteration and one of a single (pooled) pixel (with POOL, w = 2 ppb
    + 1, so the last window column and row have one element: ceil-mode windows of 1, 2 and 4 elements)."""
    ppb = 256 // (c // 8)
    w = (2 * ppb + 1) if pool else (ppb + 5)          # two tile columns, the second with 1 (pooled) pixel / 5 pixels
    if not pool and w % 2 == 0:
        w += 1
    for h in range(3, 1 << 16, 2):
        p = unpool_plan(n, h, w, c, pool, side, det, sms)
        if p.tiles > p.grid and p.wf_in_smem == wf:
            return n, h, w
    return None


# ------------------------------------------------------------------------------------------------ tail forward
def tail_fwd_blocks(n, h, sms):
    return min(n * h, 8 * sms)


def tail_det_sums(n, h, sms):
    """Doubles of the deterministic form's sums buffer (osvos_tail_fwd_deterministic_sums)."""
    return TAIL_SUMS + TAIL_VALS * tail_fwd_blocks(n, h, sms)


def find_tail_shape(sms, n=3, w=37):
    """(n, h, w) with about 2.5 rows per block (n h > 8 sms: blocks walk two or three rows), w odd so that the rows
    start at every offset 0 - 3 of a 16-byte group."""
    h = 5 * 8 * sms // (2 * n) + 1
    return n, h, w

"""Host restatement of the two convolution dispatchers that plan from the SM count, and a search for small shapes that
reach each of their schedules.

- `halo_plan` restates `conv3x3_halo_dispatch` and `launch_halo` (csrc/conv3x3_halo.cu): which instantiation of
  `conv3x3_halo_kernel<BLOCK_N, PLANES, SPLIT, LEAN, PINGPONG, DET>` a forward / data-gradient launch runs.
- `wgrad_plan` restates `plan_wgrad<128>` (csrc/wgrad_tc.cu): the item geometry and pixel-range split count of a weight
  gradient.

tests/test_conv_dispatch.py checks the restatements against the library (split counts, the compiled kernel set), and
tests/test_gpu_conv_schedules.py runs every schedule found here against fp64 and checks which kernel actually ran."""
import re
from typing import NamedTuple

TILE_W, TILE_H = 8, 16          # halo kernel output tile (kTileW x kTileH)
PATCH_W, PATCH_H = 8, 8         # weight-gradient K block (kWgPatchW x kWgPatchH)
WGRAD_NOMINAL_SMS = 132         # the deterministic weight gradient plans for this SM count (kWgNominalSms)


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ halo convolution
def halo_plan(n, h, w, cin, cout, fast, lean, det, sms):
    """-> ((BLOCK_N, PLANES, SPLIT, LEAN, PINGPONG, DET), total_tiles) of one osvos_conv3x3 launch with cout 64 or a
    multiple of 128.  ``lean``: the launch asks for nothing but bias / ReLU / act output / fused pool (no ReLU mask, no
    column sum, no fp32 output); ``det``: a column sum under OSVOS_FLAG_DETERMINISTIC."""
    assert cout == 64 or (cout > 0 and cout % 128 == 0), cout
    assert cin >= 64 and cin % 64 == 0, cin
    assert not (lean and det), "a column sum is not a lean launch"
    lean = lean and not fast
    m_tiles = _cdiv(w, TILE_W) * _cdiv(h, TILE_H) * n
    tiles128 = m_tiles * (cout // 128)
    waves128 = _cdiv(tiles128, sms)
    waves256 = _cdiv(m_tiles * (cout // 256), sms)
    if cout == 64 or (waves128 == 1 and tiles128 * 5 <= sms * 3):      # few tiles: N = 64
        block_n = 64
    elif fast and cout % 256 == 0 and waves256 * 1100 < waves128 * 700:  # fast mode only
        block_n = 256
    else:
        block_n = 128
    planes = 1 if fast else 2
    split = planes == 2 and block_n <= 128
    total = m_tiles * (cout // block_n)
    pingpong = block_n in (64, 128) and total > 2 * sms
    if pingpong:
        split = split and block_n == 64     # N = 128 ping-pong: three plain passes, no split accumulator
    return (block_n, planes, split, lean, pingpong, det), total


def _halo(block_n, planes, split, lean, pingpong, det):
    return (block_n, planes, split, lean, pingpong, det)


# every instantiation conv3x3_halo_dispatch can pick: (BLOCK_N, PLANES, SPLIT, LEAN, PINGPONG, DET)
REACHABLE_HALO = frozenset(
    # N = 64: lean exact, general exact, fast; cooperative and ping-pong
    [_halo(64, 2, True, True, pp, False) for pp in (False, True)]
    + [_halo(64, 2, True, False, pp, det) for pp in (False, True) for det in (False, True)]
    + [_halo(64, 1, False, False, pp, det) for pp in (False, True) for det in (False, True)]
    # N = 128: exact cooperative (split accumulator), exact ping-pong (three passes), fast
    + [_halo(128, 2, True, True, False, False), _halo(128, 2, False, True, True, False)]
    + [_halo(128, 2, not pp, False, pp, det) for pp in (False, True) for det in (False, True)]
    + [_halo(128, 1, False, False, pp, det) for pp in (False, True) for det in (False, True)]
    # N = 256: fast mode only, always cooperative
    + [_halo(256, 1, False, False, False, det) for det in (False, True)])


class HaloShape(NamedTuple):
    n: int
    h: int
    w: int
    cin: int
    cout: int
    fast: bool
    lean: bool          # the launch uses only the lean feature set
    det: bool           # deterministic column sum
    total_tiles: int


def _candidate_couts(target):
    block_n, _, _, _, pingpong, _ = target
    if block_n == 64:
        return (64,) if pingpong else (64, 128, 256)
    if block_n == 128:
        return (128, 256, 384, 512)
    return (256, 512)


def find_halo_shape(target, sms, cin=64, couts=None):
    """The cheapest (n, h, w, cin, cout) plus flags whose launch selects ``target`` on ``sms`` SMs, or None.

    Shapes are 3 x 29 x (8 tx - 3), that is 3 images of 2 x tx tiles: the last tile row has 13 valid rows (both m64
    halves hold valid pixels, the second only partly) and the last tile column 5 valid columns, so h % 16 != 0 and
    w % 8 != 0; h and w are odd, so the fused pool has a partial window at both edges.  Every target gets more tiles
    than SMs and total_tiles % sms != 0 (the grid is one CTA per SM), so some CTAs run a second tile - the producer
    prefetches the next tile's halo, the consumers take ring stages and phases from the tiles before, reset their
    accumulators and run a second epilogue - and the CTAs' tile counts differ: under ping-pong some CTAs take an odd
    number of tiles and some an even number, and both consumer warpgroups end a CTA's sequence.  The shapes found hold
    fewer tiles per image than there are CTAs, so a CTA's second tile lies in another image than its first
    (tests/test_conv_dispatch.py checks both).  Cost is the MAC count; ties go to the first cout in ``couts``."""
    _, planes, _, lean, _, det = target
    fast = planes == 1
    best = None
    for cout in couts or _candidate_couts(target):
        for m in range(6, 4 * sms + 1, 6):      # pixel tiles; the plan depends on (m, cout) only
            got, total = halo_plan(m, TILE_H, TILE_W, cin, cout, fast, lean, det, sms)
            if got != target:
                continue
            if total <= sms or total % sms == 0:
                continue
            shape = HaloShape(3, 2 * TILE_H - 3, 8 * (m // 6) - 3, cin, cout, fast, lean, det, total)
            assert halo_plan(shape.n, shape.h, shape.w, cin, cout, fast, lean, det, sms) == (target, total)
            cost = m * cin * cout
            if best is None or cost < best[0]:
                best = (cost, shape)
            break                                # larger m at this cout only costs more
    return None if best is None else best[1]


def halo_case_args(target):
    """Channel choices of the tested shape of ``target``: ping-pong and N = 128 schedules take cin = 192 (three K chunks,
    an odd number, so the halo ring's phase differs between consecutive tiles), the others two K chunks; the exact
    N = 128 schedules take cout = 384 (three N blocks), which the ABI accepts and the network never uses."""
    block_n, planes, _, _, pingpong, _ = target
    cin = 192 if (pingpong or block_n == 128) else 128
    couts = (384,) if (block_n == 128 and planes == 2) else None
    return {"cin": cin, "couts": couts}


def halo_cases(sms):
    """(target, shape) for every reachable instantiation on ``sms`` SMs, with the channels of halo_case_args."""
    return [(t, find_halo_shape(t, sms, **halo_case_args(t))) for t in sorted(REACHABLE_HALO)]


# ------------------------------------------------------------------------------------------------ weight gradient
class WgradPlan(NamedTuple):
    mode: str               # "tap_rows", "tap_pairs" or "nine_taps"
    tap_items: int
    m_blocks: int
    n_blocks: int
    patches_total: int
    patches_per_split: int
    splits: int
    total_items: int


def wgrad_plan(n, h, w, dz_channels, cin, sms):
    """plan_wgrad<128>(n, h, w, cp = dz_channels, cq = cin, sms).  Raises ValueError where it returns
    OSVOS_ERR_UNSUPPORTED (dz_channels neither 64 nor a multiple of 128)."""
    cp, cq = dz_channels, cin
    if _cdiv(cp, 128) * 128 != cp and cp != 64:
        raise ValueError(f"dz_channels = {cp} is not supported")
    m_blocks = _cdiv(cp, 128)
    tap_rows = cq == 64 and cp == 64
    tap_pairs = cq == 64 and not tap_rows
    tap_items = 3 if tap_rows else 5 if tap_pairs else 9
    n_blocks = 1 if (tap_rows or tap_pairs) else cq // 128
    patches_total = _cdiv(w, PATCH_W) * _cdiv(h, PATCH_H) * n
    tiles = m_blocks * n_blocks * tap_items
    max_splits = (patches_total + 3) // 4
    splits, best = 1, None
    s_hi = 4 * sms // tiles + 1
    for s in range(1, min(s_hi, max_splits) + 1):
        pps = _cdiv(patches_total, s)
        se = _cdiv(patches_total, pps)
        rounds = _cdiv(tiles * se, sms)
        cost = rounds * (pps + 2) + 4
        if best is None or cost < best:
            best, splits = cost, s
    pps = _cdiv(patches_total, splits)
    splits = _cdiv(patches_total, pps)
    mode = "tap_rows" if tap_rows else "tap_pairs" if tap_pairs else "nine_taps"
    return WgradPlan(mode, tap_items, m_blocks, n_blocks, patches_total, pps, splits, tiles * splits)


# mode -> (cin, dz_channels): tap pairs with two m blocks, nine taps with two m blocks and two n blocks
WGRAD_MODES = {"tap_rows": (64, 64), "tap_pairs": (64, 256), "nine_taps": (256, 256)}


WGRAD_REGIMES = ("one_split", "splits", "many_items")


def find_wgrad_shape(mode, regime, plan_sms, grid_sms=None, channels=None):
    """(n, h, w) with ragged patches (h % 8 != 0, w % 8 != 0) and n = 2 or 3, so a split's pixel range crosses images,
    for a plan on ``plan_sms`` SMs launched on ``grid_sms`` (default: the same; the grid is one CTA per SM):
    - "one_split": the largest (up to 64 patches) whose plan has one pixel-range split;
    - "splits": the smallest with several splits and a short last one (patches_total % patches_per_split != 0);
    - "many_items": the smallest with more items than CTAs (so CTAs run a second item through the persistent loop)
      and more than 6 patches per split (so both the fast form's 6-stage and the exact form's 3-stage operand rings
      wrap, and flip phase, within an item).  The split rule keeps the item count near a whole number of rounds, so
      this needs more (m block, n block, tap) tiles than SMs: the nine-tap mode at cin = 512, dz_channels = 640 has 180.
    ``channels``: (cin, dz_channels) instead of the mode's WGRAD_MODES entry."""
    assert regime in WGRAD_REGIMES, regime
    grid_sms = grid_sms or plan_sms
    cin, dz = channels or WGRAD_MODES[mode]
    found = None
    for patches in range(2, 4096):
        n = 3 if patches % 3 == 0 else 2 if patches % 2 == 0 else 0
        if n == 0:
            continue
        r = patches // n
        py = 2 if r % 2 == 0 else 1
        px = r // py
        h, w = 8 * py - 3, 8 * px - 1
        plan = wgrad_plan(n, h, w, dz, cin, plan_sms)
        assert plan.mode == mode and plan.patches_total == patches
        short_last = plan.splits > 1 and plan.patches_total % plan.patches_per_split != 0
        if regime == "splits" and short_last:
            return n, h, w
        if regime == "many_items" and plan.total_items > grid_sms and plan.patches_per_split > 6:
            return n, h, w
        if regime == "one_split":
            if plan.splits == 1:
                found = (n, h, w)
            if patches >= 64:
                break
    return found


# (mode, regime, (cin, dz_channels)) under test: every mode in the first two regimes, and the nine-tap mode with 5 m
# blocks x 4 n blocks of 128 (180 tiles per split) with many items
WGRAD_SHAPES = [(mode, regime, WGRAD_MODES[mode]) for mode in WGRAD_MODES for regime in WGRAD_REGIMES[:2]] + \
    [("nine_taps", "many_items", (512, 640))]


def wgrad_cases(sms):
    """(id, mode, regime, fast, det, n, h, w, cin, dz_channels, plan) for every WGRAD_SHAPES entry x {exact, fast} x
    {default, deterministic} on a device of ``sms`` SMs; the deterministic form plans at WGRAD_NOMINAL_SMS."""
    cases = []
    for mode, regime, (cin, dz) in WGRAD_SHAPES:
        for det in (False, True):
            plan_sms = WGRAD_NOMINAL_SMS if det else sms
            n, h, w = find_wgrad_shape(mode, regime, plan_sms, sms, (cin, dz))
            plan = wgrad_plan(n, h, w, dz, cin, plan_sms)
            for fast in (False, True):
                cid = f"{mode}-{regime}-{'fast' if fast else 'exact'}-{'det' if det else 'atomic'}"
                cases.append((cid, mode, regime, fast, det, n, h, w, cin, dz, plan))
    return cases


# ------------------------------------------------------------------------------------------------ kernel names
# kernel name -> number of leading integer template arguments (the rest are bool)
CONV_KERNELS = {"conv3x3_halo_kernel": 2, "wgrad_tc_kernel": 2}


def _template_value(tok):
    tok = re.sub(r"^\((?:int|bool|unsigned int|unsigned)\)", "", tok.strip())
    if tok in ("true", "false"):
        return tok == "true"
    return int(tok.rstrip("uU"))


def parse_kernel_name(name, kernels=None):
    """Demangled kernel name -> (kernel, template-argument tuple), or None for kernels not in ``kernels`` ({name: number
    of leading integer arguments}, default CONV_KERNELS).  Accepts both demangled spellings: ``<128, 2, true, false,
    ...>`` and ``<(int)128, (int)2, (bool)1, ...>``.  The leading integer arguments come back as int, the boolean
    positions after them as bool."""
    kernels = CONV_KERNELS if kernels is None else kernels
    m = re.search(r"\b(" + "|".join(map(re.escape, kernels)) + r")<([^<>]*)>", name)
    if m is None:
        return None
    n_int = kernels[m.group(1)]
    vals = [_template_value(t) for t in m.group(2).split(",")]
    vals = vals[:n_int] + [bool(v) for v in vals[n_int:]]
    return m.group(1), tuple(vals)

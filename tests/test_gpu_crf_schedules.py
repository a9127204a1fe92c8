"""The dense CRF (csrc/crf.cu, DESIGN.md §29) at every mean-field iteration and every launch regime, against fp64 of what
each iteration read.  tests/test_gpu_crf.py holds the whole T-iteration result to the restatement with an error carried
through T iterations, which at the defaults (T = 5, L = 6.5) is about 0.7 logits; here each iteration gets its own bound.

Per-iteration check.  The kernel runs at T = t - 1 and at T = t on the same inputs (T = 0 is z itself), each call through
the C entry point with a workspace of the test's own, so the label probabilities Q^(t-1) that iteration t read (the
workspace's q region, restated by _layout) can be read back after the T = t call.  u = 2^-24 is the unit of one fp32
rounding, m the largest vertex occupancy, n = min(2 ceil(3θγ) + 1, max(H, W)) the most Gaussian taps inside the frame
along a row or a column, M = max|z| + w_α + w_γ.
  - "iteration": r^(t) against tests/crf_ref.mean_field_step of that Q in fp64.  One iteration's own error, as in
    tests/test_gpu_crf.py: e_B = 2(ceil(m/256) + 9 + 18 + 7 + K + 6)u + 2u for the bilateral message (splat, 6 blurs,
    slice, the division by F(1)), e_S = 2(3n + 8)u for the Gaussian, and e_a = w_α e_B + w_γ e_S + 4uM for the update;
    r = a_k - a_0 doubles a's error, and the check allows twice that for second-order terms: |Δr| <= 4 e_a.  At the
    defaults and 480x854 that is 6e-4 (0.7 for T = 5 iterations at once); each bound is asserted below 0.01, and a
    message wrong by a percent moves r by far more.
  - "softmax": that Q against Q̂ = softmax(0, r^(t-1)) in fp64, r^(t-1) the T = t - 1 call's output.  The kernel's Q
    comes from its a of iteration t - 1, formed by crf_update_kernel<iterate>, where the T = t - 1 call's r came from
    <last>: the same source, but the compiler may contract the column pass and the update differently, each form within
    w_γ e_S + 4uM of the exact value, so the two differ by at most c = 2(w_γ e_S + 4uM) per label, and r = a_k - a_0
    was rounded once: Δr <= u max|r^(t-1)| + 2c (0 at t = 1, where both read z).  Q as a function of r has a Jacobian
    of ∞-norm max 2Q(1 - Q) <= ½, and the fp32 softmax errs by (K + 6)u: |ΔQ| <= 2(½ Δr + (K + 6)u).
Together the two hold r^(t) to mean_field_step(Q̂) within 4 e_a + (w_α + w_γ) |ΔQ|.
Regimes.  The pixel loops (elevate, slice, Gaussian rows, update) and the vertex loops (neighbours, blur) are grid-stride
loops over at most 4096 x 256 = 2^20 threads, and the splat runs one block per vertex over kSplatBlocks = 2048 blocks:
3 x 480x854 frames put 1.2 M pixels through the pixel loops; a noisy 480x854 frame at θα = 2, θβ = 1 has 2.46 M vertices
(at most 2 entries each); the default 480x854 lattice has 38 k vertices with up to 16,663 entries.
Exact checks.  Vertex counts equal the restatement's; N frames in one call equal N calls of one frame, bit for bit (a
stable sort and each segment's fixed thread order); a workspace of 0xFF bytes gives the same bits as one of zeros; with
w_α = w_γ = 0 the maps come back bit for bit.  torch.profiler confirms each call's kernels and launch counts.
At module end each family reports its largest share of its bound."""
import dataclasses
import gc
import math
import re
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import crf_ref as ref
from test_gpu_conv_schedules import KernelsRan
from test_gpu_crf import _maps, _scene

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
MEASURED = {}
BLIND = []          # profiler windows that lost crf kernel records: ((T, K, N), {kernel: records missing})


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report_measured():
    yield
    for family, v in sorted(MEASURED.items()):
        print(f"\n{family}: largest share of its bound {max(v):.3f} ({len(v)} checks)")
    if BLIND:
        print(f"\nprofiler windows that lost device records (kernels not confirmed): {len(BLIND)}: {BLIND}")


@pytest.fixture(autouse=True)
def _release():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _f32(v):
    return float(np.float32(v))


def _crf(**kw):
    from osvos_pytorch_b200 import ops
    return ops.CRF(**kw)


def _layout(n, k, h, w):
    """The workspace's region offsets, as crf_layout lays them out (each region 256-byte aligned, in this order)."""
    pixels = n * h * w
    cap, ch = ref.D1 * pixels, k + 1
    sizes = [("counts", 4 * (n + 1)), ("fstart", 4 * n), ("keys_in", 8 * cap), ("keys_out", 8 * cap),
             ("vals_in", 4 * cap), ("vals_out", 4 * cap), ("wts", 4 * cap), ("vid", 4 * cap), ("ukey", 8 * cap),
             ("seg", 4 * (cap + 1)), ("pv", 4 * cap), ("nbr", 4 * 2 * ref.D1 * cap), ("val0", 4 * ch * cap),
             ("val1", 4 * ch * cap), ("norm", 4 * pixels), ("q", 4 * ch * pixels), ("bmsg", 4 * ch * pixels),
             ("a", 4 * ch * pixels), ("t", 4 * ch * pixels), ("taps", 4 * max(h, w)), ("cub", 0)]
    off, o = {}, 0
    for name, nbytes in sizes:
        off[name] = o
        o = (o + nbytes + 255) & ~255
    return off


def _run(frames, z, crf):
    """osvos_dense_crf of frames uint8 [N,H,W,3] and maps [K,N,H,W] -> (refined maps [K,N,H,W], vertices per frame,
    the label probabilities [K+1,N,H,W] the last iteration read), all from the device, as fp64 / ints."""
    from osvos_pytorch_b200 import _native as nat
    k, n, h, w = z.shape
    nbytes = nat.load().osvos_dense_crf_workspace_bytes(n, k, h, w)
    off = _layout(n, k, h, w)
    assert 0 < off["cub"] <= nbytes
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = _native_crf(torch.from_numpy(frames).cuda(), [torch.from_numpy(z[i]).cuda() for i in range(k)], crf, ws,
                      torch.empty((k, n, h, w), device="cuda"))
    q = ws[off["q"]:off["q"] + 4 * (k + 1) * n * h * w].view(torch.float32).view(k + 1, n, h, w)
    return (out.double().cpu().numpy(), ws[:4 * n].view(torch.int32).cpu().tolist(), q.double().cpu().numpy())


def _lattice(frames, crf):
    return ref.Lattice(frames, crf.bilateral_xy, crf.bilateral_rgb, weights_f32=True)


def _bounds(lat, z, prev, w_a, w_g, theta_g, k, first):
    """(the bound of r^(t) against mean_field_step of the Q the kernel read, the bound of that Q against Q̂)."""
    m = int(lat.occupancy.max())
    h, w = z.shape[-2:]
    taps = min(2 * math.ceil(3 * theta_g) + 1, max(h, w))            # the in-frame taps of a row or a column
    mag = float(np.abs(z).max()) + w_a + w_g
    e_b = 2 * (-(-m // 256) + 9 + 18 + 7 + k + 6) * U + 2 * U
    e_s = 2 * (3 * taps + 8) * U
    e_a = w_a * e_b + w_g * e_s + 4 * U * mag
    d_r = 0.0 if first else U * float(np.abs(prev).max()) + 2 * 2 * (w_g * e_s + 4 * U * mag)
    return 2 * 2 * e_a, 2 * (d_r / 2 + (k + 6) * U)


def check(family, got, want, bound, what):
    assert not np.isnan(got).any(), (what, "NaN in the output")
    err = float(np.abs(got - want).max())
    share = err / bound
    MEASURED.setdefault(family, []).append(share)
    assert share <= 1.0, (what, err, bound)
    return share


def chain(family, frames, z, crf, lat=None):
    """Iterations 1..crf.iterations: each iteration's result against mean_field_step of the Q it read, that Q against
    softmax(0, r) of the previous call's result, and the vertex counts of every call.  ``family`` names the iteration
    checks in the report."""
    lat = _lattice(frames, crf) if lat is None else lat
    k = z.shape[0]
    w_a, w_g = _f32(crf.bilateral_weight), _f32(crf.gaussian_weight)
    zz = z.astype(np.float64)
    zero = np.zeros((1,) + zz.shape[1:])
    a0 = np.concatenate([zero, zz])
    norm = lat.filter(np.ones((lat.pixels, 1)))[:, 0]
    prev = zz
    for t in range(1, crf.iterations + 1):
        got, verts, q = _run(frames, z, dataclasses.replace(crf, iterations=t))
        assert verts == lat.per_frame.tolist()
        b_r, b_q = _bounds(lat, zz, prev, w_a, w_g, crf.gaussian_xy, k, t == 1)
        assert b_r < 0.01, b_r                                       # a wrong message moves r by far more
        check("softmax", q, ref.softmax(np.concatenate([zero, prev])), b_q, (family, t))
        a = ref.mean_field_step(lat, a0, q, norm, w_a, w_g, crf.gaussian_xy)
        check(family, got, a[1:] - a[0], b_r, (family, t))
        prev = got
    return prev


# ---- 1. every iteration against fp64 of what it read -------------------------------------------------------------------

TWO = dict(bilateral_weight=3.0, bilateral_xy=30.0, bilateral_rgb=20.0, gaussian_weight=1.5, gaussian_xy=1.3)
ITER_CASES = [
    ((7, 5), 5, 3, "default", {}),
    ((7, 5), 17, 1, "default", {}),
    ((7, 5), 2, 1, "two", dict(iterations=4, **TWO)),
    ((7, 5), 2, 2, "clamped", dict(gaussian_xy=5.0)),                 # R = 15 beyond both sides: clamped to 6
    ((33, 45), 2, 3, "default", {}),
    ((33, 45), 17, 1, "two", dict(iterations=3, **TWO)),
    ((33, 45), 1, 2, "rows", dict(gaussian_xy=13.0)),                 # 3θγ = 39: above h, below w
    ((480, 854), 1, 1, "default", {}),
    ((480, 854), 2, 1, "two", dict(iterations=3, **TWO)),
]


@pytest.mark.parametrize("hw,k,n,name,params", ITER_CASES,
                         ids=[f"{h}x{w}-k{k}-n{n}-{p}" for (h, w), k, n, p, _ in ITER_CASES])
def test_every_iteration(dev, hw, k, n, name, params):
    h, w = hw
    frames, z = _scene(h * w + n, n, h, w), _maps(k + n, k, n, h, w)
    chain("iteration", frames, z, _crf(**params))


# ---- 2. launch regimes ---------------------------------------------------------------------------------------------

def _regime(name):
    if name == "pixels":                 # 3 x 410 k pixels: the pixel loops' second pass
        frames, crf = _scene(7, 3, 480, 854), _crf()
    elif name == "vertices":             # 2.46 M vertices: the neighbour and blur loops' second pass
        frames, crf = np.random.default_rng(8).integers(0, 256, (1, 480, 854, 3), dtype=np.uint8), \
            _crf(bilateral_xy=2.0, bilateral_rgb=1.0)
    else:                                # 38 k vertices, up to 16,663 entries each: splat blocks stride vertices
        frames, crf = _scene(9, 1, 480, 854), _crf()
    lat = _lattice(frames, crf)
    if name == "pixels":
        assert lat.pixels > 1 << 20
    elif name == "vertices":
        assert lat.m > 1 << 20 and lat.occupancy.max() <= 2
    else:
        assert lat.m > 2048 and lat.occupancy.max() > 256
    return frames, crf, lat


@pytest.mark.parametrize("name", ["pixels", "vertices", "occupancy"])
def test_launch_regime(dev, name):
    frames, crf, lat = _regime(name)
    z = _maps(11, 1, frames.shape[0], 480, 854)
    chain("regime-lattice", frames, z, dataclasses.replace(crf, iterations=1, gaussian_weight=0.0), lat)
    chain("regime", frames, z, crf, lat)


# ---- 3. frame counts and the keys' range -------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 2, 4, 5, 8, 9, 1024, 1025, 2048])
def test_frame_counts(dev, n):
    """key_end_bit(n) at powers of two, one past them and at the 2048-frame limit (64-bit keys): every frame's vertices
    counted apart, and the lattice alone (T = 1, w_γ = 0) against the restatement."""
    frames = np.random.default_rng(n).integers(0, 256, (n, 2, 3, 3), dtype=np.uint8)
    z = _maps(n, 2, n, 2, 3)
    crf = _crf(iterations=1, gaussian_weight=0.0, bilateral_xy=3.0, bilateral_rgb=20.0)
    lat = _lattice(frames, crf)
    assert len(set(map(bytes, frames))) == n                          # distinct frames
    chain("frames", frames, z, crf, lat)


def _launches_none(fn, match):
    """fn() must raise before any launch: the package's launch counter is unchanged and the profiler sees no kernel."""
    from osvos_pytorch_b200 import ops
    before = ops.KERNEL_LAUNCHES[0]
    with KernelsRan(_crf_kernel) as k:
        with pytest.raises((ValueError, RuntimeError), match=match):
            fn()
    assert ops.KERNEL_LAUNCHES[0] == before
    assert not k.counts, k.counts


def test_too_many_frames_are_refused_before_any_launch(dev):
    from osvos_pytorch_b200 import _native as nat, ops
    n, h, w = 2049, 2, 3
    f = torch.zeros((n, h, w, 3), dtype=torch.uint8, device="cuda")
    m = torch.zeros((n, 1, h, w), device="cuda")
    _launches_none(lambda: ops.dense_crf(f, [m], _crf()), "2048")
    lib = nat.load()
    assert lib.osvos_dense_crf_workspace_bytes(n, 1, h, w) == 0
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.empty(n * h * w, device="cuda")
    _launches_none(lambda: _native_crf(f, [m], _crf(), ws, out), r"n <= \(1 << kFrameBits\)")


def _fits(h, w, theta_a, theta_b):
    """crf_fits' key-range test, restated: every elevated coordinate's quotient stays within ±510."""
    s = ref.scales(theta_a, theta_b)
    vmax = (w - 1, h - 1, 255, 255, 255)
    cf = [vmax[j] * s[j] for j in range(ref.D)]
    bound = 0.0
    for j in range(ref.D1):
        hi = 0.0
        for i in range(j, ref.D):
            hi += cf[i]
        bound = max(bound, hi, j * cf[j - 1] if j > 0 else 0.0)
    return math.isfinite(bound) and (bound + 20.0) / ref.D1 + 1.0 < ref.Q_BIAS - 1


def _limit(h, w, thetas):
    """The smallest factor f (a double) at which f · thetas fits: f fits, the double below it does not."""
    lo, hi = 1e-6, 1e6
    assert not _fits(h, w, *(lo * t for t in thetas)) and _fits(h, w, *(hi * t for t in thetas))
    while math.nextafter(lo, hi) < hi:
        mid = 0.5 * (lo + hi)
        if mid in (lo, hi):
            break
        if _fits(h, w, *(mid * t for t in thetas)):
            hi = mid
        else:
            lo = mid
    return hi


def _corners(h, w):
    """Random bytes with the extremes of every feature: corners 0 and 255, and pure R, G and B."""
    f = np.random.default_rng(h * w).integers(0, 256, (1, h, w, 3), dtype=np.uint8)
    f[0, 0, 0], f[0, 0, -1], f[0, -1, 0], f[0, -1, -1] = 0, 0, 0, 255
    f[0, 0, 1], f[0, 0, 2], f[0, 0, 3] = (0, 0, 255), (0, 255, 0), (255, 0, 0)
    f[0, -1, 1], f[0, -1, 2], f[0, -1, 3] = (255, 255, 0), (255, 0, 255), (0, 255, 255)
    return f


@pytest.mark.parametrize("thetas", [(1.0, 13.0), (80.0, 1.0), (1.0, 0.5)], ids=["xy", "rgb", "both"])
def test_key_range_edge(dev, thetas):
    """The library accepts exactly what the restated crf_fits accepts, at the limit's two sides and well away from it
    (refusals launch nothing); just inside the limit, on a frame holding every feature's extremes, the restatement's
    quotients stay in range and the kernel equals it: vertex counts, and the lattice alone at T = 1."""
    from osvos_pytorch_b200 import ops
    for h, w in ((480, 854), (40, 56)):
        f = torch.from_numpy(_corners(h, w)).cuda()
        m = torch.zeros((1, 1, h, w), device="cuda")
        edge = _limit(h, w, thetas)
        probes = (0.5 * edge, math.nextafter(edge, 0.0), edge, 2.0 * edge)
        assert [_fits(h, w, fac * thetas[0], fac * thetas[1]) for fac in probes] == [False, False, True, True]
        for fac in probes:
            ta, tb = fac * thetas[0], fac * thetas[1]
            crf = _crf(iterations=1, gaussian_weight=0.0, bilateral_xy=ta, bilateral_rgb=tb)
            if _fits(h, w, ta, tb):
                ops.dense_crf(f, [m], crf)
                torch.cuda.synchronize()
            else:
                _launches_none(lambda: ops.dense_crf(f, [m], crf), "crf_fits")
    frames = _corners(40, 56)
    ta, tb = edge * thetas[0], edge * thetas[1]
    crf = _crf(iterations=1, gaussian_weight=0.0, bilateral_xy=ta, bilateral_rgb=tb)
    lat = _lattice(frames, crf)                                       # elevate asserts every quotient's range
    chain("key-edge", frames, _maps(3, 2, 1, 40, 56), crf, lat)


# ---- 4. batch invariance -------------------------------------------------------------------------------------------

def _small_batch():
    frames = np.concatenate([_scene(20 + i, 1, 13, 17) for i in range(9)])
    z = _maps(20, 2, 9, 13, 17)
    frames[6], z[:, 6] = frames[2], z[:, 2]                           # two identical frames with identical maps
    return frames, z


@pytest.mark.parametrize("case", ["3x480x854", "9x13x17"])
def test_one_call_equals_single_frame_calls(dev, case):
    """Each frame has its own lattice, and the grid sizes never change the order of a sum: N frames in one call give
    the bits of N one-frame calls."""
    from osvos_pytorch_b200 import ops
    if case == "9x13x17":
        frames, z = _small_batch()
    else:
        frames, z = _scene(7, 3, 480, 854), _maps(12, 2, 3, 480, 854)
    f, zd = torch.from_numpy(frames).cuda(), torch.from_numpy(z).cuda()
    n = frames.shape[0]
    verts = torch.zeros(n, dtype=torch.int32, device="cuda")
    whole = ops.dense_crf(f, zd, _crf(), vertices=verts)
    for i in range(n):
        vi = torch.zeros(1, dtype=torch.int32, device="cuda")
        one = ops.dense_crf(f[i:i + 1].contiguous(), zd[:, i:i + 1].contiguous(), _crf(), vertices=vi)
        assert torch.equal(one[:, 0], whole[:, i]), i
        assert vi.item() == verts[i].item()
    if case == "9x13x17":
        assert torch.equal(whole[:, 6], whole[:, 2]) and verts[6].item() == verts[2].item()


# ---- 5. workspace and weights --------------------------------------------------------------------------------------

def _native_crf(f, maps, crf, ws, out):
    from osvos_pytorch_b200 import _native as nat
    n, h, w, _ = f.shape
    ptrs = (c_void_p * len(maps))(*(t.data_ptr() for t in maps))
    nat.check(nat.load().osvos_dense_crf(f.data_ptr(), ptrs, out.data_ptr(), ws.data_ptr(), n, len(maps), h, w,
                                         crf.iterations, crf.bilateral_weight, crf.bilateral_xy, crf.bilateral_rgb,
                                         crf.gaussian_weight, crf.gaussian_xy, torch.cuda.current_stream().cuda_stream),
              "osvos_dense_crf")
    return out


def _with_workspace(frames, z, crf, fill):
    from osvos_pytorch_b200 import _native as nat
    k, n, h, w = z.shape
    f = torch.from_numpy(frames).cuda()
    maps = [torch.from_numpy(z[i]).cuda() for i in range(k)]
    ws = torch.full((nat.load().osvos_dense_crf_workspace_bytes(n, k, h, w),), fill, dtype=torch.uint8, device="cuda")
    out = _native_crf(f, maps, crf, ws, torch.empty((k, n, h, w), device="cuda"))
    return out, ws[:4 * n].view(torch.int32).clone()


@pytest.mark.parametrize("shape", [(2, 61, 77), (1, 480, 854)])
def test_workspace_contents_do_not_matter(dev, shape):
    n, h, w = shape
    frames, z = _scene(30, n, h, w), _maps(30, 3, n, h, w)
    a, va = _with_workspace(frames, z, _crf(), 0xFF)
    b, vb = _with_workspace(frames, z, _crf(), 0)
    assert torch.equal(a, b) and torch.equal(va, vb)
    assert not torch.isnan(a).any()


def test_zero_weights_return_the_maps_bit_for_bit(dev):
    """w_α = w_γ = 0: a = a⁰ + 0·B + 0·S, so r = z exactly; a message read from stale workspace (NaN) would show."""
    frames, z = _scene(31, 2, 23, 29), _maps(31, 2, 2, 23, 29)
    out, _ = _with_workspace(frames, z, _crf(iterations=3, bilateral_weight=0.0, gaussian_weight=0.0), 0xFF)
    assert torch.equal(out.cpu(), torch.from_numpy(z))


def test_most_objects(dev):
    """K = 254, the merge's limit: 255 labels through every iteration."""
    frames, z = _scene(32, 2, 9, 13), _maps(32, 254, 2, 9, 13)
    chain("objects", frames, z, _crf(iterations=3))


# ---- 6. the kernels each call runs -----------------------------------------------------------------------------------

def _crf_kernel(name):
    """A crf_* kernel's (name, template args); CUB's sort and scan kernels None; any other kernel ("other", name)."""
    m = re.search(r"\bcrf_(\w+?)_kernel(?:<([^>]*)>)?", name)
    if m:
        return m.group(1), (m.group(2) or "").replace(" ", "")
    if "cub::" in name or name.startswith("Memset"):              # CUB's sort and scan, and their memsets
        return None
    return "other", name[:80]


def _expected(t):
    return {("elevate", ""): 1, ("mark", ""): 1, ("compact", ""): 1, ("neighbours", ""): 1, ("taps", ""): 1,
            ("splat", ""): t + 1, ("blur", ""): 6 * (t + 1), ("slice", ""): t + 1, ("gauss_rows", ""): t,
            ("update", "true,false"): 1, ("update", "false,false"): t - 1, ("update", "false,true"): 1}


@pytest.mark.parametrize("t,k,n", [(1, 1, 1), (2, 3, 2), (5, 2, 3)])
def test_kernels_ran(dev, t, k, n):
    """One call's kernels and launch counts.  As in test_gpu_general_tail_schedules.ran, a window that loses a record
    is run again, at most twice.  Late in the whole GPU suite torch.profiler can keep losing device records: a window
    holds fewer device records than the launch calls it recorded on the host.  On the H100, after the files before this
    one, most windows and their repeats lost crf_elevate_kernel's record; in a fresh process every window is whole.
    A window whose kernels are all recorded is checked exactly.  If it lost some but the ones it kept are all expected,
    it cannot tell whether the rest ran: it is counted in BLIND, with the kernels it missed, and reported at module
    end.  A window that records a wrong kernel, an unexpected one or more launches than expected fails."""
    from osvos_pytorch_b200 import ops
    f = torch.from_numpy(_scene(40, n, 31, 37)).cuda()
    zd = torch.from_numpy(_maps(40, k, n, 31, 37)).cuda()
    crf = _crf(iterations=t)
    expected = {key: v for key, v in _expected(t).items() if v}
    for _ in range(3):
        with KernelsRan(_crf_kernel) as kr:
            ops.dense_crf(f, zd, crf)
        if sum(kr.counts.values()) >= sum(expected.values()):
            break
    got = dict(kr.counts)
    launches = sum(c for name, d, c in kr.seen if d == "CPU" and name.startswith("cudaLaunchKernel"))
    records = sum(c for name, d, c in kr.seen if d == "CUDA" and not name.startswith(("Memset", "Memcpy")))
    if got != expected and records < launches and all(c <= expected.get(key, 0) for key, c in got.items()):
        BLIND.append(((t, k, n), {key: v - got.get(key, 0) for key, v in expected.items() if got.get(key, 0) < v}))
        return
    assert got == expected, (kr.counts, kr.seen[:20])

// Connected components of masks and the component filter of K fused maps (DESIGN.md §30).
//
// Labelling, one plane (a frame, or an object's map of one frame) per blockIdx.z / blockIdx.y:
//   1. cc_local_kernel: each 32x16 tile is labelled in shared memory by union-find, every link from the larger root to
//      the smaller with atomicMin, so each tile-local root is its component's smallest raster index; the roots are
//      written to global memory as plane raster indices (the tile's raster order is the plane's).  A warp's ballot
//      gives each row's runs, so only the first contact between two runs is a union;
//   2. cc_border_kernel: the same unions over the edges that cross a tile border, in global memory;
//   3. cc_compress_kernel: every pixel's label becomes its root, which is then its component's first pixel in raster
//      order whatever the scheduling was.
// connected_components then flags the roots, CUB scans the flags (inclusive, over all planes) and cc_number_kernel
// numbers each component by its root's rank in the plane: scipy.ndimage.label's numbering, with no sort.
//
// The filter (one call: all K·N planes labelled at once; `near` then takes the frames in order, one launch sequence
// each, since a frame's prior is the previous frame's kept mask):
//   4. the compress pass also adds each component's area at its root (integer atomics, aggregated per warp);
//   5. near: the exact squared distance D to the prior P (the column pass of edt.cuh, then a row pass that takes each
//      component's minimum of D with atomicMin at its root);
//   6. cf_decide_kernel: per plane, C* = the maximum of (area << 32) | ~root by 64-bit atomicMax (the root orders the
//      components as their labels do, so ties go to the smallest label), the component count and the count within the
//      radius;
//   7. cf_write_kernel: z' = z, or -z on the pixels of dropped components; the kept mask; |F| and the pixels removed.
// Everything after the z > 0 test is integer, so nothing depends on the launch configuration.  Nothing is read back.
#include <limits.h>

#include <cub/cub.cuh>

#include "edt.cuh"
#include "merge.cuh"

namespace osvos {
namespace {

constexpr int kTileW = 32;           // a warp per tile row
constexpr int kTileH = 16;
constexpr int kThreads = 256;        // per-pixel passes
constexpr int kMaxBlocksX = 1024;
constexpr int kMaxPlanesPerGrid = 65535;

// The foreground of a labelling: a uint8 mask (nonzero) or an fp32 map (z > 0, so NaN and ±0 are background).  Plane q
// of a launch is frame q of the masks, or object q / nf, frame j0 + q % nf of the maps.
struct MaskPlanes {
  const uint8_t* mask;
  __device__ __forceinline__ bool fg(int q, size_t hw, size_t i) const { return __ldg(mask + q * hw + i) != 0; }
};

struct MapPlanes {
  MergeMaps m;
  int j0, nf;
  __device__ __forceinline__ const float* plane(int q, size_t hw) const {
    return m.map[q / nf] + static_cast<size_t>(j0 + q % nf) * hw;
  }
  __device__ __forceinline__ bool fg(int q, size_t hw, size_t i) const { return __ldg(plane(q, hw) + i) > 0.f; }
};

// Root of x in the parent array p (every p[x] <= x; a root has p[x] == x).  Parents only decrease, so a stale read is
// still an ancestor; reads bypass L1, where another SM's atomics would not be seen.
__device__ __forceinline__ int find_root(const int* p, int x) {
  int px = __ldcg(p + x);
  while (px != x) {
    x = px;
    px = __ldcg(p + x);
  }
  return x;
}

__device__ __forceinline__ int find_root_shared(volatile int* p, int x) {
  int px = p[x];
  while (px != x) {
    x = px;
    px = p[x];
  }
  return x;
}

// Union by atomicMin: the larger root is linked under the smaller; a lost race retries from the value it saw.
__device__ __forceinline__ void unite_shared(int* p, int a, int b) {
  volatile int* vp = p;
  for (;;) {
    a = find_root_shared(vp, a);
    b = find_root_shared(vp, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(p + b, a);
    if (old == b) return;
    b = old;
  }
}

__device__ __forceinline__ void unite_global(int* p, int a, int b) {
  for (;;) {
    a = find_root(p, a);
    b = find_root(p, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(p + b, a);
    if (old == b) return;
    b = old;
  }
}

// Whether run-based unions join a pixel p, in a row run that starts at p (run_start) or continues from its left, to the
// row above: `u`, `ul`, `ur` are the foreground of the pixels above p, up-left and up-right.  Every run of the row above
// that touches p's run is united with it once, at the first pixel where they touch:
//   4: at p when the pixel above is set and p starts its run or the pixel up-left is not set;
//   8: at a run's start, with the up-left pixel if set, else the one above; and at any p whose up-right pixel starts a
//      run above (set, with the pixel above not set).
template <int CONN>
__device__ __forceinline__ void unite_with_row_above(int* p, bool shared, int i, int up_i, bool run_start, bool u,
                                                     bool ul, bool ur) {
  auto unite = [&](int a, int b) { if (shared) unite_shared(p, a, b); else unite_global(p, a, b); };
  if (CONN == 4) {
    if (u && (run_start || !ul)) unite(i, up_i);
  } else {
    if (run_start) {
      if (ul) unite(i, up_i - 1);
      else if (u) unite(i, up_i);
    }
    if (ur && !u) unite(i, up_i + 1);
  }
}

// 1. grid (tiles across, tiles down, planes); block (kTileW, kTileH): one warp per tile row.  A ballot gives each row's
// runs; every pixel starts out linked to its run's first pixel, and run-based unions join the rows.  labels[q][i]: the
// root's plane raster index, -1 for background.  The filter's per-pixel accumulators (area, and with near the minimum
// distance) are reset here.
template <typename Src, int CONN>
__global__ void __launch_bounds__(kTileW * kTileH)
cc_local_kernel(Src src, int* __restrict__ labels, int* __restrict__ area, int* __restrict__ mind, int planes, int h,
                int w) {
  __shared__ int par[kTileH * kTileW];
  __shared__ unsigned rows[kTileH];
  const int lx = threadIdx.x, ly = threadIdx.y, li = ly * kTileW + lx;
  const int x = blockIdx.x * kTileW + lx, y = blockIdx.y * kTileH + ly;
  const bool in = x < w && y < h;
  const size_t hw = static_cast<size_t>(h) * w, i = static_cast<size_t>(y) * w + x;
  for (int q = blockIdx.z; q < planes; q += gridDim.z) {
    const bool fg = in && src.fg(q, hw, i);
    const unsigned bits = __ballot_sync(0xffffffffu, fg);
    const unsigned bg_left = ~bits & ((1u << lx) - 1u);
    const int start = bg_left ? 32 - __clz(bg_left) : 0;
    par[li] = fg ? ly * kTileW + start : -1;
    if (lx == 0) rows[ly] = bits;
    __syncthreads();
    if (fg && ly > 0) {
      const unsigned up = rows[ly - 1];
      unite_with_row_above<CONN>(par, true, li, li - kTileW, start == lx, (up >> lx) & 1u,
                                 lx > 0 && ((up >> (lx - 1)) & 1u), lx + 1 < kTileW && ((up >> (lx + 1)) & 1u));
    }
    __syncthreads();
    if (in) {
      const size_t o = q * hw + i;
      int g = -1;
      if (fg) {
        const int r = find_root_shared(par, li);
        g = (blockIdx.y * kTileH + r / kTileW) * w + blockIdx.x * kTileW + r % kTileW;
      }
      labels[o] = g;
      if (area != nullptr) area[o] = 0;
      if (mind != nullptr) mind[o] = INT_MAX;
    }
    __syncthreads();                                 // par and rows are reused by the next plane
  }
}

// 2. the same grid: the edges across tile borders, in global memory, reduced as in the tile:
//   - a tile's top row (one warp) against the row above, by the run rule (the up-left pixel of lane 0 and the up-right
//     pixel of lane 31 are read from the neighbouring tiles);
//   - the left column against the pixel to its left (and at 8 up-left): not needed when the pixel above and the one
//     up-left are both set, since both are then joined through the row above;
//   - at 8, the right column below the top row against its up-right pixel: not needed when the pixel above or the one
//     to the right is set.
template <int CONN>
__global__ void __launch_bounds__(kTileW * kTileH)
cc_border_kernel(int* __restrict__ labels, int planes, int h, int w) {
  const int lx = threadIdx.x, ly = threadIdx.y;
  const int x = blockIdx.x * kTileW + lx, y = blockIdx.y * kTileH + ly;
  const bool in = x < w && y < h;
  const bool top = ly == 0 && y > 0;                 // the same for the whole warp
  const bool left = lx == 0 && x > 0 && y < h;
  const bool right = CONN == 8 && lx == kTileW - 1 && ly > 0 && x + 1 < w && y < h;
  if (!top && !left && !right) return;
  const size_t hw = static_cast<size_t>(h) * w;
  const int i = y * w + x;
  for (int q = blockIdx.z; q < planes; q += gridDim.z) {
    int* p = labels + q * hw;
    const bool f = in && __ldcg(p + i) >= 0;
    if (top) {
      const bool fu = in && __ldcg(p + i - w) >= 0;
      const unsigned fb = __ballot_sync(0xffffffffu, f), ub = __ballot_sync(0xffffffffu, fu);
      if (f) {
        const bool ul = lx > 0 ? (ub >> (lx - 1)) & 1u : x > 0 && __ldcg(p + i - w - 1) >= 0;
        const bool ur = lx + 1 < kTileW ? (ub >> (lx + 1)) & 1u : x + 1 < w && __ldcg(p + i - w + 1) >= 0;
        unite_with_row_above<CONN>(p, false, i, i - w, lx == 0 || !((fb >> (lx - 1)) & 1u), fu, ul, ur);
      }
    }
    if (!f) continue;
    if (left) {
      const bool fl = __ldcg(p + i - 1) >= 0;
      const bool fu = y > 0 && __ldcg(p + i - w) >= 0, ful = y > 0 && __ldcg(p + i - w - 1) >= 0;
      if (!(fu && ful)) {
        if (fl) unite_global(p, i, i - 1);
        else if (CONN == 8 && ful) unite_global(p, i, i - w - 1);
      }
    }
    if (right && __ldcg(p + i - w + 1) >= 0 && __ldcg(p + i - w) < 0 && __ldcg(p + i + 1) < 0)
      unite_global(p, i, i - w + 1);
  }
}

// Per-pixel passes: blockIdx.y (and its grid stride) the plane, blockIdx.x and threadIdx.x a block-stride loop over the
// plane's pixels whose trip count is the same for every thread of the block, so whole warps take each step together.
#define CC_PLANE_LOOP(planes, hw)                                                                         \
  for (int q = blockIdx.y; q < (planes); q += gridDim.y)                                                  \
    for (size_t base = static_cast<size_t>(blockIdx.x) * blockDim.x; base < (hw);                         \
         base += static_cast<size_t>(gridDim.x) * blockDim.x)

// 3. labels -> roots.  connected_components: `flags` = 1 at each root.  The filter: each component's area, added at its
// root by one atomic per warp and root.
__global__ void __launch_bounds__(kThreads)
cc_compress_kernel(int* __restrict__ labels, int* __restrict__ flags, int* __restrict__ area, int planes, size_t hw) {
  CC_PLANE_LOOP(planes, hw) {
    const size_t i = base + threadIdx.x;
    int* p = labels + q * hw;
    int r = -1;
    if (i < hw) {
      const int l = p[i];
      if (l >= 0) {
        r = find_root(p, l);
        p[i] = r;
      }
      if (flags != nullptr) flags[q * hw + i] = r == static_cast<int>(i);
    }
    if (area != nullptr) {
      const unsigned same = __match_any_sync(0xffffffffu, r);
      if (r >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(area + q * hw + r, __popc(same));
    }
  }
}

// 4. connected_components: label = the root's rank among the plane's roots (1-based), from the inclusive scan of the
// flags over all planes; counts[q] = the plane's number of roots.
__global__ void __launch_bounds__(kThreads)
cc_number_kernel(int* __restrict__ labels, const int* __restrict__ scan, int* __restrict__ counts, int planes,
                 size_t hw) {
  CC_PLANE_LOOP(planes, hw) {
    const size_t i = base + threadIdx.x;
    if (i >= hw) continue;
    const int before = q > 0 ? __ldg(scan + q * hw - 1) : 0;
    int* p = labels + q * hw;
    const int r = p[i];
    p[i] = r >= 0 ? __ldg(scan + q * hw + r) - before : 0;
    if (i == hw - 1) counts[q] = __ldg(scan + q * hw + i) - before;
  }
}

// 5. near: blockIdx.x = row, blockIdx.y = object k of frame j (plane k·n + j of labels / mind); g holds the column pass
// over the prior of frame j.  Each foreground pixel's D goes to its root's minimum (one atomic per warp and root).  An
// empty envelope means an empty prior: D stays "infinite" (INT_MAX) and no component is near it.
__global__ void __launch_bounds__(kRowThreads)
cf_distance_rows_kernel(const int* __restrict__ g, const int* __restrict__ labels, int* __restrict__ mind, int n, int j,
                        int h, int w) {
  extern __shared__ uint32_t stack[];
  const int k = blockIdx.y, y = blockIdx.x;
  const int* grow = g + (static_cast<size_t>(k) * h + y) * w;
  const int count = row_envelope(grow, w, stack);
  if (count == 0) return;
  const size_t hw = static_cast<size_t>(h) * w, plane = (static_cast<size_t>(k) * n + j) * hw;
  const int* lrow = labels + plane + static_cast<size_t>(y) * w;
  int* m = mind + plane;
  for (int x0 = 0; x0 < w; x0 += kRowThreads) {
    const int x = x0 + threadIdx.x;
    const int r = x < w ? __ldg(lrow + x) : -1;
    const unsigned same = __match_any_sync(0xffffffffu, r);
    if (r >= 0) {
      const int d = __reduce_min_sync(same, row_distance(grow, stack, count, x));
      if ((threadIdx.x & 31) == __ffs(same) - 1) atomicMin(m + r, d);
    }
  }
}

// Per-plane decisions of the filter, zeroed before the call.
struct PlaneState {
  unsigned long long* best;   // (area << 32) | ~root of C*
  int* ncomp;                 // components
  int* nnear;                 // components within the radius of the prior (near)
};

__device__ __forceinline__ void warp_add(int v, int* dst) {
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(dst, v);
}

// 6. grid.y over the planes of frames j0 .. j0 + nf - 1 (plane q of the launch: object q / nf, frame j0 + q % nf).
__global__ void __launch_bounds__(kThreads)
cf_decide_kernel(const int* __restrict__ labels, const int* __restrict__ area, const int* __restrict__ mind,
                 PlaneState st, int n, int j0, int nf, int planes, size_t hw, long long r2) {
  CC_PLANE_LOOP(planes, hw) {
    const size_t i = base + threadIdx.x;
    const size_t pq = static_cast<size_t>(q / nf) * n + j0 + q % nf;
    const size_t o = pq * hw + i;
    const bool root = i < hw && __ldg(labels + o) == static_cast<int>(i);
    unsigned long long key = 0;
    if (root) key = static_cast<unsigned long long>(__ldg(area + o)) << 32 | (~static_cast<uint32_t>(i));
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, s);
      key = other > key ? other : key;
    }
    if ((threadIdx.x & 31) == 0 && key) atomicMax(st.best + pq, key);
    warp_add(root, st.ncomp + pq);
    if (mind != nullptr) warp_add(root && __ldg(mind + o) <= r2, st.nnear + pq);
  }
}

// 7. the same planes.  With near and a component within the radius, every such component is kept; otherwise C*.
// stats[pq] = {components, components kept, |F|, pixels removed}; the last two were zeroed before the call.
__global__ void __launch_bounds__(kThreads)
cf_write_kernel(MapPlanes src, const int* __restrict__ labels, const int* __restrict__ mind, PlaneState st,
                float* __restrict__ out, uint8_t* __restrict__ kept, uint8_t* __restrict__ cur, int* __restrict__ stats,
                int n, int planes, size_t hw, long long r2) {
  CC_PLANE_LOOP(planes, hw) {
    const size_t i = base + threadIdx.x;
    const int k = q / src.nf, j = src.j0 + q % src.nf;
    const size_t pq = static_cast<size_t>(k) * n + j;
    const int ncomp = __ldcg(st.ncomp + pq);
    const int nnear = mind != nullptr ? __ldcg(st.nnear + pq) : 0;
    const uint32_t best = ~static_cast<uint32_t>(__ldcg(st.best + pq) & 0xffffffffu);
    bool fg = false, keep = false;
    if (i < hw) {
      const float z = __ldg(src.plane(q, hw) + i);
      fg = z > 0.f;
      if (fg) {
        const int r = __ldg(labels + pq * hw + i);
        keep = nnear > 0 ? __ldg(mind + pq * hw + r) <= r2 : static_cast<uint32_t>(r) == best;
      }
      out[pq * hw + i] = fg && !keep ? -z : z;
      kept[pq * hw + i] = fg && keep;
      if (cur != nullptr) cur[static_cast<size_t>(k) * hw + i] = fg && keep;
      if (i == 0) {
        stats[4 * pq] = ncomp;
        stats[4 * pq + 1] = nnear > 0 ? nnear : (ncomp > 0 ? 1 : 0);
      }
    }
    warp_add(fg, stats + 4 * pq + 2);
    warp_add(fg && !keep, stats + 4 * pq + 3);
  }
}

#undef CC_PLANE_LOOP

size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

dim3 tile_grid(int planes, int h, int w) {
  return dim3((w + kTileW - 1) / kTileW, (h + kTileH - 1) / kTileH, planes < kMaxPlanesPerGrid ? planes : kMaxPlanesPerGrid);
}

dim3 pixel_grid(int planes, size_t hw) {
  const size_t bx = (hw + kThreads - 1) / kThreads;
  return dim3(static_cast<unsigned>(bx < kMaxBlocksX ? bx : kMaxBlocksX),
              planes < kMaxPlanesPerGrid ? planes : kMaxPlanesPerGrid);
}

bool sizes_ok(int n, int k, int h, int w) {
  if (n <= 0 || k <= 0 || h <= 0 || w <= 0 || h >= 32768 || w >= 32768) return false;
  return static_cast<unsigned long long>(n) * k * h * w < (1ull << 31);
}

// Steps 1-3 over `planes` planes.
template <typename Src>
cudaError_t label_planes(Src src, int* labels, int* flags, int* area, int* mind, int planes, int h, int w,
                         int connectivity, cudaStream_t stream) {
  const dim3 tg = tile_grid(planes, h, w), tb(kTileW, kTileH);
  const size_t hw = static_cast<size_t>(h) * w;
  if (connectivity == 4) {
    cc_local_kernel<Src, 4><<<tg, tb, 0, stream>>>(src, labels, area, mind, planes, h, w);
    cc_border_kernel<4><<<tg, tb, 0, stream>>>(labels, planes, h, w);
  } else {
    cc_local_kernel<Src, 8><<<tg, tb, 0, stream>>>(src, labels, area, mind, planes, h, w);
    cc_border_kernel<8><<<tg, tb, 0, stream>>>(labels, planes, h, w);
  }
  cc_compress_kernel<<<pixel_grid(planes, hw), kThreads, 0, stream>>>(labels, flags, area, planes, hw);
  return cudaGetLastError();
}

cudaError_t scan_bytes(size_t items, size_t* bytes) {
  return cub::DeviceScan::InclusiveSum(nullptr, *bytes, static_cast<const int*>(nullptr), static_cast<int*>(nullptr),
                                       static_cast<int>(items));
}

struct FilterLayout {
  size_t labels, area, mind, g, cur, best, ncomp, nnear, total;
};

FilterLayout filter_layout(int n, int k, int h, int w, bool near) {
  FilterLayout l{};
  const size_t hw = static_cast<size_t>(h) * w, planes = static_cast<size_t>(n) * k;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o = align256(o + bytes); return at; };
  l.best = take(sizeof(unsigned long long) * planes);     // best, ncomp, nnear: one zeroed range
  l.ncomp = take(sizeof(int) * planes);
  l.nnear = take(sizeof(int) * planes);
  l.labels = take(sizeof(int) * planes * hw);
  l.area = take(sizeof(int) * planes * hw);
  l.mind = near ? take(sizeof(int) * planes * hw) : 0;
  l.g = near ? take(sizeof(int) * k * hw) : 0;
  l.cur = near ? take(k * hw) : 0;
  l.total = o;
  return l;
}

}  // namespace
}  // namespace osvos

using namespace osvos;

extern "C" size_t osvos_connected_components_workspace_bytes(int n, int h, int w) {
  if (!sizes_ok(n, 1, h, w)) return 0;
  const size_t items = static_cast<size_t>(n) * h * w;
  size_t cub_bytes = 0;
  if (scan_bytes(items, &cub_bytes) != cudaSuccess) return 0;
  return 2 * align256(sizeof(int) * items) + align256(cub_bytes);
}

extern "C" int osvos_connected_components(const uint8_t* masks, int* labels, int* counts, void* workspace, int n, int h,
                                          int w, int connectivity, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(masks != nullptr && labels != nullptr && counts != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(sizes_ok(n, 1, h, w));
  OSVOS_CHECK_ARG(connectivity == 4 || connectivity == 8);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(labels) & 3) == 0 && (reinterpret_cast<uintptr_t>(counts) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(workspace) & 255) == 0);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t hw = static_cast<size_t>(h) * w, items = static_cast<size_t>(n) * hw;
  size_t cub_bytes = 0;
  OSVOS_CHECK_CUDA(scan_bytes(items, &cub_bytes));
  char* ws = static_cast<char*>(workspace);
  int* flags = reinterpret_cast<int*>(ws);
  int* scan = reinterpret_cast<int*>(ws + align256(sizeof(int) * items));
  void* tmp = ws + 2 * align256(sizeof(int) * items);
  OSVOS_CHECK_CUDA(label_planes(MaskPlanes{masks}, labels, flags, nullptr, nullptr, n, h, w, connectivity, stream));
  OSVOS_CHECK_CUDA(cub::DeviceScan::InclusiveSum(tmp, cub_bytes, flags, scan, static_cast<int>(items), stream));
  cc_number_kernel<<<pixel_grid(n, hw), kThreads, 0, stream>>>(labels, scan, counts, n, hw);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" size_t osvos_filter_components_workspace_bytes(int n, int k, int h, int w, int mode) {
  if (!sizes_ok(n, k, h, w) || k > OSVOS_MERGE_MAX_OBJECTS || (mode != OSVOS_COMPONENTS_LARGEST &&
                                                             mode != OSVOS_COMPONENTS_NEAR))
    return 0;
  return filter_layout(n, k, h, w, mode == OSVOS_COMPONENTS_NEAR).total;
}

extern "C" int osvos_filter_components(const float* const* maps, const uint8_t* prior, float* out, uint8_t* kept,
                                       int* stats, void* workspace, int n, int k, int h, int w, int mode, int radius,
                                       int connectivity, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(maps != nullptr && out != nullptr && kept != nullptr && stats != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(k >= 1 && k <= OSVOS_MERGE_MAX_OBJECTS && sizes_ok(n, k, h, w));
  OSVOS_CHECK_ARG(mode == OSVOS_COMPONENTS_LARGEST || mode == OSVOS_COMPONENTS_NEAR);
  OSVOS_CHECK_ARG(radius >= 0 && (connectivity == 4 || connectivity == 8));
  for (int i = 0; i < k; ++i)
    OSVOS_CHECK_ARG(maps[i] != nullptr && (reinterpret_cast<uintptr_t>(maps[i]) & 3) == 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(stats) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(workspace) & 255) == 0);
  const bool near = mode == OSVOS_COMPONENTS_NEAR;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static uint64_t rows_done = 0;                     // rows wider than 12288 need more than 48 KiB of envelope
  if (near) OSVOS_CHECK_CUDA(ensure_dynamic_smem(cf_distance_rows_kernel, 4 * 32767, &rows_done));
  const FilterLayout l = filter_layout(n, k, h, w, near);
  char* ws = static_cast<char*>(workspace);
  int* labels = reinterpret_cast<int*>(ws + l.labels);
  int* area = reinterpret_cast<int*>(ws + l.area);
  int* mind = near ? reinterpret_cast<int*>(ws + l.mind) : nullptr;
  int* g = near ? reinterpret_cast<int*>(ws + l.g) : nullptr;
  uint8_t* cur = near ? reinterpret_cast<uint8_t*>(ws + l.cur) : nullptr;
  const PlaneState st{reinterpret_cast<unsigned long long*>(ws + l.best), reinterpret_cast<int*>(ws + l.ncomp),
                      reinterpret_cast<int*>(ws + l.nnear)};
  const size_t hw = static_cast<size_t>(h) * w;
  const int planes = n * k;
  // every squared distance in a frame is at most 2·32766² < 46340² < INT_MAX (an empty prior's "infinite" D): a larger
  // radius means the same as 46340
  const long long rc = radius < 46340 ? radius : 46340, r2 = rc * rc;
  MapPlanes src{};
  for (int i = 0; i < k; ++i) src.m.map[i] = maps[i];
  src.j0 = 0;
  src.nf = n;
  OSVOS_CHECK_CUDA(cudaMemsetAsync(ws + l.best, 0, l.labels - l.best, stream));
  OSVOS_CHECK_CUDA(cudaMemsetAsync(stats, 0, sizeof(int) * 4 * static_cast<size_t>(planes), stream));
  OSVOS_CHECK_CUDA(label_planes(src, labels, nullptr, area, mind, planes, h, w, connectivity, stream));
  if (!near) {
    cf_decide_kernel<<<pixel_grid(planes, hw), kThreads, 0, stream>>>(labels, area, nullptr, st, n, 0, n, planes, hw,
                                                                      r2);
    cf_write_kernel<<<pixel_grid(planes, hw), kThreads, 0, stream>>>(src, labels, nullptr, st, out, kept, nullptr,
                                                                     stats, n, planes, hw, r2);
    OSVOS_CHECK_CUDA(cudaGetLastError());
    return OSVOS_OK;
  }
  const dim3 col_grid((w + kColWidth - 1) / kColWidth, k), col_block(kColWidth, kColGroups), row_grid(h, k);
  const int smem = static_cast<int>(sizeof(uint32_t)) * w;
  for (int j = 0; j < n; ++j) {                      // frame j's prior is frame j - 1's kept mask
    const uint8_t* p = j == 0 ? prior : cur;
    if (p != nullptr) {
      edt_columns_kernel<kFeatureSet><<<col_grid, col_block, 0, stream>>>(p, g, h, w);
      cf_distance_rows_kernel<<<row_grid, kRowThreads, smem, stream>>>(g, labels, mind, n, j, h, w);
    }
    MapPlanes fj = src;
    fj.j0 = j;
    fj.nf = 1;
    cf_decide_kernel<<<pixel_grid(k, hw), kThreads, 0, stream>>>(labels, area, mind, st, n, j, 1, k, hw, r2);
    cf_write_kernel<<<pixel_grid(k, hw), kThreads, 0, stream>>>(fj, labels, mind, st, out, kept, cur, stats, n, k, hw,
                                                                r2);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  return OSVOS_OK;
}

// The exact separable squared Euclidean distance transform over integer squared distances, shared by the online
// adaptation targets (adapt.cu, DESIGN.md §28) and the component filter's distance to the prior mask (components.cu,
// DESIGN.md §30):
//   1. edt_columns_kernel: per column, the squared distance to the nearest feature of that column, or kNone;
//   2. a row kernel of the caller's: row_envelope builds the lower envelope of the row's parabolas, row_distance reads
//      D(x) from it.
#pragma once
#include "common.cuh"

namespace osvos {

// Squared distances: a column distance² is at most 32766² < 2^30 and (x - x')² + g at most 2 * 32766² < 2^31 - 1, so
// int32 holds every value that is formed.  A column without a feature is marked kNone; the row pass leaves such columns
// out of the envelope, so the marker is never added to anything.
constexpr int kNone = -1;
constexpr int kColWidth = 32;     // columns per column-pass block (one warp-row of consecutive bytes)
constexpr int kColGroups = 16;    // row groups per column-pass block
constexpr int kRowThreads = 64;   // threads per row-pass block (one row per block)

enum : int { kFeatureBackground = 0, kFeatureSet = 1 };

template <int MODE>
__device__ __forceinline__ bool is_feature(const uint8_t* __restrict__ src, size_t o) {
  const uint8_t v = __ldg(src + o);
  return MODE == kFeatureBackground ? v == 0 : v != 0;
}

// blockIdx.y = frame; blockIdx.x = a strip of kColWidth columns; threadIdx.y = a group of consecutive rows.  Each thread
// finds the first and last feature of its rows, the block exchanges them, then the thread sweeps its rows down (nearest
// feature above) and up (nearest feature below) and writes the smaller distance squared, or kNone.
template <int MODE>
__global__ void __launch_bounds__(kColWidth * kColGroups)
edt_columns_kernel(const uint8_t* __restrict__ src, int* __restrict__ g, int h, int w) {
  __shared__ int first[kColGroups][kColWidth], last[kColGroups][kColWidth];
  const int f = blockIdx.y;
  const int x = blockIdx.x * kColWidth + threadIdx.x;
  const int r = threadIdx.y;
  const int chunk = (h + kColGroups - 1) / kColGroups;
  const int y0 = min(h, r * chunk), y1 = min(h, y0 + chunk);
  const size_t hw = static_cast<size_t>(h) * w;
  const uint8_t* s = src + f * hw;
  int* gf = g + f * hw;
  int fst = kNone, lst = kNone;
  if (x < w) {
    for (int y = y0; y < y1; ++y) {
      if (is_feature<MODE>(s, static_cast<size_t>(y) * w + x)) {
        if (fst == kNone) fst = y;
        lst = y;
      }
    }
  }
  first[r][threadIdx.x] = fst;
  last[r][threadIdx.x] = lst;
  __syncthreads();
  if (x >= w) return;
  int above = kNone, below = kNone;
  for (int rr = 0; rr < r; ++rr)
    if (last[rr][threadIdx.x] != kNone) above = last[rr][threadIdx.x];
  for (int rr = kColGroups - 1; rr > r; --rr)
    if (first[rr][threadIdx.x] != kNone) below = first[rr][threadIdx.x];
  for (int y = y0; y < y1; ++y) {
    const size_t o = static_cast<size_t>(y) * w + x;
    if (is_feature<MODE>(s, o)) above = y;
    gf[o] = above == kNone ? kNone : y - above;        // distance (not squared) to the nearest feature above
  }
  for (int y = y1 - 1; y >= y0; --y) {
    const size_t o = static_cast<size_t>(y) * w + x;
    if (is_feature<MODE>(s, o)) below = y;
    int d = gf[o];
    if (below != kNone && (d == kNone || below - y < d)) d = below - y;
    gf[o] = d == kNone ? kNone : d * d;
  }
}

// floor(a / b) for b > 0.
__device__ __forceinline__ int floor_div(int a, int b) {
  const int q = a / b;
  return (a % b != 0 && a < 0) ? q - 1 : q;
}

// The last x at which column i's parabola is at most column u's (i < u): (x - i)² + gi <= (x - u)² + gu
// <=> x <= (u² - i² + gu - gi) / (2 (u - i)).  The numerator lies in [-2^30, 2^31 - 1): int32.
__device__ __forceinline__ int parabola_sep(int i, int gi, int u, int gu) {
  return floor_div(u * u - i * i + gu - gi, 2 * (u - i));
}

// Lower envelope of row y's parabolas (Meijster et al.), built by thread 0 into `stack` (entry q: the column s_q in the
// low 16 bits and the first x it wins, t_q, in the high 16); returns the number of entries (0: no column of the row has a
// feature, i.e. the frame has none).  The walk is sequential; it bounds the kernel's time (DESIGN.md §28).  Then every
// thread finds, for each of its x, the last entry with t_q <= x.
static __device__ int row_envelope(const int* __restrict__ grow, int w, uint32_t* stack) {
  __shared__ int count;
  if (threadIdx.x == 0) {
    int q = -1;
    for (int u = 0; u < w; ++u) {
      const int gu = __ldg(grow + u);
      if (gu == kNone) continue;
      while (q >= 0) {
        const int tq = static_cast<int>(stack[q] >> 16), sq = static_cast<int>(stack[q] & 0xffffu);
        const int dq = tq - sq, du = tq - u;
        if (dq * dq + __ldg(grow + sq) > du * du + gu) --q;   // u beats s_q already where s_q starts
        else break;
      }
      if (q < 0) {
        q = 0;
        stack[0] = static_cast<uint32_t>(u);            // t = 0
      } else {
        const int sq = static_cast<int>(stack[q] & 0xffffu);
        const int t = 1 + parabola_sep(sq, __ldg(grow + sq), u, gu);
        if (t < w) stack[++q] = (static_cast<uint32_t>(t) << 16) | static_cast<uint32_t>(u);
      }
    }
    count = q + 1;
  }
  __syncthreads();
  return count;
}

// D(x) of the row from its envelope: binary search for the last entry with t_q <= x.
__device__ __forceinline__ int row_distance(const int* __restrict__ grow, const uint32_t* stack, int count, int x) {
  int lo = 0, hi = count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (static_cast<int>(stack[mid] >> 16) <= x) lo = mid;
    else hi = mid - 1;
  }
  const int s = static_cast<int>(stack[lo] & 0xffffu);
  const int d = x - s;
  return d * d + grow[s];
}

}  // namespace osvos

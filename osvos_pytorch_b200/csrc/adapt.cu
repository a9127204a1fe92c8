// Online adaptation targets (DESIGN.md §28): per frame, the eroded last mask E, the exact squared distance D to E, and the
// labels 1 / 0 / -1 of the void objective.  Both E and D come from one exact separable squared Euclidean distance
// transform over integer squared distances, run twice:
//   1. columns of the background of M (M = last_mask != 0)  -> g[y][x] = squared distance to the nearest background pixel
//      of column x, or "none";
//   2. rows (lower envelope of the parabolas (x - x')² + g[y][x'])  -> E = M ∧ (no background in the frame ∨ D_bg > e²),
//      written as bytes into the workspace, |E| counted;
//   3. columns of E, as 1;
//   4. rows, as 2 -> D, and the labels written straight from it, #positive and #negative counted.
// Everything is integer: the counts are sums of integers, so the output does not depend on the launch configuration.
// The column pass and the row envelope live in edt.cuh, shared with the component filter (components.cu).
#include "edt.cuh"

namespace osvos {

__device__ __forceinline__ void block_add(int v, int* dst) {
  __shared__ int part[kRowThreads / 32];
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();                                 // `part` may still be read by a previous call
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < kRowThreads / 32; ++i) t += part[i];
    if (t) atomicAdd(dst, t);
  }
}

// blockIdx.x = row, blockIdx.y = frame.  g holds the column pass over M's background: E = M ∧ (D_bg > e²), or E = M when
// the frame has no background (an empty envelope).
__global__ void __launch_bounds__(kRowThreads)
erode_rows_kernel(const uint8_t* __restrict__ mask, const int* __restrict__ g, uint8_t* __restrict__ eroded,
                  int* __restrict__ counts, int h, int w, long long e2) {
  extern __shared__ uint32_t stack[];
  const int f = blockIdx.y, y = blockIdx.x;
  const size_t row = (static_cast<size_t>(f) * h + y) * w;
  const int* grow = g + row;
  const int count = row_envelope(grow, w, stack);
  int n = 0;
  for (int x = threadIdx.x; x < w; x += kRowThreads) {
    bool e = __ldg(mask + row + x) != 0;
    if (e && count > 0) e = row_distance(grow, stack, count, x) > e2;
    eroded[row + x] = e;
    n += e;
  }
  block_add(n, counts + 3 * f);
}

// g holds the column pass over E.  Negative: E non-empty (a non-empty envelope) and D > d²; positive: not negative and
// logit > threshold; labels 0 / 1 / -1.
__global__ void __launch_bounds__(kRowThreads)
label_rows_kernel(const float* __restrict__ logits, const int* __restrict__ g, float* __restrict__ labels,
                  int* __restrict__ counts, int h, int w, long long d2, float threshold) {
  extern __shared__ uint32_t stack[];
  const int f = blockIdx.y, y = blockIdx.x;
  const size_t row = (static_cast<size_t>(f) * h + y) * w;
  const int* grow = g + row;
  const int count = row_envelope(grow, w, stack);
  int pos = 0, neg = 0;
  for (int x = threadIdx.x; x < w; x += kRowThreads) {
    const bool negative = count > 0 && row_distance(grow, stack, count, x) > d2;
    const bool positive = !negative && __ldg(logits + row + x) > threshold;
    labels[row + x] = negative ? 0.f : (positive ? 1.f : -1.f);
    pos += positive;
    neg += negative;
  }
  block_add(pos, counts + 3 * f + 1);
  block_add(neg, counts + 3 * f + 2);
}

}  // namespace osvos

using namespace osvos;

extern "C" size_t osvos_adaptation_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  const size_t pixels = static_cast<size_t>(n) * h * w;
  return pixels * sizeof(int) + pixels;            // g, then E
}

extern "C" int osvos_adaptation_labels(const float* logits, const uint8_t* last_mask, float* labels, int* counts,
                                       void* workspace, int n, int h, int w, float logit_threshold, int erosion_r,
                                       int distance_r, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(logits != nullptr && last_mask != nullptr && labels != nullptr && counts != nullptr &&
                  workspace != nullptr);
  OSVOS_CHECK_ARG(n > 0 && n < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768);
  OSVOS_CHECK_ARG(erosion_r >= 0 && distance_r >= 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 3) == 0 && (reinterpret_cast<uintptr_t>(labels) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(counts) & 3) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 3) == 0);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int* g = static_cast<int*>(workspace);
  uint8_t* eroded = reinterpret_cast<uint8_t*>(g + static_cast<size_t>(n) * h * w);
  const int smem = static_cast<int>(sizeof(uint32_t)) * w;       // the row's envelope: at most w entries
  // rows wider than 12288 need more than 48 KiB: opt in once per device, for the widest frame
  static uint64_t erode_done = 0, label_done = 0;
  constexpr int kMaxSmem = static_cast<int>(sizeof(uint32_t)) * 32767;
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(erode_rows_kernel, kMaxSmem, &erode_done));
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(label_rows_kernel, kMaxSmem, &label_done));
  const dim3 col_grid((w + kColWidth - 1) / kColWidth, n), col_block(kColWidth, kColGroups);
  const dim3 row_grid(h, n);
  const long long e2 = static_cast<long long>(erosion_r) * erosion_r;
  const long long d2 = static_cast<long long>(distance_r) * distance_r;
  OSVOS_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 3 * static_cast<size_t>(n), stream));
  edt_columns_kernel<kFeatureBackground><<<col_grid, col_block, 0, stream>>>(last_mask, g, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  erode_rows_kernel<<<row_grid, kRowThreads, smem, stream>>>(last_mask, g, eroded, counts, h, w, e2);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  edt_columns_kernel<kFeatureSet><<<col_grid, col_block, 0, stream>>>(eroded, g, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  label_rows_kernel<<<row_grid, kRowThreads, smem, stream>>>(logits, g, labels, counts, h, w, d2, logit_threshold);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

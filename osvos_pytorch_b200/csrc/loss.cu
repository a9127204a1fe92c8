// class_balanced_cross_entropy_loss (objective.cuh) as two bandwidth-bound kernels with 128-bit loads, warp-shuffle
// reductions and one fp64 atomic per block and quantity:
//   forward : sums = {S_pos, S_neg, P, N}, loss[0] = (Nn/N * S_pos + P/N * S_neg) / divisor
//   backward: dx = g * w * (sigmoid(x) - y) / divisor
// The void forms (OSVOS_FLAG_VOID_LABELS, osvos_cbce_bwd_void) leave pixels with y < 0 out of every sum and count, and
// give them zero gradient.
#include "objective.cuh"

namespace osvos {

constexpr int kLossThreads = 256;

// DET: each block stores its sums in its own row behind sums[5] (plain stores), and the last block adds the rows in
// block order instead of the fp64 atomics.
// VOID (OSVOS_FLAG_VOID_LABELS): N = #(y >= 0) is a fourth block sum (sums[3]) instead of the element count, and
// N == 0 gives loss 0.
template <bool DET, bool VOID>
__device__ __forceinline__ void cbce_fwd_body(const float* __restrict__ x, const float* __restrict__ label, size_t total,
                                              double* __restrict__ sums, double divisor, float* __restrict__ loss) {
  CbceSums<1, false, VOID> acc;
  const size_t nvec = total / 4;
  for (size_t v = blockIdx.x * static_cast<size_t>(kLossThreads) + threadIdx.x; v < nvec;
       v += static_cast<size_t>(gridDim.x) * kLossThreads) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + v);
    const float4 lv = __ldg(reinterpret_cast<const float4*>(label) + v);
    acc.add({xv.x}, lv.x);
    acc.add({xv.y}, lv.y);
    acc.add({xv.z}, lv.z);
    acc.add({xv.w}, lv.w);
  }
  if (blockIdx.x == 0 && threadIdx.x < (total & 3)) {
    const size_t e = nvec * 4 + threadIdx.x;
    acc.add({x[e]}, label[e]);
  }
  // the last block to arrive (counter in sums[4]): loss[0] = numerator / divisor ; sums[3] = N
  const bool last = commit_block_sums<kLossThreads, 5, DET>(acc.v, sums, IdentitySlot());
  if (last && threadIdx.x == 0) {
    const double tot = VOID ? __ldcg(sums + 3) : static_cast<double>(total);
    if constexpr (!VOID) sums[3] = tot;
    loss[0] = !VOID || tot > 0.0
                  ? static_cast<float>(cbce_numerator(__ldcg(sums + 0), __ldcg(sums + 1), __ldcg(sums + 2), tot) / divisor)
                  : 0.f;
  }
}

template <bool DET = false>
__global__ void __launch_bounds__(kLossThreads)
cbce_fwd_kernel(const float* __restrict__ x, const float* __restrict__ label, size_t total, double* __restrict__ sums,
                double divisor, float* __restrict__ loss) {
  cbce_fwd_body<DET, false>(x, label, total, sums, divisor, loss);
}

template <bool DET>
__global__ void __launch_bounds__(kLossThreads)
cbce_fwd_void_kernel(const float* __restrict__ x, const float* __restrict__ label, size_t total,
                     double* __restrict__ sums, double divisor, float* __restrict__ loss) {
  cbce_fwd_body<DET, true>(x, label, total, sums, divisor, loss);
}

// VOID: void pixels (y < 0) get a zero gradient, and N = sums[3] == 0 (every pixel void) gives zero everywhere.
template <bool VOID>
__device__ __forceinline__ void cbce_bwd_body(const float* __restrict__ x, const float* __restrict__ label,
                                              const double* __restrict__ sums, const float* __restrict__ grad_out,
                                              float scale, size_t total, float* __restrict__ dx) {
  const double p = sums[2], n = sums[3];
  const float g = (grad_out ? __ldg(grad_out) : 1.f) * scale;
  float w_pos, w_neg;
  if (VOID && !(n > 0.0)) {
    w_pos = w_neg = 0.f;
  } else {
    w_pos = cbce_pos_weight(p, n) * g;
    w_neg = cbce_neg_weight(p, n) * g;
  }
  const size_t nvec = total / 4;
  for (size_t v = blockIdx.x * static_cast<size_t>(kLossThreads) + threadIdx.x; v < nvec;
       v += static_cast<size_t>(gridDim.x) * kLossThreads) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + v);
    const float4 lv = __ldg(reinterpret_cast<const float4*>(label) + v);
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    const float ls[4] = {lv.x, lv.y, lv.z, lv.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sg = sigmoid(xs[j]);
      o[j] = ls[j] >= 0.5f ? w_pos * (sg - 1.f) : w_neg * sg;
      if constexpr (VOID) o[j] = ls[j] < 0.f ? 0.f : o[j];
    }
    reinterpret_cast<float4*>(dx)[v] = make_float4(o[0], o[1], o[2], o[3]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (total & 3)) {
    const size_t e = nvec * 4 + threadIdx.x;
    const float sg = sigmoid(x[e]);
    const float le = label[e];
    float o = le >= 0.5f ? w_pos * (sg - 1.f) : w_neg * sg;
    if constexpr (VOID) o = le < 0.f ? 0.f : o;
    dx[e] = o;
  }
}

__global__ void __launch_bounds__(kLossThreads)
cbce_bwd_kernel(const float* __restrict__ x, const float* __restrict__ label, const double* __restrict__ sums,
                const float* __restrict__ grad_out, float scale, size_t total, float* __restrict__ dx) {
  cbce_bwd_body<false>(x, label, sums, grad_out, scale, total, dx);
}

__global__ void __launch_bounds__(kLossThreads)
cbce_bwd_void_kernel(const float* __restrict__ x, const float* __restrict__ label, const double* __restrict__ sums,
                     const float* __restrict__ grad_out, float scale, size_t total, float* __restrict__ dx) {
  cbce_bwd_body<true>(x, label, sums, grad_out, scale, total, dx);
}

}  // namespace osvos

using namespace osvos;

static int loss_grid(size_t total) {
  size_t blocks = (total / 4 + kLossThreads - 1) / kLossThreads;
  const size_t cap = static_cast<size_t>(device_sm_count()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

constexpr int kCbceFlags = OSVOS_FLAG_DETERMINISTIC | OSVOS_FLAG_VOID_LABELS;

extern "C" size_t osvos_cbce_fwd_sums(size_t numel, int flags) {
  if (numel == 0 || (flags & ~kCbceFlags) != 0) return 0;
  const size_t vals = (flags & OSVOS_FLAG_VOID_LABELS) ? 4 : 3;
  return (flags & OSVOS_FLAG_DETERMINISTIC) ? 5 + vals * static_cast<size_t>(loss_grid(numel)) : 5;
}

extern "C" int osvos_cbce_fwd(const float* output, const float* label, size_t numel, double divisor, double* sums,
                              float* loss, int flags, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(output != nullptr && label != nullptr && sums != nullptr && loss != nullptr && numel > 0);
  OSVOS_CHECK_ARG(((reinterpret_cast<uintptr_t>(output) | reinterpret_cast<uintptr_t>(label)) & 15) == 0);
  OSVOS_CHECK_ARG(divisor > 0);
  OSVOS_CHECK_ARG((flags & ~kCbceFlags) == 0);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // deterministic: the block rows are written in full, so in both forms only the five leading values (with the arrival
  // counter) need zeroing
  OSVOS_CHECK_CUDA(cudaMemsetAsync(sums, 0, 5 * sizeof(double), stream));
  const int grid = loss_grid(numel);
  const bool det = (flags & OSVOS_FLAG_DETERMINISTIC) != 0;
  if (flags & OSVOS_FLAG_VOID_LABELS) {
    if (det)
      cbce_fwd_void_kernel<true><<<grid, kLossThreads, 0, stream>>>(output, label, numel, sums, divisor, loss);
    else
      cbce_fwd_void_kernel<false><<<grid, kLossThreads, 0, stream>>>(output, label, numel, sums, divisor, loss);
  } else if (det) {
    cbce_fwd_kernel<true><<<grid, kLossThreads, 0, stream>>>(output, label, numel, sums, divisor, loss);
  } else {
    cbce_fwd_kernel<false><<<grid, kLossThreads, 0, stream>>>(output, label, numel, sums, divisor, loss);
  }
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

static int cbce_bwd(bool void_labels, const float* output, const float* label, const double* sums,
                    const float* grad_out, double divisor, size_t numel, float* grad_in, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(output != nullptr && label != nullptr && sums != nullptr && grad_in != nullptr && numel > 0);
  OSVOS_CHECK_ARG(((reinterpret_cast<uintptr_t>(output) | reinterpret_cast<uintptr_t>(label) |
                    reinterpret_cast<uintptr_t>(grad_in)) & 15) == 0);
  const float scale = static_cast<float>(1.0 / divisor);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (void_labels)
    cbce_bwd_void_kernel<<<loss_grid(numel), kLossThreads, 0, stream>>>(output, label, sums, grad_out, scale, numel,
                                                                        grad_in);
  else
    cbce_bwd_kernel<<<loss_grid(numel), kLossThreads, 0, stream>>>(output, label, sums, grad_out, scale, numel,
                                                                   grad_in);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_cbce_bwd(const float* output, const float* label, const double* sums, const float* grad_out,
                              double divisor, size_t numel, float* grad_in, osvos_stream_t stream) {
  return cbce_bwd(false, output, label, sums, grad_out, divisor, numel, grad_in, stream);
}

extern "C" int osvos_cbce_bwd_void(const float* output, const float* label, const double* sums, const float* grad_out,
                                   double divisor, size_t numel, float* grad_in, osvos_stream_t stream) {
  return cbce_bwd(true, output, label, sums, grad_out, divisor, numel, grad_in, stream);
}

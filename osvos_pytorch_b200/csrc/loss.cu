// class_balanced_cross_entropy_loss (layers/osvos_layers.py:19-48 of the
// reference) as two bandwidth-bound kernels with 128-bit loads, warp-shuffle
// reductions and one fp64 atomic per block and quantity:
//   forward : sums = {S_pos = sum_{y=1} (softplus(x) - x), S_neg = sum_{y=0} softplus(x), P, N}
//             loss = (Nn/N * S_pos + P/N * S_neg) / divisor,  Nn = N - P      (:38-46)
//   backward: dx = g * w * (sigmoid(x) - y) / divisor, w = y*Nn/N + (1-y)*P/N
#include "common.cuh"

namespace osvos {

constexpr int kLossThreads = 256;

__device__ __forceinline__ float softplus_l(float x) { return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x))); }

// DET: each block stores its three sums in its own row behind sums[5] (plain stores), and the last block adds the rows
// in block order instead of the fp64 atomics.
template <bool DET = false>
__global__ void __launch_bounds__(kLossThreads)
cbce_fwd_kernel(const float* __restrict__ x, const float* __restrict__ label, size_t total, double* __restrict__ sums,
                double divisor, float* __restrict__ loss) {
  float s_pos = 0.f, s_neg = 0.f, cnt = 0.f;
  const size_t nvec = total / 4;
  for (size_t v = blockIdx.x * static_cast<size_t>(kLossThreads) + threadIdx.x; v < nvec;
       v += static_cast<size_t>(gridDim.x) * kLossThreads) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + v);
    const float4 lv = __ldg(reinterpret_cast<const float4*>(label) + v);
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    const float ls[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sp = softplus_l(xs[j]);
      if (ls[j] >= 0.5f) {
        s_pos += sp - xs[j];
        cnt += 1.f;
      } else {
        s_neg += sp;
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < (total & 3)) {
    const size_t e = nvec * 4 + threadIdx.x;
    const float xe = x[e];
    const float sp = softplus_l(xe);
    if (label[e] >= 0.5f) {
      s_pos += sp - xe;
      cnt += 1.f;
    } else {
      s_neg += sp;
    }
  }
  float vals[3] = {s_pos, s_neg, cnt};
  __shared__ float red[kLossThreads / 32][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) vals[i] += __shfl_xor_sync(0xffffffffu, vals[i], off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    red[warp][0] = vals[0];
    red[warp][1] = vals[1];
    red[warp][2] = vals[2];
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double acc = 0.0;
    for (int w = 0; w < kLossThreads / 32; ++w) acc += static_cast<double>(red[w][threadIdx.x]);
    if constexpr (DET)
      sums[5 + 3 * static_cast<size_t>(blockIdx.x) + threadIdx.x] = acc;
    else
      atomicAdd(sums + threadIdx.x, acc);
  }
  // last block to arrive (counter in sums[4]): loss[0] = (Nn/N * S_pos + P/N * S_neg) / divisor ; sums[3] = N
  const bool last = last_block_arrives(reinterpret_cast<unsigned int*>(sums + 4));
  if constexpr (DET) {
    if (last) {
      __shared__ double dred[kLossThreads];
      for (int i = 0; i < 3; ++i) {
        const double t = block_ordered_sum(sums + 5 + i, static_cast<int>(gridDim.x), 3, dred);
        if (threadIdx.x == 0) sums[i] = t;
      }
    }
  }
  if (last && threadIdx.x == 0) {
    const double tot = static_cast<double>(total);
    const double p = __ldcg(sums + 2), nn = tot - p;
    sums[3] = tot;
    loss[0] = static_cast<float>((nn / tot * __ldcg(sums + 0) + p / tot * __ldcg(sums + 1)) / divisor);
  }
}

__global__ void __launch_bounds__(kLossThreads)
cbce_bwd_kernel(const float* __restrict__ x, const float* __restrict__ label, const double* __restrict__ sums,
                const float* __restrict__ grad_out, float scale, size_t total, float* __restrict__ dx) {
  const double p = sums[2], n = sums[3];
  const float g = (grad_out ? __ldg(grad_out) : 1.f) * scale;
  const float w_pos = static_cast<float>((n - p) / n) * g;
  const float w_neg = static_cast<float>(p / n) * g;
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
      const float sg = 1.f / (1.f + __expf(-xs[j]));
      o[j] = ls[j] >= 0.5f ? w_pos * (sg - 1.f) : w_neg * sg;
    }
    reinterpret_cast<float4*>(dx)[v] = make_float4(o[0], o[1], o[2], o[3]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (total & 3)) {
    const size_t e = nvec * 4 + threadIdx.x;
    const float sg = 1.f / (1.f + __expf(-x[e]));
    dx[e] = label[e] >= 0.5f ? w_pos * (sg - 1.f) : w_neg * sg;
  }
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

extern "C" size_t osvos_cbce_fwd_sums(size_t numel, int flags) {
  if (numel == 0 || (flags & ~OSVOS_FLAG_DETERMINISTIC) != 0) return 0;
  return (flags & OSVOS_FLAG_DETERMINISTIC) ? 5 + 3 * static_cast<size_t>(loss_grid(numel)) : 5;
}

extern "C" int osvos_cbce_fwd(const float* output, const float* label, size_t numel, double divisor, double* sums,
                              float* loss, int flags, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(output != nullptr && label != nullptr && sums != nullptr && loss != nullptr && numel > 0);
  OSVOS_CHECK_ARG(((reinterpret_cast<uintptr_t>(output) | reinterpret_cast<uintptr_t>(label)) & 15) == 0);
  OSVOS_CHECK_ARG(divisor > 0);
  OSVOS_CHECK_ARG((flags & ~OSVOS_FLAG_DETERMINISTIC) == 0);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // deterministic: the block rows are written in full, so in both forms only the five leading values (with the arrival
  // counter) need zeroing
  OSVOS_CHECK_CUDA(cudaMemsetAsync(sums, 0, 5 * sizeof(double), stream));
  if (flags & OSVOS_FLAG_DETERMINISTIC)
    cbce_fwd_kernel<true><<<loss_grid(numel), kLossThreads, 0, stream>>>(output, label, numel, sums, divisor, loss);
  else
    cbce_fwd_kernel<false><<<loss_grid(numel), kLossThreads, 0, stream>>>(output, label, numel, sums, divisor, loss);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_cbce_bwd(const float* output, const float* label, const double* sums, const float* grad_out,
                              double divisor, size_t numel, float* grad_in, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(output != nullptr && label != nullptr && sums != nullptr && grad_in != nullptr && numel > 0);
  OSVOS_CHECK_ARG(((reinterpret_cast<uintptr_t>(output) | reinterpret_cast<uintptr_t>(label) |
                    reinterpret_cast<uintptr_t>(grad_in)) & 15) == 0);
  cbce_bwd_kernel<<<loss_grid(numel), kLossThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
      output, label, sums, grad_out, static_cast<float>(1.0 / divisor), numel, grad_in);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// class_balanced_cross_entropy_loss (layers/osvos_layers.py:19-48 of the
// reference) as two bandwidth-bound kernels with 128-bit loads, warp-shuffle
// reductions and one fp64 atomic per block and quantity:
//   forward : sums = {S_pos = sum_{y=1} (softplus(x) - x), S_neg = sum_{y=0} softplus(x), P, N}
//             loss = (Nn/N * S_pos + P/N * S_neg) / divisor,  Nn = N - P      (:38-46)
//   backward: dx = g * w * (sigmoid(x) - y) / divisor, w = y*Nn/N + (1-y)*P/N
// The void forms (OSVOS_FLAG_VOID_LABELS, osvos_cbce_bwd_void) leave pixels with y < 0 out of every sum and count, and
// give them zero gradient.
#include "common.cuh"

namespace osvos {

constexpr int kLossThreads = 256;

__device__ __forceinline__ float softplus_l(float x) { return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x))); }

// DET: each block stores its sums in its own row behind sums[5] (plain stores), and the last block adds the rows in
// block order instead of the fp64 atomics.
// VOID (OSVOS_FLAG_VOID_LABELS): a label y < 0 is a void pixel, counted in neither class; N = #(y >= 0) is a fourth
// block sum (sums[3]) instead of the element count, and N == 0 gives loss 0.
template <bool DET, bool VOID>
__device__ __forceinline__ void cbce_fwd_body(const float* __restrict__ x, const float* __restrict__ label, size_t total,
                                              double* __restrict__ sums, double divisor, float* __restrict__ loss) {
  constexpr int kVals = VOID ? 4 : 3;
  float s_pos = 0.f, s_neg = 0.f, cnt = 0.f, cnt_all = 0.f;
  const size_t nvec = total / 4;
  for (size_t v = blockIdx.x * static_cast<size_t>(kLossThreads) + threadIdx.x; v < nvec;
       v += static_cast<size_t>(gridDim.x) * kLossThreads) {
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x) + v);
    const float4 lv = __ldg(reinterpret_cast<const float4*>(label) + v);
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    const float ls[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if constexpr (VOID) {
        if (ls[j] < 0.f) continue;
        cnt_all += 1.f;
      }
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
    const float le = label[e];
    if (!VOID || le >= 0.f) {
      if constexpr (VOID) cnt_all += 1.f;
      const float sp = softplus_l(xe);
      if (le >= 0.5f) {
        s_pos += sp - xe;
        cnt += 1.f;
      } else {
        s_neg += sp;
      }
    }
  }
  float vals[kVals];
  vals[0] = s_pos, vals[1] = s_neg, vals[2] = cnt;
  if constexpr (VOID) vals[3] = cnt_all;
  __shared__ float red[kLossThreads / 32][kVals];
#pragma unroll
  for (int i = 0; i < kVals; ++i)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) vals[i] += __shfl_xor_sync(0xffffffffu, vals[i], off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kVals; ++i) red[warp][i] = vals[i];
  }
  __syncthreads();
  if (threadIdx.x < kVals) {
    double acc = 0.0;
    for (int w = 0; w < kLossThreads / 32; ++w) acc += static_cast<double>(red[w][threadIdx.x]);
    if constexpr (DET)
      sums[5 + kVals * static_cast<size_t>(blockIdx.x) + threadIdx.x] = acc;
    else
      atomicAdd(sums + threadIdx.x, acc);
  }
  // last block to arrive (counter in sums[4]): loss[0] = (Nn/N * S_pos + P/N * S_neg) / divisor ; sums[3] = N
  const bool last = last_block_arrives(reinterpret_cast<unsigned int*>(sums + 4));
  if constexpr (DET) {
    if (last) {
      __shared__ double dred[kLossThreads];
      for (int i = 0; i < kVals; ++i) {
        const double t = block_ordered_sum(sums + 5 + i, static_cast<int>(gridDim.x), kVals, dred);
        if (threadIdx.x == 0) sums[i] = t;
      }
    }
  }
  if (last && threadIdx.x == 0) {
    if constexpr (VOID) {
      const double tot = __ldcg(sums + 3);
      const double p = __ldcg(sums + 2), nn = tot - p;
      loss[0] = tot > 0.0 ? static_cast<float>((nn / tot * __ldcg(sums + 0) + p / tot * __ldcg(sums + 1)) / divisor)
                          : 0.f;
    } else {
      const double tot = static_cast<double>(total);
      const double p = __ldcg(sums + 2), nn = tot - p;
      sums[3] = tot;
      loss[0] = static_cast<float>((nn / tot * __ldcg(sums + 0) + p / tot * __ldcg(sums + 1)) / divisor);
    }
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
    w_pos = static_cast<float>((n - p) / n) * g;
    w_neg = static_cast<float>(p / n) * g;
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
      const float sg = 1.f / (1.f + __expf(-xs[j]));
      o[j] = ls[j] >= 0.5f ? w_pos * (sg - 1.f) : w_neg * sg;
      if constexpr (VOID) o[j] = ls[j] < 0.f ? 0.f : o[j];
    }
    reinterpret_cast<float4*>(dx)[v] = make_float4(o[0], o[1], o[2], o[3]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (total & 3)) {
    const size_t e = nvec * 4 + threadIdx.x;
    const float sg = 1.f / (1.f + __expf(-x[e]));
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

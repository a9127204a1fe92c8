// Ingest of decoded DAVIS frames (reference dataloaders/davis_2016.py:88-108 make_img_gt_pair + custom_transforms.py
// ToTensor): the host decodes JPEG / PNG to uint8 and copies the bytes; the float conversion, the mean subtraction,
// the mask normalisation, the NHWC -> NCHW transpose and the training augmentation run here.  Bandwidth-bound kernels.
//
// Bit-exactness: the reference computes np.float32(v) - np.float32(mean) (one fp32 rounding; __fsub_rn so nothing is
// contracted) and gt / max(gt.max(), 1e-8) in float64 over fp32 byte values.  The quotient of two integers below 256 is
// the same whether rounded to fp32 directly or first to fp64 (double rounding is innocuous for division when the wide
// format has at least 2p + 2 bits), so __fdiv_rn gives the reference's gt.astype(np.float32).
#include "warp.cuh"

namespace osvos {

constexpr int kIngestThreads = 256;
constexpr int kIngestPx = 4 * kIngestThreads;      // pixels per block: four per thread
constexpr int kStatsBytes = 16 * 1024;            // mask bytes reduced per block

// uint8 [n][hw][3] -> fp32 [n][3][hw].  The block's 3 * 1024 source bytes are read as aligned 32-bit words into shared
// memory (the first and last word may hold bytes of a neighbouring pixel range: a 4-byte-aligned word that holds a
// byte of the frame never leaves the memory page holding that byte), so loads are coalesced whatever the source
// alignment (a 480p row is 2562 bytes).  Each thread then writes 4 consecutive pixels of each plane, as one float4
// where the plane address is 16-byte aligned.
__global__ void __launch_bounds__(kIngestThreads)
image_from_bgr8_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int hw, float m0, float m1, float m2) {
  __shared__ uint32_t words[kIngestPx * 3 / 4 + 2];
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * kIngestPx;
  const int np = min(kIngestPx, hw - p0);
  const uint8_t* s = src + (static_cast<size_t>(n) * hw + p0) * 3;
  const int mis = static_cast<int>(reinterpret_cast<uintptr_t>(s) & 3);
  const uint32_t* ws = reinterpret_cast<const uint32_t*>(s - mis);
  const int nw = (mis + 3 * np + 3) >> 2;
  for (int i = threadIdx.x; i < nw; i += kIngestThreads) words[i] = __ldg(ws + i);
  __syncthreads();
  const uint8_t* b = reinterpret_cast<const uint8_t*>(words) + mis;
  const int px = 4 * threadIdx.x;
  if (px >= np) return;
  const int cnt = min(4, np - px);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float mean = ch == 0 ? m0 : ch == 1 ? m1 : m2;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < cnt ? __fsub_rn(__uint2float_rn(b[3 * (px + j) + ch]), mean) : 0.f;
    float* d = dst + (static_cast<size_t>(n) * 3 + ch) * hw + p0 + px;
    if (cnt == 4 && (reinterpret_cast<uintptr_t>(d) & 15) == 0) {
      *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
      for (int j = 0; j < cnt; ++j) d[j] = v[j];
    }
  }
}

// Per-frame max and smallest non-zero byte of a uint8 mask, as stats[2n] = max, stats[2n+1] = 256 - smallest non-zero
// byte (0 when the frame is all zero), both by atomicMax into a zeroed workspace.  Word loads as above.
__global__ void __launch_bounds__(kIngestThreads)
label_stats_kernel(const uint8_t* __restrict__ src, uint32_t* __restrict__ stats, int hw) {
  const int n = blockIdx.y;
  const int b0 = blockIdx.x * kStatsBytes;
  const int nb = min(kStatsBytes, hw - b0);
  const uint8_t* s = src + static_cast<size_t>(n) * hw + b0;
  const int mis = static_cast<int>(reinterpret_cast<uintptr_t>(s) & 3);
  const uint32_t* ws = reinterpret_cast<const uint32_t*>(s - mis);
  const int nw = (mis + nb + 3) >> 2;
  uint32_t mx = 0, inv_min = 0;
  for (int i = threadIdx.x; i < nw; i += kIngestThreads) {
    const uint32_t word = __ldg(ws + i);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int off = 4 * i + k - mis;
      const uint32_t v = (word >> (8 * k)) & 255u;
      if (off >= 0 && off < nb && v != 0) {
        mx = max(mx, v);
        inv_min = max(inv_min, 256u - v);
      }
    }
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  inv_min = __reduce_max_sync(0xffffffffu, inv_min);
  if ((threadIdx.x & 31) == 0 && inv_min != 0) {
    atomicMax(stats + 2 * n, mx);
    atomicMax(stats + 2 * n + 1, inv_min);
  }
}

// stats[2n+1] <- 1 when every byte of frame n is 0 or its max (the normalised mask is all 0 / 1), else 0.
__global__ void label_flags_kernel(uint32_t* __restrict__ stats, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t inv_min = stats[2 * i + 1];
  stats[2 * i + 1] = inv_min == 0 || 256u - inv_min == stats[2 * i] ? 1u : 0u;
}

// uint8 [n][hw] -> fp32 [n][hw], v / max(float(frame max), 1e-8f); four bytes -> one float4 per thread.
__global__ void __launch_bounds__(kIngestThreads)
label_from_u8_kernel(const uint8_t* __restrict__ src, const uint32_t* __restrict__ stats, float* __restrict__ dst, int hw) {
  const int n = blockIdx.y;
  const int p = blockIdx.x * kIngestPx + 4 * threadIdx.x;
  if (p >= hw) return;
  const int cnt = min(4, hw - p);
  const float denom = fmaxf(__uint2float_rn(__ldg(stats + 2 * n)), 1e-8f);
  const uint8_t* s = src + static_cast<size_t>(n) * hw + p;
  float* d = dst + static_cast<size_t>(n) * hw + p;
  uint8_t b[4] = {0, 0, 0, 0};
  if (cnt == 4 && (reinterpret_cast<uintptr_t>(s) & 3) == 0) {
    const uint32_t word = __ldg(reinterpret_cast<const uint32_t*>(s));
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = static_cast<uint8_t>(word >> (8 * j));
  } else {
    for (int j = 0; j < cnt; ++j) b[j] = __ldg(s + j);
  }
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = __fdiv_rn(__uint2float_rn(b[j]), denom);
  if (cnt == 4 && (reinterpret_cast<uintptr_t>(d) & 15) == 0) {
    *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    for (int j = 0; j < cnt; ++j) d[j] = v[j];
  }
}

// uint8 id maps [n][hw] -> fp32 [n][hw] labels (label_of_id); four bytes -> one float4 per thread.
__global__ void __launch_bounds__(kIngestThreads)
labels_from_ids_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int hw, uint32_t object) {
  const int n = blockIdx.y;
  const int p = blockIdx.x * kIngestPx + 4 * threadIdx.x;
  if (p >= hw) return;
  const int cnt = min(4, hw - p);
  const uint8_t* s = src + static_cast<size_t>(n) * hw + p;
  float* d = dst + static_cast<size_t>(n) * hw + p;
  uint8_t b[4] = {0, 0, 0, 0};
  if (cnt == 4 && (reinterpret_cast<uintptr_t>(s) & 3) == 0) {
    const uint32_t word = __ldg(reinterpret_cast<const uint32_t*>(s));
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = static_cast<uint8_t>(word >> (8 * j));
  } else {
    for (int j = 0; j < cnt; ++j) b[j] = __ldg(s + j);
  }
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = label_of_id(b[j], object);
  if (cnt == 4 && (reinterpret_cast<uintptr_t>(d) & 15) == 0) {
    *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    for (int j = 0; j < cnt; ++j) d[j] = v[j];
  }
}

}  // namespace osvos

using namespace osvos;

#define OSVOS_CHECK_FRAME_DIMS(n, h, w) OSVOS_CHECK_ARG(n > 0 && n < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768)

extern "C" int osvos_image_from_bgr8(const uint8_t* src, float* dst, int n, int h, int w, float mean_b, float mean_g,
                                     float mean_r, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && dst != nullptr);
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  const int hw = h * w;
  const dim3 grid((hw + kIngestPx - 1) / kIngestPx, n);
  image_from_bgr8_kernel<<<grid, kIngestThreads, 0, static_cast<cudaStream_t>(stream_)>>>(src, dst, hw, mean_b, mean_g,
                                                                                           mean_r);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_label_stats_u8(const uint8_t* src, uint32_t* stats, int n, int h, int w, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && stats != nullptr);
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int hw = h * w;
  OSVOS_CHECK_CUDA(cudaMemsetAsync(stats, 0, sizeof(uint32_t) * 2 * n, stream));
  label_stats_kernel<<<dim3((hw + kStatsBytes - 1) / kStatsBytes, n), kIngestThreads, 0, stream>>>(src, stats, hw);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  label_flags_kernel<<<(n + 255) / 256, 256, 0, stream>>>(stats, n);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_label_from_u8(const uint8_t* src, const uint32_t* stats, float* dst, int n, int h, int w,
                                   osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && stats != nullptr && dst != nullptr);
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  const int hw = h * w;
  label_from_u8_kernel<<<dim3((hw + kIngestPx - 1) / kIngestPx, n), kIngestThreads, 0,
                         static_cast<cudaStream_t>(stream_)>>>(src, stats, dst, hw);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_affine_warp_u8(const uint8_t* image_src, const uint8_t* label_src, const uint32_t* label_stats,
                                    float* image_dst, float* label_dst, const double* inv_matrices_host,
                                    const int* flips_host, int n, int h, int w, float mean_b, float mean_g, float mean_r,
                                    osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(inv_matrices_host != nullptr && (image_src != nullptr || label_src != nullptr));
  OSVOS_CHECK_ARG((image_src == nullptr) == (image_dst == nullptr));
  OSVOS_CHECK_ARG((label_src == nullptr) == (label_dst == nullptr) && (label_src == nullptr) == (label_stats == nullptr));
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (image_src != nullptr) {
    const int st = launch_affine_warp(WarpSrcBgr8{image_src, h, w, mean_b, mean_g, mean_r}, image_dst,
                                      inv_matrices_host, flips_host, n, 3, h, w, OSVOS_WARP_CUBIC, stream);
    if (st != OSVOS_OK) return st;
  }
  if (label_src != nullptr) {
    return launch_affine_warp(WarpSrcLabel8{label_src, label_stats, h, w}, label_dst, inv_matrices_host, flips_host, n,
                              1, h, w, OSVOS_WARP_CUBIC, stream);
  }
  return OSVOS_OK;
}

// osvos_affine_warp_u8 over a batch gathered from a device-resident store: output sample i is store frame
// index_host[i].  The indices travel in the kernel's parameter table, so the gather costs no copy.
extern "C" int osvos_affine_warp_u8_indexed(const uint8_t* image_store, const uint8_t* label_store,
                                            const uint32_t* label_stats, float* image_dst, float* label_dst,
                                            const int* index_host, const double* inv_matrices_host,
                                            const int* flips_host, int n, int n_store, int h, int w, float mean_b,
                                            float mean_g, float mean_r, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(index_host != nullptr && inv_matrices_host != nullptr);
  OSVOS_CHECK_ARG(image_store != nullptr || label_store != nullptr);
  OSVOS_CHECK_ARG((image_store == nullptr) == (image_dst == nullptr));
  OSVOS_CHECK_ARG((label_store == nullptr) == (label_dst == nullptr) &&
                  (label_store == nullptr) == (label_stats == nullptr));
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  OSVOS_CHECK_ARG(n_store > 0);
  for (int i = 0; i < n; ++i) OSVOS_CHECK_ARG(index_host[i] >= 0 && index_host[i] < n_store);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (image_store != nullptr) {
    const int st = launch_affine_warp(WarpSrcBgr8{image_store, h, w, mean_b, mean_g, mean_r}, image_dst,
                                      inv_matrices_host, flips_host, n, 3, h, w, OSVOS_WARP_CUBIC, stream, index_host);
    if (st != OSVOS_OK) return st;
  }
  if (label_store != nullptr) {
    return launch_affine_warp(WarpSrcLabel8{label_store, label_stats, h, w}, label_dst, inv_matrices_host, flips_host,
                              n, 1, h, w, OSVOS_WARP_CUBIC, stream, index_host);
  }
  return OSVOS_OK;
}

extern "C" int osvos_labels_from_ids(const uint8_t* ids, float* dst, int n, int h, int w, int object,
                                     osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(ids != nullptr && dst != nullptr && object >= 0 && object < 255);
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  const int hw = h * w;
  labels_from_ids_kernel<<<dim3((hw + kIngestPx - 1) / kIngestPx, n), kIngestThreads, 0,
                           static_cast<cudaStream_t>(stream_)>>>(ids, dst, hw, static_cast<uint32_t>(object));
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// The id mode of osvos_affine_warp_u8 (index_host == NULL) and osvos_affine_warp_u8_indexed: the same matrices, flips
// and nearest fixed-point walk, with the label of each sampled id.
extern "C" int osvos_affine_warp_ids(const uint8_t* ids_store, float* label_dst, const int* index_host,
                                     const double* inv_matrices_host, const int* flips_host, int n, int n_store, int h,
                                     int w, int object, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(ids_store != nullptr && label_dst != nullptr && inv_matrices_host != nullptr);
  OSVOS_CHECK_ARG(object >= 0 && object < 255);
  OSVOS_CHECK_FRAME_DIMS(n, h, w);
  if (index_host != nullptr) {
    OSVOS_CHECK_ARG(n_store > 0);
    for (int i = 0; i < n; ++i) OSVOS_CHECK_ARG(index_host[i] >= 0 && index_host[i] < n_store);
  }
  return launch_affine_warp(WarpSrcIds8{ids_store, h, w, static_cast<uint32_t>(object)}, label_dst, inv_matrices_host,
                            flips_host, n, 1, h, w, OSVOS_WARP_NEAREST, static_cast<cudaStream_t>(stream_),
                            index_host);
}

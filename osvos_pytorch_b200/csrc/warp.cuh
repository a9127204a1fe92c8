// ScaleNRotate + RandomHorizontalFlip gather (reference dataloaders/custom_transforms.py:7-54, :87-100), shared by the
// fp32 entry point (augment.cu) and the uint8 one that reads decoded frames (frames.cu).  A restatement of OpenCV's
// warpAffine: fixed-point coordinates, 1/32-pixel bicubic table with A = -0.75, BORDER_CONSTANT 0.  The kernel is
// templated on where a tap's value comes from; everything after the load is the same code for every source, so a
// source that produces the same fp32 value as a stored fp32 tensor gives a bit-identical output.
#pragma once
#include "common.cuh"

namespace osvos {

constexpr int kWarpMaxSamples = 32;
// Per-launch host data, passed by value as a __grid_constant__ parameter (1,792 bytes): no device table, no copy.
// src[s] is the source sample that destination slot sample0 + s reads (and whose mask mode it uses).
struct WarpTable {
  double m[kWarpMaxSamples][6];
  int flip[kWarpMaxSamples];
  int src[kWarpMaxSamples];
};
static_assert(sizeof(WarpTable) == 1792, "WarpTable is a kernel parameter; keep it well inside the 4 KB limit");

__device__ __forceinline__ void cubic_coeffs(float x, float* c) {
  const float A = -0.75f;
  c[0] = ((A * (x + 1.f) - 5.f * A) * (x + 1.f) + 8.f * A) * (x + 1.f) - 4.f * A;
  c[1] = ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f;
  c[2] = ((A + 2.f) * (1.f - x) - (A + 3.f)) * (1.f - x) * (1.f - x) + 1.f;
  c[3] = 1.f - c[0] - c[1] - c[2];
}

// fp32 planes [n][c][h][w].
struct WarpSrcF32 {
  const float* p;
  int c, h, w;
  struct Sample {
    const float* base;
    size_t plane;
    int w;
    __device__ __forceinline__ float operator()(int ch, int y, int x) const {
      return __ldg(base + ch * plane + static_cast<size_t>(y) * w + x);
    }
  };
  __device__ __forceinline__ int mode(int, int m) const { return m; }
  __device__ __forceinline__ Sample sample(int s) const {
    const size_t plane = static_cast<size_t>(h) * w;
    return {p + static_cast<size_t>(s) * c * plane, plane, w};
  }
};

// The ingest value of a decoded BGR frame [n][h][w][3] uint8: float(v) - mean[ch], one fp32 rounding
// (osvos_image_from_bgr8).
struct WarpSrcBgr8 {
  const uint8_t* p;
  int h, w;
  float m0, m1, m2;
  struct Sample {
    const uint8_t* base;
    int w;
    float m0, m1, m2;
    __device__ __forceinline__ float operator()(int ch, int y, int x) const {
      const float v = __uint2float_rn(__ldg(base + (static_cast<size_t>(y) * w + x) * 3 + ch));
      return __fsub_rn(v, ch == 0 ? m0 : ch == 1 ? m1 : m2);
    }
  };
  __device__ __forceinline__ int mode(int, int m) const { return m; }
  __device__ __forceinline__ Sample sample(int s) const {
    return {p + static_cast<size_t>(s) * h * w * 3, w, m0, m1, m2};
  }
};

// The ingest value of a uint8 mask [n][h][w]: float(v) / max(float(frame max), 1e-8f) (osvos_label_from_u8).  The
// interpolation is chosen per sample from the binary flag of osvos_label_stats_u8: nearest for a 0/1 mask, cubic
// otherwise (custom_transforms.py:46-49).
struct WarpSrcLabel8 {
  const uint8_t* p;
  const uint32_t* stats;  // [n][2] = {max, binary}
  int h, w;
  struct Sample {
    const uint8_t* base;
    float denom;
    int w;
    __device__ __forceinline__ float operator()(int, int y, int x) const {
      return __fdiv_rn(__uint2float_rn(__ldg(base + static_cast<size_t>(y) * w + x)), denom);
    }
  };
  __device__ __forceinline__ int mode(int s, int) const {
    return __ldg(stats + 2 * s + 1) ? OSVOS_WARP_NEAREST : OSVOS_WARP_CUBIC;
  }
  __device__ __forceinline__ Sample sample(int s) const {
    return {p + static_cast<size_t>(s) * h * w, fmaxf(__uint2float_rn(__ldg(stats + 2 * s)), 1e-8f), w};
  }
};

// The label of a DAVIS-2017 object-id byte: -1 for 255 (void), 1 for an object (1..254, or == object when object != 0),
// 0 else (osvos_labels_from_ids).
__device__ __forceinline__ float label_of_id(uint32_t v, uint32_t object) {
  return v == 255u ? -1.f : (object != 0u ? v == object : v != 0u) ? 1.f : 0.f;
}

// uint8 id maps [n][h][w], always sampled nearest (out-of-frame samples are 0 like the mask's).
struct WarpSrcIds8 {
  const uint8_t* p;
  int h, w;
  uint32_t object;
  struct Sample {
    const uint8_t* base;
    int w;
    uint32_t object;
    __device__ __forceinline__ float operator()(int, int y, int x) const {
      return label_of_id(__ldg(base + static_cast<size_t>(y) * w + x), object);
    }
  };
  __device__ __forceinline__ int mode(int, int) const { return OSVOS_WARP_NEAREST; }
  __device__ __forceinline__ Sample sample(int s) const { return {p + static_cast<size_t>(s) * h * w, w, object}; }
};

template <class Src>
__global__ void __launch_bounds__(256)
affine_warp_kernel(const Src src, float* __restrict__ dst, const __grid_constant__ WarpTable t, int sample0, int c, int h,
                   int w, int mode) {
  const int s = blockIdx.z;
  const int y = blockIdx.y;
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= w) return;
  const double* m = t.m[s];
  const int flip = t.flip[s];
  const int si = t.src[s];
  mode = src.mode(si, mode);
  const int round_delta = mode == OSVOS_WARP_NEAREST ? 512 : 16;
  const int X0 = __double2int_rn((m[1] * y + m[2]) * 1024.0) + round_delta;
  const int Y0 = __double2int_rn((m[4] * y + m[5]) * 1024.0) + round_delta;
  const int Xf = X0 + __double2int_rn(m[0] * x * 1024.0);
  const int Yf = Y0 + __double2int_rn(m[3] * x * 1024.0);
  const size_t plane = static_cast<size_t>(h) * w;
  const typename Src::Sample sp = src.sample(si);
  float* dbase = dst + static_cast<size_t>(sample0 + s) * c * plane + static_cast<size_t>(y) * w + x;
  if (mode == OSVOS_WARP_NEAREST) {
    const int sx = Xf >> 10, sy = Yf >> 10;
    const bool in = sx >= 0 && sx < w && sy >= 0 && sy < h;
    const int ux = flip ? w - 1 - sx : sx;
    for (int ch = 0; ch < c; ++ch) dbase[ch * plane] = in ? sp(ch, sy, ux) : 0.f;
    return;
  }
  const int X = Xf >> 5, Y = Yf >> 5;
  const int sx = (X >> 5) - 1, sy = (Y >> 5) - 1;
  float cx[4], cy[4];
  cubic_coeffs(static_cast<float>(X & 31) * (1.f / 32.f), cx);
  cubic_coeffs(static_cast<float>(Y & 31) * (1.f / 32.f), cy);
  for (int ch = 0; ch < c; ++ch) {
    float sum = 0.f;
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
      const int yy = sy + ky;
      if (yy < 0 || yy >= h) continue;
#pragma unroll
      for (int kx = 0; kx < 4; ++kx) {
        const int xx = sx + kx;
        if (xx < 0 || xx >= w) continue;
        const int ux = flip ? w - 1 - xx : xx;
        sum += sp(ch, yy, ux) * (cy[ky] * cx[kx]);
      }
    }
    dbase[ch * plane] = sum;
  }
}

// Enqueues the warp of n samples in chunks of kWarpMaxSamples (the matrices travel as a kernel parameter).  Output
// sample i reads source sample index_host[i], or sample i when index_host is NULL.
template <class Src>
int launch_affine_warp(const Src& src, float* dst, const double* inv_matrices_host, const int* flips_host, int n, int c,
                       int h, int w, int mode, cudaStream_t stream, const int* index_host = nullptr) {
  for (int s0 = 0; s0 < n; s0 += kWarpMaxSamples) {
    const int cnt = n - s0 < kWarpMaxSamples ? n - s0 : kWarpMaxSamples;
    WarpTable t;
    for (int i = 0; i < cnt; ++i) {
      for (int k = 0; k < 6; ++k) t.m[i][k] = inv_matrices_host[static_cast<size_t>(s0 + i) * 6 + k];
      t.flip[i] = flips_host ? flips_host[s0 + i] : 0;
      t.src[i] = index_host ? index_host[s0 + i] : s0 + i;
    }
    const dim3 grid((w + 255) / 256, h, cnt);
    affine_warp_kernel<Src><<<grid, 256, 0, stream>>>(src, dst, t, s0, c, h, w, mode);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  return OSVOS_OK;
}

}  // namespace osvos

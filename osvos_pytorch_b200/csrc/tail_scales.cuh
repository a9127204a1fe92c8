// Host-side geometry and forward grid shared by the two side-branch tails (tail.cu, tail_general.cu).
#pragma once
#include "common.cuh"

namespace osvos {

// Scale k's side map is the input after k + 1 ceil-mode 2x2 poolings (hk x wk); its deconvolution has stride
// s = 2^(k+1) and kernel 2s, and center_crop takes floor(d/2) rows / columns off its top / left
// (layers/osvos_layers.py:52-56).
struct TailGeometry {
  int hk, wk, s, top, left;
};
static inline TailGeometry tail_geometry(int k, int h, int w) {
  int hk = h, wk = w;
  for (int i = 0; i <= k; ++i) hk = (hk + 1) / 2, wk = (wk + 1) / 2;
  const int s = 2 << k;
  return {hk, wk, s, ((hk + 1) * s - h) / 2, ((wk + 1) * s - w) / 2};
}

// the forward tails' grid: one output row per block iteration, at most 8 blocks per SM
static inline int tail_fwd_blocks(int n, int h) {
  size_t blocks = static_cast<size_t>(n) * h;
  const size_t cap = static_cast<size_t>(device_sm_count()) * 8;
  return static_cast<int>(blocks > cap ? cap : blocks);
}

}  // namespace osvos

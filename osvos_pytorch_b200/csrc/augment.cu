// Device-side ScaleNRotate + RandomHorizontalFlip (reference dataloaders/custom_transforms.py:7-54, :87-100) on fp32
// tensors: one gather kernel per tensor (warp.cuh).  HBM-bound: every destination pixel reads a 4x4 (cubic) or 1x1
// (nearest) source window through L1/L2; stores are coalesced along x.
#include "warp.cuh"

using namespace osvos;

extern "C" int osvos_affine_warp(const float* src, float* dst, const double* inv_matrices_host, const int* flips_host,
                                 int n, int c, int h, int w, int mode, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && dst != nullptr && src != dst && inv_matrices_host != nullptr);
  OSVOS_CHECK_ARG(n > 0 && c > 0 && h > 0 && w > 0 && h < 32768 && w < 32768);
  OSVOS_CHECK_ARG(mode == OSVOS_WARP_CUBIC || mode == OSVOS_WARP_NEAREST);
  return launch_affine_warp(WarpSrcF32{src, c, h, w}, dst, inv_matrices_host, flips_host, n, c, h, w, mode,
                            static_cast<cudaStream_t>(stream_));
}

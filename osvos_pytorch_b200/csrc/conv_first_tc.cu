// conv1_1 (3 -> 64 channels, 3x3, pad 1) + bias + ReLU on the tensor cores.
//
// K = 27 is too small for TMA-fed operands (and the frame is NCHW fp32), so the im2col A tile is BUILT in
// shared memory by warpgroup 0 straight from the caller's frame: row m = pixel, k = ci*9 + 3r + s,
// split into bf16 hi / lo, written in the canonical K-major SWIZZLE_128B layout (16-byte chunk j of row m
// lands at chunk j ^ (m & 7)).  Only k < 32 is ever written or read: two wgmma K-steps x three passes per
// 64-row half of a 128-pixel tile.  The 64 x 27 weight matrix is converted once per CTA into the same
// layout (B operand, resident).  Warpgroups 1 and 2 issue the wgmma for the two halves and run the shared
// conv epilogue (bias, ReLU, split-bf16 act store; staged through shared memory and stored with TMA when the output
// planes allow it).  Generic-proxy smem writes are made visible to the
// tensor core with fence.proxy.async before the mbarrier arrive.
//
// Replaces stages[0][0..1] of the reference (networks/vgg_osvos.py:61,142-143).
#include <string.h>

#include "conv_common.cuh"

namespace osvos {

constexpr int kFirstStages = 3;
constexpr int kFirstStageBytes = 2 * kABytes;           // hi + lo planes of the A tile (128 rows x 128 B each)
constexpr int kFirstBBytes = 2 * 64 * 128;              // hi + lo planes of the weights (64 rows x 128 B)
template <bool STAGED>
constexpr int kFirstSmem = kFirstStages * kFirstStageBytes + kFirstBBytes + (STAGED ? 2 * kStageBoxBytes : 0) + 1024 + 256;

template <int PLANES, bool STAGED>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_first_tc_kernel(const float* __restrict__ x, const float* __restrict__ wgt, const __grid_constant__ OutMaps out,
                     const ConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_b = smem + kFirstStages * kFirstStageBytes;
  uint8_t* smem_stage = smem_b + kFirstBBytes;   // STAGED: one staging box per consumer warpgroup
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_stage + (STAGED ? 2 * kStageBoxBytes : 0));
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kFirstStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kFirstStages; ++i) {
      mbar_init(&full_bar[i], 128);
      mbar_init(&empty_bar[i], 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  // PDL: the weights may have been rewritten by the previous kernel of the stream (the optimizer step), so even
  // the resident B operand is built after the wait; only barrier init overlaps its tail.
  pdl_wait();
  pdl_launch_dependents();
  // resident B operand: rows = co, k = ci*9 + 3r + s (the OIHW flattening), chunks 0..3 (k < 32)
  for (int i = threadIdx.x; i < 64 * 4; i += kConvThreads) {
    const int co = i >> 2, chunk = i & 3;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int k0 = chunk * 8 + 2 * t;
      const float v0 = k0 < 27 ? wgt[co * 27 + k0] : 0.f;
      const float v1 = k0 + 1 < 27 ? wgt[co * 27 + k0 + 1] : 0.f;
      __nv_bfloat16 h0, l0, h1, l1;
      split_bf16(v0, h0, l0);
      split_bf16(v1, h1, l1);
      hi[t] = pack_bf16x2(h0, h1);
      lo[t] = pack_bf16x2(l0, l1);
    }
    *reinterpret_cast<uint4*>(smem_b + sw128_offset(co, chunk)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(smem_b + 64 * 128 + sw128_offset(co, chunk)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp >= 4) {
    // -------------------------------------------------------------- consumer warpgroups: wgmma + epilogue
    const int wg = (warp - 4) >> 2, wl = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const uint64_t db_hi = make_smem_desc(smem_b, 16, 1024, kDescSW128);
    const uint64_t db_lo = db_hi + ((64 * 128) >> 4);
    int stage = 0;
    uint32_t phase = 0;
    float acc[32];
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t da_hi = make_smem_desc(smem + stage * kFirstStageBytes + wg * 64 * 128, 16, 1024, kDescSW128);
      const uint64_t da_lo = da_hi + (kABytes >> 4);
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (PLANES == 2) {
          wgmma_bf16<64>(acc, da_lo + 2 * k, db_hi + 2 * k, 1);
          wgmma_bf16<64>(acc, da_hi + 2 * k, db_lo + 2 * k, 1);
        }
        wgmma_bf16<64>(acc, da_hi + 2 * k, db_hi + 2 * k, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      if (leader) mbar_arrive(&empty_bar[stage]);
      if (++stage == kFirstStages) {
        stage = 0;
        phase ^= 1;
      }
      if constexpr (STAGED)
        conv_epilogue_staged(p, out, acc, tile, wg, wl, lane, smem_stage + wg * kStageBoxBytes, 1 + wg, leader);
      else
        conv_epilogue<64, false>(p, acc, tile, wg, wl, lane);
    }
    if (STAGED && leader) bulk_wait_group<0>();
  } else {
    // ------------------------------------------------------------- A builders (warpgroup 0: one pixel per thread)
    const int row = threadIdx.x;  // GEMM row = pixel of the tile
    const int ly = row / kTileW, lx = row % kTileW;
    int stage = 0;
    uint32_t phase = 0;
    const size_t plane_sz = static_cast<size_t>(p.h) * p.w;
    // Register double buffering: the 27 taps of the NEXT tile are requested before the current tile is converted and
    // written, so the global-load latency overlaps the shared-memory work and the wait for a free stage.
    auto load_tile = [&](int tile, float (&v)[27]) {
      int nb, tx, ty, img;
      decode_tile(p, tile, nb, tx, ty, img);
      const int y = ty * kTileH + ly, xx = tx * kTileW + lx;
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float* pl = x + (static_cast<size_t>(img) * 3 + ci) * plane_sz;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const int iy = y + r - 1;
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            const int ix = xx + s - 1;
            v[ci * 9 + r * 3 + s] =
                (iy >= 0 && iy < p.h && ix >= 0 && ix < p.w) ? __ldg(pl + static_cast<size_t>(iy) * p.w + ix) : 0.f;
          }
        }
      }
    };
    float vn[27];
    if (static_cast<int>(blockIdx.x) < p.total_tiles) load_tile(blockIdx.x, vn);
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      float v[32];
#pragma unroll
      for (int k = 0; k < 27; ++k) v[k] = vn[k];
#pragma unroll
      for (int k = 27; k < 32; ++k) v[k] = 0.f;
      if (tile + static_cast<int>(gridDim.x) < p.total_tiles) load_tile(tile + gridDim.x, vn);
      mbar_wait(&empty_bar[stage], phase ^ 1);
      uint8_t* st = smem + stage * kFirstStageBytes;
#pragma unroll
      for (int chunk = 0; chunk < 4; ++chunk) {
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          __nv_bfloat16 h0, l0, h1, l1;
          split_bf16(v[chunk * 8 + 2 * t], h0, l0);
          split_bf16(v[chunk * 8 + 2 * t + 1], h1, l1);
          hi[t] = pack_bf16x2(h0, h1);
          lo[t] = pack_bf16x2(l0, l1);
        }
        *reinterpret_cast<uint4*>(st + sw128_offset(row, chunk)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        if (PLANES == 2)
          *reinterpret_cast<uint4*>(st + kABytes + sw128_offset(row, chunk)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
      }
      fence_proxy_async_smem();
      mbar_arrive(&full_bar[stage]);
      if (++stage == kFirstStages) {
        stage = 0;
        phase ^= 1;
      }
    }
  }
}

int conv_first_tc_launch(const float* x, const float* w_oihw, const float* bias, void* y_hi, void* y_lo, int n, int h,
                         int w, int flags, cudaStream_t stream) {
  osvos_conv3x3_args a;
  memset(&a, 0, sizeof(a));
  a.bias = bias;
  a.y_hi = y_hi;
  a.y_lo = (flags & OSVOS_FLAG_FAST) ? nullptr : y_lo;
  a.n = n;
  a.h = h;
  a.w = w;
  a.cin = 64;  // unused by the epilogue; keeps k_chunks well defined
  a.cout = 64;
  a.flags = flags;
  ConvParams p;
  fill_conv_params(p, &a, 64);
  const bool fast = (flags & OSVOS_FLAG_FAST) != 0;
  const bool staged = outputs_tma_aligned(&a);
  OutMaps out;
  if (staged) {
    const int rc = encode_output_maps(&out, &a);
    if (rc) return rc;
  } else {
    memset(&out, 0, sizeof(out));
  }
  auto kern = staged ? (fast ? conv_first_tc_kernel<1, true> : conv_first_tc_kernel<2, true>)
                     : (fast ? conv_first_tc_kernel<1, false> : conv_first_tc_kernel<2, false>);
  const int smem = staged ? kFirstSmem<true> : kFirstSmem<false>;
  static uint64_t attr_done[4] = {0, 0, 0, 0};   // per instantiation: bit d = device d has the shared-memory opt-in
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(kern, smem, &attr_done[(staged ? 2 : 0) + (fast ? 1 : 0)]));
  const int sms = device_sm_count();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  OSVOS_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kConvThreads), smem, stream, x, w_oihw, out, p));
  return OSVOS_OK;
}

}  // namespace osvos

// Stage 1 of the trunk as ONE kernel (inference): conv1_1 (3 -> 64, + bias + ReLU) computed INSIDE conv1_2's kernel,
// on the 18 x 10-pixel halo patch conv1_2 reads anyway, so that the 105 MB split-bf16 map between the two layers is
// never written to or read from memory.  Replaces stages[0] of the reference (networks/vgg_osvos.py:61,140-143: conv,
// ReLU, conv, ReLU) and the first max pool (:140) when the caller only needs the pooled output.
//
// conv1_2 part = conv3x3_halo_kernel<64, exact> (conv3x3_halo.cu): nine taps as nine wgmma descriptors into the halo
// patch, weight slabs streamed by TMA through a ring, N-concatenated split accumulator, epilogue with the fused 2 x 2
// max pool.  What changes is WHO fills the activation stage: not a TMA box but warps 1 .. 3 of the CTA, which evaluate
// conv1_1 (27 fp32 multiply-adds per output: two pixel rounds x 64 x 27 FMAs plus the shared-memory weight loads, some
// 4-5 k issue slots per builder warp and tile - about as long as the tile's wgmma time) for the 180 halo pixels of the
// NEXT tile while the consumer warpgroups run conv1_2 on the current one, apply bias and ReLU, ZERO
// the halo pixels that lie outside the image (they are conv1_2's zero padding, not conv1_1 evaluated outside the
// frame), split into hi / lo and write the rows exactly where the TMA box of the unfused kernel would have put them
// (generic-proxy writes + fence.proxy.async before the mbarrier arrive).
// The builders bound the kernel: on an H100 it measured slower than conv1_1 and conv1_2 as two kernels (553 vs 584
// frames/s at 480x854), so the engine uses it only with OSVOS_FUSE_STAGE1=1.
#include <stdlib.h>
#include <string.h>

#include "conv_common.cuh"

namespace osvos {

constexpr int kS1Pitch = 10;                                        // halo patch row pitch in pixels (packed rows)
constexpr int kS1HaloRows = kTileH + 2;                             // 18
constexpr int kS1HaloPx = kS1HaloRows * kS1Pitch;                   // 180 halo pixels per tile
constexpr int kS1APlane = (kS1HaloPx * 128 + 1023) / 1024 * 1024;   // 23552 B: one plane of one activation stage
constexpr int kS1AStage = 2 * kS1APlane;
constexpr int kS1AStages = 2;
constexpr int kS1BPlane = 64 * 128;                                 // conv1_2 weight slab, one plane (64 co x 64 ci)
constexpr int kS1BStage = 2 * kS1BPlane;
constexpr int kS1BStages = 5;
constexpr int kS1W1Bytes = (64 * 27 + 64) * 4;                      // conv1_1 weights + bias, fp32
constexpr int kS1Builders = 96;                                     // warps 1 .. 3
constexpr int kS1Smem = kS1AStages * kS1AStage + kS1BStages * kS1BStage + kS1W1Bytes + 1024 + 512;
static_assert(kS1Smem <= 227 * 1024, "stage-1 kernel exceeds the per-CTA shared memory");
static_assert(kS1Smem + 4096 < (1 << 18), "descriptor start-address field would overflow");

struct Stage1Params {
  const float* x;    // [n,3,h,w] fp32 frame
  const float* w1;   // conv1_1 weight [64,3,3,3]
  const float* b1;   // conv1_1 bias [64] or NULL
};

__global__ void __launch_bounds__(kConvThreads, 1)
conv_stage1_fused_kernel(const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                         const Stage1Params s1, const ConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + kS1AStages * kS1AStage;
  float* w1s = reinterpret_cast<float*>(smem_b + kS1BStages * kS1BStage);   // [64][27] weights, then [64] bias
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(w1s) + kS1W1Bytes);
  uint64_t* a_full = bars;                       // [2] builders -> consumers   (96 arrivals)
  uint64_t* a_empty = bars + 2;                  // [2] consumers -> builders   (one per consumer warpgroup)
  uint64_t* b_full = bars + 4;                   // [kS1BStages] TMA -> consumers
  uint64_t* b_empty = bars + 4 + kS1BStages;     // [kS1BStages] consumers -> TMA producer

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_w_hi);
    tma_prefetch_desc(&map_w_lo);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], kS1Builders);
      mbar_init(&a_empty[i], 2);
    }
    for (int i = 0; i < kS1BStages; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], 2);
    }
    fence_barrier_init();
  }
  pdl_wait();               // the frame / the weights may come from the previous kernel of the stream
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < 64 * 27 + 64; i += kConvThreads)
    w1s[i] = i < 64 * 27 ? __ldg(s1.w1 + i) : (s1.b1 ? __ldg(s1.b1 + i - 64 * 27) : 0.f);
  __syncthreads();

  if (warp == 0) {
    // ------------------------------------------------------------ TMA producer: conv1_2 weight slabs only
    if (elect_one()) {
      int b_stage = 0;
      uint32_t b_phase = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          mbar_wait(&b_empty[b_stage], b_phase ^ 1);
          uint8_t* st = smem_b + b_stage * kS1BStage;
          mbar_arrive_expect_tx(&b_full[b_stage], kS1BStage);
          tma_load_3d(&map_w_hi, &b_full[b_stage], st, 0, 0, tap);
          tma_load_3d(&map_w_lo, &b_full[b_stage], st + kS1BPlane, 0, 0, tap);
          if (++b_stage == kS1BStages) {
            b_stage = 0;
            b_phase ^= 1;
          }
        }
      }
    }
    __syncwarp();
  } else if (warp < 4) {
    // ------------------------------------------------------------ builders: conv1_1 of the halo patch -> activation stage
    const int t = threadIdx.x - 32;
    const size_t plane_sz = static_cast<size_t>(p.h) * p.w;
    int a_stage = 0;
    uint32_t a_phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int nb, tx, ty, img;
      decode_tile(p, tile, nb, tx, ty, img);
      mbar_wait(&a_empty[a_stage], a_phase ^ 1);   // conv1_2's MMAs of two tiles ago have read this stage
      uint8_t* st = smem_a + a_stage * kS1AStage;
      for (int pix = t; pix < kS1HaloPx; pix += kS1Builders) {
        const int hy = pix / kS1Pitch, hx = pix - hy * kS1Pitch;
        const int y = ty * kTileH - 1 + hy, xx = tx * kTileW - 1 + hx;
        const bool inside = y >= 0 && y < p.h && xx >= 0 && xx < p.w;
        float v[27];
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const float* pl = s1.x + (static_cast<size_t>(img) * 3 + ci) * plane_sz;
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const int iy = y + r - 1;
#pragma unroll
            for (int s = 0; s < 3; ++s) {
              const int ix = xx + s - 1;
              v[ci * 9 + r * 3 + s] =
                  (inside && iy >= 0 && iy < p.h && ix >= 0 && ix < p.w) ? __ldg(pl + static_cast<size_t>(iy) * p.w + ix) : 0.f;
            }
          }
        }
#pragma unroll 1
        for (int chunk = 0; chunk < 8; ++chunk) {    // 8 output channels = one 16-byte chunk of each plane's row
          float f[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int co = chunk * 8 + e;
            float acc = w1s[64 * 27 + co];
#pragma unroll
            for (int k = 0; k < 27; ++k) acc = fmaf(w1s[co * 27 + k], v[k], acc);
            f[e] = inside ? fmaxf(acc, 0.f) : 0.f;   // ReLU; halo pixels outside the frame are conv1_2's zero padding
          }
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) split_pack2(f[2 * e], f[2 * e + 1], hi[e], lo[e]);
          const uint32_t off = sw128_offset(pix, chunk);
          *reinterpret_cast<uint4*>(st + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(st + kS1APlane + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
      }
      fence_proxy_async_smem();
      mbar_arrive(&a_full[a_stage]);
      if (++a_stage == kS1AStages) {
        a_stage = 0;
        a_phase ^= 1;
      }
    }
  } else {
    // -------------------------------------------------- consumer warpgroups: conv1_2 (wgmma) + epilogue, 64 rows each
    const int wg = (warp - 4) >> 2, wl = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    constexpr uint64_t kDescA = desc_template(16, kS1Pitch * 128, kDescSW128);
    constexpr uint64_t kDescB = desc_template(16, 1024, kDescSW128);
    const uint32_t smem_a_u32 = smem_u32(smem_a) + wg * 8 * kS1Pitch * 128, smem_b_u32 = smem_u32(smem_b);
    float acc[64];
    int a_stage = 0, b_stage = 0;
    uint32_t a_phase = 0, b_phase = 0;
    StageRelease pending;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      mbar_wait(&a_full[a_stage], a_phase);
      const uint64_t da0 = kDescA | static_cast<uint64_t>((smem_a_u32 + a_stage * kS1AStage) >> 4);
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const uint32_t tap_off = static_cast<uint32_t>(((tap / 3) * kS1Pitch + (tap % 3)) * (128 >> 4));
        mbar_wait(&b_full[b_stage], b_phase);
        const uint64_t db_hi = kDescB | static_cast<uint64_t>((smem_b_u32 + b_stage * kS1BStage) >> 4);
        const uint64_t da_hi = da0 + tap_off;
        const uint64_t da_lo = da_hi + (kS1APlane >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
          wgmma_bf16<128>(acc, da_hi + 2 * k, db_hi + 2 * k, 1);   // [A_hi.B_hi | A_hi.B_lo]
          wgmma_bf16<64>(acc, da_lo + 2 * k, db_hi + 2 * k, 1);    // + A_lo.B_hi
        }
        wgmma_commit();
        wgmma_wait<1>();
        pending.release(leader);
        pending.bar_b = &b_empty[b_stage];
        if (tap == 8) pending.bar_a = &a_empty[a_stage];
        if (++b_stage == kS1BStages) {
          b_stage = 0;
          b_phase ^= 1;
        }
      }
      if (++a_stage == kS1AStages) {
        a_stage = 0;
        a_phase ^= 1;
      }
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      pending.release(leader);
      conv_epilogue<64, true, true>(p, acc, tile, wg, wl, lane);   // pooled / act output only
    }
  }
}

}  // namespace osvos

using namespace osvos;

extern "C" int osvos_stage1_fused(const osvos_stage1_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->x != nullptr && a->w1 != nullptr && a->w2_packed != nullptr);
  OSVOS_CHECK_ARG(a->n > 0 && a->h > 0 && a->w > 0 && a->h <= 65535 && a->n <= 65535);
  OSVOS_CHECK_ARG((a->y_hi != nullptr && a->y_lo != nullptr) || (a->pool_hi != nullptr && a->pool_lo != nullptr));
  OSVOS_CHECK_ARG((a->y_hi == nullptr) == (a->y_lo == nullptr) && (a->pool_hi == nullptr) == (a->pool_lo == nullptr));
  {
    const uintptr_t any = reinterpret_cast<uintptr_t>(a->y_hi) | reinterpret_cast<uintptr_t>(a->y_lo) |
                          reinterpret_cast<uintptr_t>(a->pool_hi) | reinterpret_cast<uintptr_t>(a->pool_lo);
    OSVOS_CHECK_ARG((any & 3) == 0);   // the epilogue stores bf16x2 words
    OSVOS_CHECK_ARG(((reinterpret_cast<uintptr_t>(a->b1) | reinterpret_cast<uintptr_t>(a->b2) |
                      reinterpret_cast<uintptr_t>(a->w2_packed)) & 15) == 0);
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  osvos_conv3x3_args c;
  memset(&c, 0, sizeof(c));
  c.w_packed = a->w2_packed;
  c.bias = a->b2;
  c.y_hi = a->y_hi;
  c.y_lo = a->y_lo;
  c.pool_hi = a->pool_hi;
  c.pool_lo = a->pool_lo;
  c.n = a->n, c.h = a->h, c.w = a->w, c.cin = 64, c.cout = 64;
  c.flags = OSVOS_FLAG_RELU;
  ConvParams p;
  fill_conv_params(p, &c, 64);
  CUtensorMap mw_hi, mw_lo;
  int rc = encode_weight_maps(&mw_hi, &mw_lo, &c, 64);
  if (rc) return rc;
  Stage1Params s1;
  s1.x = a->x;
  s1.w1 = a->w1;
  s1.b1 = a->b1;
  const int sms = device_sm_count();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  auto kern = conv_stage1_fused_kernel;
  static uint64_t attr_done = 0;
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(kern, kS1Smem, &attr_done));
  OSVOS_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kConvThreads), kS1Smem, stream, mw_hi, mw_lo, s1, p));
  return OSVOS_OK;
}

// Shared pieces of the wgmma implicit-GEMM convolution kernels (conv3x3_halo.cu, conv_first_tc.cu,
// conv_stage1_fused.cu): tile geometry, parameters, tile decode and the epilogue (accumulator registers ->
// bias / ReLU / mask / split-bf16 / pool / column sums -> global).
#pragma once
#include <stdlib.h>

#include "common.cuh"
#include "ptx.cuh"

namespace osvos {

constexpr int kTileW = 8;     // pixels per patch row  (= one 8-row swizzle atom)
constexpr int kTileH = 16;    // patch rows
constexpr int kBlockM = 128;  // kTileW * kTileH
constexpr int kBlockK = 64;   // channels per K block (128 B of bf16)
// Warp roles of the conv kernels: warpgroup 0 feeds shared memory (TMA producer warp, or the threads that build an
// operand), warpgroups 1 and 2 issue the wgmma for GEMM rows 0 .. 63 / 64 .. 127 of a tile and run its epilogue (or, in
// the halo kernel's ping-pong schedule, each takes every other tile whole).
constexpr int kConvThreads = 384;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KiB per plane

struct ConvParams {
  const float* bias;
  __nv_bfloat16* y_hi;
  __nv_bfloat16* y_lo;
  float* y_f32;
  const __nv_bfloat16* mask_hi;
  __nv_bfloat16* pool_hi;  // optional fused 2x2 ceil-mode max pool of the output
  __nv_bfloat16* pool_lo;
  float* colsum;           // optional fused per-channel sum of the output (bias gradient), atomically accumulated; with
                           // OSVOS_FLAG_DETERMINISTIC partial rows [pixel tile][half][warp][cout] written with plain stores
  int n, h, w, cin, cout;
  int tiles_x, tiles_y, n_blocks, total_tiles, k_chunks;
  int flags;
  // Timing ablations (OSVOS_ABLATE bit mask, diagnosis only - results are garbage): 1 = no weight TMA loads,
  // 2 = no activation TMA loads, 4 = no wgmma, 8 = no global stores in the epilogue, 16 = no epilogue at all.
  // 0 in production.
  int ablate;
};

__device__ __forceinline__ void decode_tile(const ConvParams& p, int tile, int& nb, int& tx, int& ty, int& img) {
  nb = tile % p.n_blocks;
  int m = tile / p.n_blocks;
  tx = m % p.tiles_x;
  m /= p.tiles_x;
  ty = m % p.tiles_y;
  img = m / p.tiles_y;
}

__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

// Two floats -> packed bf16x2 "hi" word (one F2FP) and the packed residual "lo" word: v ~= hi + lo.
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));            // upper half <- b, lower half <- a
  const float ra = a - __uint_as_float(hi << 16);
  const float rb = b - __uint_as_float(hi & 0xFFFF0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(rb), "f"(ra));
}

// The m64 half `wg` (0, 1) of a tile is GEMM rows 64 wg .. 64 wg + 63 of the 128-pixel tile, i.e. patch rows
// 8 wg .. 8 wg + 7; `acc` is a consumer warpgroup's accumulator for that half.  Its wgmma accumulator fragment (wgmma.cuh) gives thread (warp wl of the warpgroup, lane) the
// pixels (lx = lane / 4, ly = 8 wg + 2 wl) and (lx, ly + 1) - the two rows of a 2 x 2 pooling window - and the channel
// pairs 8j + 2 (lane % 4) + {0, 1}: the x partner of the window is lane ^ 4.
//
// The epilogue runs straight from those registers: bias, ReLU, ReLU mask of a later layer, fp32 / split-bf16 act output,
// fused 2 x 2 ceil-mode max pool and fused per-channel column sums (bias gradient).
// SPLIT_ACC: the accumulator holds 2 * BLOCK_N columns - [A_hi.B_hi | A_hi.B_lo] (+ A_lo.B_hi in the first half) from one
// N-concatenated wgmma - and the result is the sum of the two halves.
// LEAN: the plain-forward feature set only (bias, ReLU, split-bf16 act output and / or fused pool); the mask, fp32 output
// and column-sum code is not compiled in, which takes it out of the consumer warpgroups' instruction stream.
// Both forms compute every value with the same operations in the same order: their outputs are bit-identical.
// DET: the column sums go to partial rows (OSVOS_FLAG_DETERMINISTIC) instead of atomics.
template <int BLOCK_N, bool SPLIT_ACC, bool LEAN = false, bool DET = false>
__device__ __forceinline__ void conv_epilogue(const ConvParams& p, const float* acc, int tile, int wg, int wl, int lane) {
  if (p.ablate & 16) return;
  int nb, tx, ty, img;
  decode_tile(p, tile, nb, tx, ty, img);
  const int lx = lane >> 2;
  const int x = tx * kTileW + lx;
  const int y0 = ty * kTileH + wg * 8 + wl * 2;   // even: the top row of a pooling window
  const bool va = (y0 < p.h) && (x < p.w), vb = (y0 + 1 < p.h) && (x < p.w);
  const bool relu = (p.flags & OSVOS_FLAG_RELU) != 0;
  const bool masked = !LEAN && (p.flags & OSVOS_FLAG_RELU_MASK) != 0;
  const bool store_ok = !(p.ablate & 8);
  const size_t pix[2] = {(static_cast<size_t>(img) * p.h + y0) * p.w + x, (static_cast<size_t>(img) * p.h + y0 + 1) * p.w + x};
  const bool valid[2] = {va, vb};
  const int oh = (p.h + 1) >> 1, ow = (p.w + 1) >> 1;
  const bool pool_writer = va && !(lx & 1) && store_ok;
  const size_t opix = (static_cast<size_t>(img) * oh + (y0 >> 1)) * ow + (x >> 1);
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int c = 8 * j + 2 * (lane & 3);
    const int ch = nb * BLOCK_N + c;
    const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + ch)) : make_float2(0.f, 0.f);
    float f[2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float v = e ? b.y : b.x;
        v += acc[4 * j + 2 * h + e];
        if (SPLIT_ACC) v += acc[BLOCK_N / 2 + 4 * j + 2 * h + e];
        f[h][e] = relu ? fmaxf(v, 0.f) : v;
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!LEAN && masked && valid[h]) {
        const uint32_t m = __ldg(reinterpret_cast<const unsigned int*>(p.mask_hi + pix[h] * p.cout + ch));
        if (!(bf16_lo_to_float(m) > 0.f)) f[h][0] = 0.f;
        if (!(bf16_hi_to_float(m) > 0.f)) f[h][1] = 0.f;
      }
      if (valid[h] && store_ok) {
        if (!LEAN && p.y_f32) *reinterpret_cast<float2*>(p.y_f32 + pix[h] * p.cout + ch) = make_float2(f[h][0], f[h][1]);
        if (p.y_hi) {
          uint32_t hi, lo;
          split_pack2(f[h][0], f[h][1], hi, lo);
          *reinterpret_cast<uint32_t*>(p.y_hi + pix[h] * p.cout + ch) = hi;
          if (p.y_lo) *reinterpret_cast<uint32_t*>(p.y_lo + pix[h] * p.cout + ch) = lo;
        }
      }
    }
    if (!LEAN && p.colsum) {   // per-channel sum over the tile's valid pixels: the 8 x-lanes of a channel pair are lanes ^ 4, 8, 16
      float s0 = (va ? f[0][0] : 0.f) + (vb ? f[1][0] : 0.f);
      float s1 = (va ? f[0][1] : 0.f) + (vb ? f[1][1] : 0.f);
#pragma unroll
      for (int o = 4; o <= 16; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      }
      if (lane < 4) {
        if constexpr (DET) {   // one partial row per (pixel tile, m64 half, warp), reduced in order later
          const size_t prow = (static_cast<size_t>(tile / p.n_blocks) * 2 + wg) * 4 + wl;
          *reinterpret_cast<float2*>(p.colsum + prow * p.cout + ch) = make_float2(s0, s1);
        } else {
          atomicAdd(p.colsum + ch, s0);
          atomicAdd(p.colsum + ch + 1, s1);
        }
      }
    }
    if (p.pool_hi) {  // MaxPool2d(2, 2, ceil_mode=True); out-of-image members of the window are excluded
      float m0 = fmaxf(va ? f[0][0] : -INFINITY, vb ? f[1][0] : -INFINITY);
      float m1 = fmaxf(va ? f[0][1] : -INFINITY, vb ? f[1][1] : -INFINITY);
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 4));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 4));
      if (pool_writer) {
        uint32_t hi, lo;
        split_pack2(m0, m1, hi, lo);
        *reinterpret_cast<uint32_t*>(p.pool_hi + opix * p.cout + ch) = hi;
        if (p.pool_lo) *reinterpret_cast<uint32_t*>(p.pool_lo + opix * p.cout + ch) = lo;
      }
    }
  }
}

// ---- staged epilogue: registers -> shared memory -> TMA store (conv1_1) -------------------------------------------
// Per consumer warpgroup, one staging box: one plane of 64 channels of its m64 half (8 x 8 pixels, 64 rows of 128 B),
// SWIZZLE_128B like the tensor maps that store it.  A multiple of 1024 B, so consecutive boxes keep the swizzle phase.
constexpr int kStageBoxBytes = 64 * 64 * 2;

// Output tensor maps of the staged epilogue: {cout, w, h, n} with box {64, 8, 8, 1}.  The lo map of a hi-only output is
// left zeroed and never used.
struct OutMaps {
  CUtensorMap y_hi, y_lo;
};

// The plain forward epilogue of a 64-channel tile (bias, ReLU, split-bf16 act output) with the same operations in the
// same order as conv_epilogue<64, false>, so the outputs are bit-identical; only the route to global memory differs.  For
// each output plane the warpgroup writes its values into `box` (the 8 pixel rows of a warp store land in 8 different
// 16-byte swizzle slots: no bank conflicts), fences them to the async proxy, and one thread issues the TMA store, which
// drains while the next plane is computed or the next tile's MMAs run, instead of 4-byte stores that each cover a
// partial sector of 8 lines.  The box is rewritten only after the previous store has read it (wait_group.read), so the
// hi and lo planes take two rounds and the values are recomputed for the second: that costs a few ALU instructions and
// keeps the lo words out of the register file.  Edge tiles rely on TMA clipping the stores at the tensor bounds.  The
// caller waits for the stores (bulk_wait_group<0>) on `leader` before the kernel exits.
__device__ __forceinline__ void conv_epilogue_staged(const ConvParams& p, const OutMaps& maps, const float* acc, int tile,
                                                     int half, int wl, int lane, uint8_t* box, int bar_id, bool leader) {
  if (p.ablate & 16) return;
  int nb, tx, ty, img;
  decode_tile(p, tile, nb, tx, ty, img);
  const int lx = lane >> 2;
  const bool relu = (p.flags & OSVOS_FLAG_RELU) != 0;
  const bool store_ok = !(p.ablate & 8);
  const int planes = p.y_lo ? 2 : 1;
  const uint32_t act_row = smem_u32(box) + (wl * 2 * 8 + lx) * 128;   // pixel (lx, 2 wl); the row below is 8 rows on
  const uint32_t col = 4 * (lane & 3);
#pragma unroll 1
  for (int plane = 0; plane < planes; ++plane) {
    if (leader) bulk_wait_group_read<0>();
    named_bar_sync(bar_id, 128);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = nb * 64 + 8 * j + 2 * (lane & 3);
      const float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + ch)) : make_float2(0.f, 0.f);
      float f[2][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = e ? b.y : b.x;
          v += acc[4 * j + 2 * h + e];
          f[h][e] = relu ? fmaxf(v, 0.f) : v;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t hi, lo;
        split_pack2(f[h][0], f[h][1], hi, lo);
        st_shared_u32(act_row + h * 8 * 128 + ((j ^ lx) << 4) + col, plane ? lo : hi);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(bar_id, 128);
    if (leader && store_ok) {
      tma_store_4d(plane ? &maps.y_lo : &maps.y_hi, box, nb * 64, tx * kTileW, ty * kTileH + half * 8, img);
      bulk_commit_group();
    }
  }
}


// ---- host helpers shared by the launchers ------------------------------------------------
static inline void fill_conv_params(ConvParams& p, const osvos_conv3x3_args* a, int block_n) {
  p.bias = a->bias;
  p.y_hi = static_cast<__nv_bfloat16*>(a->y_hi);
  p.y_lo = static_cast<__nv_bfloat16*>(a->y_lo);
  p.y_f32 = a->y_f32;
  p.mask_hi = static_cast<const __nv_bfloat16*>(a->mask_hi);
  p.pool_hi = static_cast<__nv_bfloat16*>(a->pool_hi);
  p.pool_lo = static_cast<__nv_bfloat16*>(a->pool_lo);
  p.colsum = a->colsum;
  p.n = a->n;
  p.h = a->h;
  p.w = a->w;
  p.cin = a->cin;
  p.cout = a->cout;
  p.tiles_x = (a->w + kTileW - 1) / kTileW;
  p.tiles_y = (a->h + kTileH - 1) / kTileH;
  p.n_blocks = a->cout / block_n;
  p.total_tiles = p.tiles_x * p.tiles_y * a->n * p.n_blocks;
  p.k_chunks = a->cin / kBlockK;
  p.flags = a->flags;
  {
    static int ablate = -1;
    if (ablate < 0) {
      const char* e = getenv("OSVOS_ABLATE");
      ablate = e ? atoi(e) : 0;
    }
    p.ablate = ablate;
  }
}

// Packed weights [plane][tap][cout][cin] -> two 3-D maps with box {64, block_n, 1}.
static inline int encode_weight_maps(CUtensorMap* hi, CUtensorMap* lo, const osvos_conv3x3_args* a, int block_n) {
  const size_t plane = static_cast<size_t>(9) * a->cout * a->cin;  // elements
  const uint64_t dims[3] = {(uint64_t)a->cin, (uint64_t)a->cout, 9};
  const uint64_t strides[2] = {(uint64_t)a->cin * 2, (uint64_t)a->cout * a->cin * 2};
  const uint32_t box[3] = {kBlockK, (uint32_t)block_n, 1};
  const __nv_bfloat16* wp = static_cast<const __nv_bfloat16*>(a->w_packed);
  int rc = encode_tensor_map(hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, wp, dims, strides, box,
                             CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  return encode_tensor_map(lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 3, wp + plane, dims, strides, box,
                           CU_TENSOR_MAP_SWIZZLE_128B);
}

// TMA stores need 16-byte aligned bases (the row strides, multiples of cout * 2 B, are); the ABI promises only the
// 4-byte alignment of a channel pair, so launches with other outputs keep the direct-store epilogue.
static inline bool outputs_tma_aligned(const osvos_conv3x3_args* a) {
  return ((reinterpret_cast<uintptr_t>(a->y_hi) | reinterpret_cast<uintptr_t>(a->y_lo)) & 15) == 0;
}

static inline int encode_output_maps(OutMaps* m, const osvos_conv3x3_args* a) {
  memset(m, 0, sizeof(*m));
  const uint64_t c = a->cout;
  const uint64_t dims[4] = {c, (uint64_t)a->w, (uint64_t)a->h, (uint64_t)a->n};
  const uint64_t strides[3] = {c * 2, c * 2 * a->w, c * 2 * a->w * a->h};
  const uint32_t box[4] = {64, kTileW, kTileH / 2, 1};
  int rc = encode_tensor_map(&m->y_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4, a->y_hi, dims, strides, box,
                             CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc == OSVOS_OK && a->y_lo)
    rc = encode_tensor_map(&m->y_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4, a->y_lo, dims, strides, box,
                           CU_TENSOR_MAP_SWIZZLE_128B);
  return rc;
}

int conv_first_tc_launch(const float* x, const float* w_oihw, const float* bias, void* y_hi, void* y_lo, int n, int h,
                         int w, int flags, cudaStream_t stream);
int side_conv_dispatch(const osvos_conv3x3_args* a, cudaStream_t stream);
int side_conv_multi_dispatch(const osvos_conv3x3_args* const* args, int count, cudaStream_t stream);

}  // namespace osvos

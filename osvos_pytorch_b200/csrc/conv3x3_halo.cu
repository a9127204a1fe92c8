// 3x3 convolution as a wgmma implicit GEMM with HALO REUSE (sm_90a).
//
// GEMM view: M = 128 pixels of an 8 x 16 output tile, N = output channels, K = 9 taps x input channels.  The
// activation operand is loaded ONCE per (tile, 64-channel chunk) as the 18-row x 10-px halo patch (one TMA box,
// SWIZZLE_128B) and the nine taps are nine wgmma descriptors into it: tap (r, s) starts at smem row (r * kPitch + s);
// the 16 tile rows are sixteen 8-row swizzle groups at stride SBO = kPitch * 128 B.  That divides the activation
// traffic through L2 -> smem by ~6 relative to one shifted box per tap.  The weight slabs stream through their own,
// deeper ring (one stage per tap), and the next chunk's halo is prefetched while the current one is being consumed.
//
// kPitch is the smem row pitch in pixels: 10 packs the patch rows (1280 B); a tap descriptor then starts at any
// 128-byte row, which relies on the hardware applying the 128-byte swizzle to the absolute shared-memory address
// (the descriptor's base-offset field stays 0), as the TMA unit does when it writes the box.
//
// Precision: exact mode carries every operand as split bf16 (hi + lo) and sums A_hi.B_hi + A_hi.B_lo + A_lo.B_hi in
// fp32; fast mode uses the hi planes only.
#include "conv_common.cuh"

namespace osvos {

constexpr int kHaloRows = kTileH + 2;  // 18
constexpr int kPitch = kTileW + 2;     // 10: the halo patch's rows, packed

template <int BLOCK_N, int PLANES, bool SPLIT>
struct HaloCfg {
  static constexpr int kABoxBytes = kHaloRows * kPitch * 128;               // one plane, one chunk
  static constexpr int kAPlaneBytes = (kABoxBytes + 1023) / 1024 * 1024;    // keep 1 KiB alignment
  static constexpr int kAStageBytes = PLANES * kAPlaneBytes;
  static constexpr int kAStages = 2;
  static constexpr int kBPlaneBytes = BLOCK_N * 128;
  static constexpr int kBStageBytes = PLANES * kBPlaneBytes;
  static constexpr int kBudget = 225 * 1024 - kAStages * kAStageBytes;   // 227 KiB per CTA minus align/barriers
  static constexpr int kBStagesRaw = kBudget / kBStageBytes;
  static constexpr int kBStages = kBStagesRaw > 9 ? 9 : kBStagesRaw;
  // Exact mode with BLOCK_N <= 128: N-concatenated split-B.  The hi and lo weight planes are contiguous in the B
  // stage, so ONE wgmma of N = 2 * BLOCK_N computes [A_hi.B_hi | A_hi.B_lo] into two column halves of the
  // accumulator; with the N = BLOCK_N pass A_lo.B_hi that is 2 instructions per K step instead of 3.  The epilogue
  // adds the halves.
  static constexpr bool kSplitAcc = SPLIT;
  static_assert(!SPLIT || (PLANES == 2 && BLOCK_N <= 128), "split accumulators need two planes and 2 * BLOCK_N <= 256");
  static constexpr int kAccCols = kSplitAcc ? 2 * BLOCK_N : BLOCK_N;
  static constexpr int kAcc = kAccCols / 2;                                 // accumulator registers per consumer thread
  static constexpr int kSmemBytes = kAStages * kAStageBytes + kBStages * kBStageBytes + 1024 + 512;
  static_assert(kBStages >= 2, "weight ring too shallow");
  static_assert(kSmemBytes <= 227 * 1024, "more than the per-CTA shared memory of sm_90");
  static_assert(kSmemBytes + 4096 < (1 << 18), "descriptor start-address field would overflow");
  static_assert(kBStageBytes % 1024 == 0, "B stage must keep 1024-byte alignment");
};

// Two schedules for the consumer warpgroups 1 and 2:
//  - cooperative (PINGPONG = false): both take every tile, rows 0 .. 63 and 64 .. 127, and reach the epilogue together,
//    so the tensor pipe idles while they run it.
//  - ping-pong: the CTA's k-th tile goes to warpgroup k % 2, which computes all 128 rows as two m64 halves; one
//    warpgroup's epilogue runs while the other issues the next tile's MMAs.  Both read the ONE ring the producer fills in
//    tile order, each skipping the other's stages, and each stage is released by the one warpgroup that read it.  Named
//    barriers 1 and 2 hand the ring over in tile order: warpgroup k % 2 starts waiting on tile k's full barriers only
//    after tile k - 1's owner has passed its last full wait.  Without that, a warpgroup a whole ring round ahead of the
//    producer would pass a parity wait on a phase that has not happened yet.
template <int BLOCK_N, int PLANES, bool SPLIT, bool LEAN, bool PINGPONG, bool DET = false>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3x3_halo_kernel(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                    const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                    const ConvParams p) {
  using Cfg = HaloCfg<BLOCK_N, PLANES, SPLIT>;
  constexpr int SA = Cfg::kAStages, SB = Cfg::kBStages;
  constexpr int kHalves = PINGPONG ? 2 : 1;   // m64 halves of the tile per consumer warpgroup
  static_assert(!PINGPONG || kHalves * Cfg::kAcc <= 128, "a ping-pong warpgroup holds the whole tile's accumulator");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + SA * Cfg::kAStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + SB * Cfg::kBStageBytes);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + SA;
  uint64_t* b_full = bars + 2 * SA;
  uint64_t* b_empty = bars + 2 * SA + SB;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&map_x_hi);
    tma_prefetch_desc(&map_w_hi);
    if (PLANES == 2) {
      tma_prefetch_desc(&map_x_lo);
      tma_prefetch_desc(&map_w_lo);
    }
    constexpr uint32_t kReaders = PINGPONG ? 1 : 2;   // consumer warpgroups that read (and release) each stage
    for (int i = 0; i < SA; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], kReaders);
    }
    for (int i = 0; i < SB; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], kReaders);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: everything above touched only shared memory and the kernel parameters; the previous kernel's outputs
  // (activations, masks, pooled planes, workspaces) are first accessed below.
  pdl_wait();
  pdl_launch_dependents();

  // Ping-pong: the producer warpgroup (warps 0 - 3, all of which must execute the dec) hands registers to the two
  // consumers, whose warpgroups each hold a whole tile's accumulator: 40 * 128 + 232 * 256 <= 64 K.
  if (warp < 4) {
    if (PINGPONG) setmaxnreg_dec<40>();
    if (warp != 0) return;
    // ------------------------------------------------------------ TMA producer (one elected thread)
    // ONE elected thread runs the whole loop, taps unrolled (the tap coordinate is an immediate), tile coordinates
    // decoded once per tile.
    if (elect_one()) {
      int a_stage = 0, b_stage = 0;
      uint32_t a_phase = 0, b_phase = 0;
      const bool skip_a = (p.ablate & 2) != 0, skip_b = (p.ablate & 1) != 0;
      auto issue_a = [&](int x0, int y0, int img, int kc) {
        mbar_wait(&a_empty[a_stage], a_phase ^ 1);
        if (skip_a) {
          mbar_arrive(&a_full[a_stage]);
        } else {
          uint8_t* st = smem_a + a_stage * Cfg::kAStageBytes;
          mbar_arrive_expect_tx(&a_full[a_stage], PLANES * Cfg::kABoxBytes);
          tma_load_4d(&map_x_hi, &a_full[a_stage], st, kc * kBlockK, x0, y0, img);
          if (PLANES == 2) tma_load_4d(&map_x_lo, &a_full[a_stage], st + Cfg::kAPlaneBytes, kc * kBlockK, x0, y0, img);
        }
        if (++a_stage == SA) {
          a_stage = 0;
          a_phase ^= 1;
        }
      };
      int nb = 0, tx = 0, ty = 0, img = 0;
      const int w_first = static_cast<int>(blockIdx.x), w_stride = static_cast<int>(gridDim.x);
      if (w_first < p.total_tiles) {
        decode_tile(p, w_first, nb, tx, ty, img);
        issue_a(tx * kTileW - 1, ty * kTileH - 1, img, 0);
      }
      for (int tile = w_first; tile < p.total_tiles; tile += w_stride) {
        const bool has_next = tile + w_stride < p.total_tiles;
        int nnb = 0, ntx = 0, nty = 0, nimg = 0;
        if (has_next) decode_tile(p, tile + w_stride, nnb, ntx, nty, nimg);
        const int n0 = nb * BLOCK_N;
        for (int kc = 0; kc < p.k_chunks; ++kc) {
          const int c0 = kc * kBlockK;
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            if (tap == 3) {  // prefetch the next chunk's halo while this one is being consumed
              if (kc + 1 < p.k_chunks) issue_a(tx * kTileW - 1, ty * kTileH - 1, img, kc + 1);
              else if (has_next) issue_a(ntx * kTileW - 1, nty * kTileH - 1, nimg, 0);
            }
            mbar_wait(&b_empty[b_stage], b_phase ^ 1);
            if (skip_b) {
              mbar_arrive(&b_full[b_stage]);
            } else {
              uint8_t* st = smem_b + b_stage * Cfg::kBStageBytes;
              mbar_arrive_expect_tx(&b_full[b_stage], Cfg::kBStageBytes);
              tma_load_3d(&map_w_hi, &b_full[b_stage], st, c0, n0, tap);
              if (PLANES == 2) tma_load_3d(&map_w_lo, &b_full[b_stage], st + Cfg::kBPlaneBytes, c0, n0, tap);
            }
            if (++b_stage == SB) {
              b_stage = 0;
              b_phase ^= 1;
            }
          }
        }
        nb = nnb, tx = ntx, ty = nty, img = nimg;
      }
    }
    __syncwarp();
  } else {
    if (PINGPONG) setmaxnreg_inc<232>();
    // ----------------------------------- consumer warpgroups: wgmma + epilogue, 64 rows (cooperative) or 128 (ping-pong)
    // The nine taps are nine descriptors into the halo patch: tap (r, s) starts at smem row (r * kPitch + s), the eight
    // patch rows of an m64 half are eight 8-row swizzle groups at stride SBO = kPitch * 128 B.
    const int wg = (warp - 4) >> 2, wl = warp & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    constexpr uint64_t kDescA = desc_template(16, kPitch * 128, kDescSW128);
    constexpr uint64_t kDescB = desc_template(16, 1024, kDescSW128);
    constexpr uint32_t kLoPlaneA = Cfg::kAPlaneBytes >> 4, kLoPlaneB = Cfg::kBPlaneBytes >> 4;
    constexpr uint32_t kHalfA = (8 * kPitch * 128) >> 4;   // rows 64 .. 127 of the tile start 8 patch rows down
    const uint32_t smem_a_u32 = smem_u32(smem_a) + (PINGPONG ? 0 : wg * 8 * kPitch * 128), smem_b_u32 = smem_u32(smem_b);
    const bool skip_mma = (p.ablate & 4) != 0;
    float acc[kHalves][Cfg::kAcc];
    StageRelease pending;
    // k: the tile's place in the CTA's sequence, which is also the order the producer fills the rings in
    constexpr int kOwners = PINGPONG ? 2 : 1;   // warpgroups the CTA's tiles are dealt to in turn
    for (int k = PINGPONG ? wg : 0;; k += kOwners) {
      const int tile = static_cast<int>(blockIdx.x) + k * static_cast<int>(gridDim.x);
      if (tile >= p.total_tiles) break;
      const bool has_next = tile + static_cast<int>(gridDim.x) < p.total_tiles;
      const int a_seq = k * p.k_chunks, b_seq = 9 * a_seq;   // ring slots filled for the CTA's earlier tiles
      int a_stage = a_seq % SA, b_stage = b_seq % SB;
      uint32_t a_phase = (a_seq / SA) & 1, b_phase = (b_seq / SB) & 1;
      if (PINGPONG && k > 0) named_bar_sync(1 + wg, 256);    // tile k - 1 has passed its last full wait
#pragma unroll
      for (int h = 0; h < kHalves; ++h)
#pragma unroll
        for (int i = 0; i < Cfg::kAcc; ++i) acc[h][i] = 0.f;
      for (int kc = 0; kc < p.k_chunks; ++kc) {
        mbar_wait(&a_full[a_stage], a_phase);
        const uint64_t da0 = kDescA | static_cast<uint64_t>((smem_a_u32 + a_stage * Cfg::kAStageBytes) >> 4);
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t tap_off = static_cast<uint32_t>(((tap / 3) * kPitch + (tap % 3)) * (128 >> 4));
          mbar_wait(&b_full[b_stage], b_phase);
          if (PINGPONG && tap == 8 && kc == p.k_chunks - 1 && has_next) named_bar_arrive(1 + (wg ^ 1), 256);
          const uint64_t db_hi = kDescB | static_cast<uint64_t>((smem_b_u32 + b_stage * Cfg::kBStageBytes) >> 4);
          wgmma_fence();
#pragma unroll
          for (int h = 0; h < kHalves; ++h) {
            const uint64_t da_hi = da0 + h * kHalfA + tap_off;
            const uint64_t da_lo = da_hi + kLoPlaneA;
            if (skip_mma) continue;   // ablation bit 4
#pragma unroll
            for (int ks = 0; ks < kBlockK / 16; ++ks) {
              if constexpr (Cfg::kSplitAcc) {
                wgmma_bf16<2 * BLOCK_N>(acc[h], da_hi + 2 * ks, db_hi + 2 * ks, 1);   // [A_hi.B_hi | A_hi.B_lo]
                wgmma_bf16<BLOCK_N>(acc[h], da_lo + 2 * ks, db_hi + 2 * ks, 1);       // + A_lo.B_hi into the first half
              } else if constexpr (PLANES == 2) {
                wgmma_bf16<BLOCK_N>(acc[h], da_lo + 2 * ks, db_hi + 2 * ks, 1);
                wgmma_bf16<BLOCK_N>(acc[h], da_hi + 2 * ks, db_hi + kLoPlaneB + 2 * ks, 1);
                wgmma_bf16<BLOCK_N>(acc[h], da_hi + 2 * ks, db_hi + 2 * ks, 1);
              } else {
                wgmma_bf16<BLOCK_N>(acc[h], da_hi + 2 * ks, db_hi + 2 * ks, 1);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<1>();               // the previous tap's group is done: its stages may be refilled
          pending.release(leader);
          pending.bar_b = &b_empty[b_stage];
          if (tap == 8) pending.bar_a = &a_empty[a_stage];
          if (++b_stage == SB) {
            b_stage = 0;
            b_phase ^= 1;
          }
        }
        if (++a_stage == SA) {
          a_stage = 0;
          a_phase ^= 1;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < kHalves; ++h) wgmma_fence_operands(acc[h]);
      pending.release(leader);
#pragma unroll
      for (int h = 0; h < kHalves; ++h)
        conv_epilogue<BLOCK_N, Cfg::kSplitAcc, LEAN, DET>(p, acc[h], tile, PINGPONG ? h : wg, wl, lane);
    }
  }
}

// Exact mode with BLOCK_N <= 128 takes the N-concatenated split accumulator (HaloCfg), except under ping-pong for
// BLOCK_N = 128 (below).
// DET: OSVOS_FLAG_DETERMINISTIC with column sums (partial rows instead of atomics).
template <int BLOCK_N, int PLANES, bool LEAN = false, bool DET = false>
static int launch_halo(const osvos_conv3x3_args* a, cudaStream_t stream) {
  constexpr bool kSplit = PLANES == 2 && BLOCK_N <= 128;
  using Cfg = HaloCfg<BLOCK_N, PLANES, kSplit>;
  ConvParams p;
  fill_conv_params(p, a, BLOCK_N);
  const int sms = device_sm_count();
  CUtensorMap mx_hi, mx_lo, mw_hi, mw_lo;
  {
    const uint64_t dims[4] = {(uint64_t)a->cin, (uint64_t)a->w, (uint64_t)a->h, (uint64_t)a->n};
    const uint64_t strides[3] = {(uint64_t)a->cin * 2, (uint64_t)a->w * a->cin * 2,
                                 (uint64_t)a->h * a->w * a->cin * 2};
    const uint32_t box[4] = {kBlockK, kPitch, kHaloRows, 1};
    int rc = encode_tensor_map(&mx_hi, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4, a->x_hi, dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = encode_tensor_map(&mx_lo, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4, PLANES == 2 ? a->x_lo : a->x_hi, dims,
                           strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  int rc = encode_weight_maps(&mw_hi, &mw_lo, a, BLOCK_N);
  if (rc) return rc;
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  // Ping-pong for the tile widths whose whole-tile accumulator fits one warpgroup: 128 columns, so N = 128 takes the
  // three-pass form there (the split pair would need 256).  A CTA with T tiles then hides T - 1 epilogues, but its last
  // one is a whole tile's run by one warpgroup, twice the cooperative schedule's share per warpgroup: against T
  // half-tile epilogues that gains from T = 3 on.  So ping-pong wherever some CTA gets three tiles or more.
  constexpr bool kCanPingPong = BLOCK_N == 64 || BLOCK_N == 128;
  const bool pingpong = kCanPingPong && p.total_tiles > 2 * sms;
  auto kern = pingpong ? conv3x3_halo_kernel<BLOCK_N, PLANES, kSplit && BLOCK_N == 64, LEAN, kCanPingPong, DET>
                       : conv3x3_halo_kernel<BLOCK_N, PLANES, kSplit, LEAN, false, DET>;
  static uint64_t attr_done[2] = {0, 0};   // per kernel: bit d = device d has the shared-memory opt-in
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(kern, Cfg::kSmemBytes, &attr_done[pingpong]));
  OSVOS_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(kConvThreads), Cfg::kSmemBytes, stream, mx_hi, mx_lo,
                              mw_hi, mw_lo, p));
  return OSVOS_OK;
}

// cout 64 or a multiple of 128 (cout 2 and 16 go to side_conv.cu)
template <bool DET>
static int conv3x3_halo_dispatch(const osvos_conv3x3_args* a, cudaStream_t stream) {
  const bool fast = (a->flags & OSVOS_FLAG_FAST) != 0;
  // the lean epilogue serves launches that use nothing but bias / ReLU / split-bf16 act output / fused pool (exact mode)
  const bool lean = !fast && !(a->flags & OSVOS_FLAG_RELU_MASK) && a->colsum == nullptr && a->y_f32 == nullptr;
  const int m_tiles = ((a->w + kTileW - 1) / kTileW) * ((a->h + kTileH - 1) / kTileH) * a->n;
  const int sms = device_sm_count();
  const long tiles128 = static_cast<long>(m_tiles) * (a->cout / 128);
  const long waves128 = (tiles128 + sms - 1) / sms;
  const long waves256 = (static_cast<long>(m_tiles) * (a->cout / 256) + sms - 1) / sms;
  // few tiles (stage 5 at 480x854: 56 of 128 x 128): N = 64 tiles double the CTA count at ~0.8x the time per tile.
  if (a->cout == 64 || (waves128 == 1 && tiles128 * 5 <= static_cast<long>(sms) * 3)) {
    if (lean) return launch_halo<64, 2, true>(a, stream);
    return fast ? launch_halo<64, 1, false, DET>(a, stream) : launch_halo<64, 2, false, DET>(a, stream);
  }
  // Fast mode: N = 256 tiles whenever that does not cost a wave.  The cost model per (tap, 64-channel) step (N = 128 ~ 700
  // cycles, N = 256 ~ 1100, one instruction each) is carried over from the first tensor-core generation this was tuned on;
  // the fast-mode choice has not been measured on an H100.
  // Exact mode never takes N = 256: at ~2200 cycles against ~1000 it would need waves256 * 2.2 < waves128, and
  // waves128 = ceil(2T / S) <= 2 ceil(T / S) = 2 waves256 for any T tiles of 256 on S SMs.  (So the exact-mode A/B in
  // DESIGN.md section 8, 552-553 frames/s with and without 256-wide tiles, ran the same kernels in both arms.)
  if (fast) {
    const bool prefer256 = waves256 * 1100 < waves128 * 700;
    if (a->cout % 256 == 0 && prefer256) return launch_halo<256, 1, false, DET>(a, stream);
    return launch_halo<128, 1, false, DET>(a, stream);
  }
  if (lean) return launch_halo<128, 2, true>(a, stream);
  return launch_halo<128, 2, false, DET>(a, stream);
}

static int check_conv_args(const osvos_conv3x3_args* a) {
  OSVOS_CHECK_ARG(a != nullptr);
  OSVOS_CHECK_ARG(a->n > 0 && a->h > 0 && a->w > 0);
  OSVOS_CHECK_ARG(a->cin >= 64 && a->cin % 64 == 0);
  OSVOS_CHECK_ARG(a->cout == 2 || a->cout == 16 || a->cout == 64 || (a->cout > 0 && a->cout % 128 == 0));
  // cout == 2: the folded side branch (osvos_fold_side_weights_multi) - pq is the only output, bias = the 2 folded biases
  OSVOS_CHECK_ARG(a->cout != 2 || (a->pq != nullptr && a->y_hi == nullptr && a->y_f32 == nullptr && a->pool_hi == nullptr &&
                                   a->colsum == nullptr && !(a->flags & (OSVOS_FLAG_RELU | OSVOS_FLAG_RELU_MASK))));
  // cout == 16: side_prep - fp32 features and / or projections only (no pool or colsum either, below)
  OSVOS_CHECK_ARG(a->cout != 16 || (a->y_hi == nullptr && a->y_lo == nullptr && !(a->flags & OSVOS_FLAG_RELU_MASK)));
  OSVOS_CHECK_ARG(a->x_hi != nullptr && a->w_packed != nullptr);
  OSVOS_CHECK_ARG((a->flags & OSVOS_FLAG_FAST) || a->x_lo != nullptr);
  OSVOS_CHECK_ARG(a->y_hi != nullptr || a->y_f32 != nullptr || a->pq != nullptr || a->pool_hi != nullptr);
  OSVOS_CHECK_ARG(!(a->flags & OSVOS_FLAG_RELU_MASK) || a->mask_hi != nullptr);
  OSVOS_CHECK_ARG(a->pq == nullptr || a->cout == 2 || (a->cout == 16 && a->proj_w != nullptr));
  OSVOS_CHECK_ARG((a->pool_hi == nullptr && a->colsum == nullptr) || a->cout >= 64);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->x_hi) & 15) == 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->w_packed) & 15) == 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->bias) & 15) == 0);
  OSVOS_CHECK_ARG(!(a->flags & OSVOS_FLAG_DETERMINISTIC) || (reinterpret_cast<uintptr_t>(a->colsum) & 7) == 0);
  if (a->cout >= 64) {   // the epilogue moves channel pairs: 4-byte bf16x2 words, 8-byte float2
    const uintptr_t bf16_planes = reinterpret_cast<uintptr_t>(a->y_hi) | reinterpret_cast<uintptr_t>(a->y_lo) |
                                  reinterpret_cast<uintptr_t>(a->pool_hi) | reinterpret_cast<uintptr_t>(a->pool_lo) |
                                  reinterpret_cast<uintptr_t>(a->mask_hi);
    OSVOS_CHECK_ARG((bf16_planes & 3) == 0);
    OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->y_f32) & 7) == 0);
  }
  return OSVOS_OK;
}

}  // namespace osvos

using namespace osvos;

extern "C" int osvos_side_folded_multi(const osvos_conv3x3_args* args, int count, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(args != nullptr && count > 0 && count <= 4);
  const osvos_conv3x3_args* order[4];
  for (int k = 0; k < count; ++k) {
    int rc = check_conv_args(&args[k]);
    if (rc) return rc;
    OSVOS_CHECK_ARG(args[k].cout == 2);
    OSVOS_CHECK_ARG((args[k].flags & OSVOS_FLAG_FAST) == (args[0].flags & OSVOS_FLAG_FAST));
    order[k] = &args[k];
  }
  // deepest scale first: its tiles hold the most channel chunks, and the round-robin deal balances better that way
  for (int i = 1; i < count; ++i)
    for (int j = i; j > 0 && order[j]->cin > order[j - 1]->cin; --j) {
      const osvos_conv3x3_args* t = order[j];
      order[j] = order[j - 1];
      order[j - 1] = t;
    }
  return side_conv_multi_dispatch(order, count, static_cast<cudaStream_t>(stream_));
}

extern "C" int osvos_conv3x3(const osvos_conv3x3_args* a, osvos_stream_t stream_) {
  int rc = check_conv_args(a);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // the folded side branch (cout == 2) and side_prep (cout == 16): nine-taps-along-N kernel (side_conv.cu)
  if (a->cout == 2 || a->cout == 16) return side_conv_dispatch(a, stream);
  // deterministic column sums: partial rows instead of atomics (the other outputs are the same either way)
  if ((a->flags & OSVOS_FLAG_DETERMINISTIC) && a->colsum != nullptr) return conv3x3_halo_dispatch<true>(a, stream);
  return conv3x3_halo_dispatch<false>(a, stream);
}

extern "C" size_t osvos_conv3x3_colsum_rows(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  // 8 partial rows (2 m64 halves x 4 warps) per 128-pixel tile; see conv_epilogue
  return static_cast<size_t>(n) * ((h + kTileH - 1) / kTileH) * ((w + kTileW - 1) / kTileW) * 8;
}

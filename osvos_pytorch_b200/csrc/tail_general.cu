// Side-branch tail with GENERAL deconvolution weights (the reference's upscale[i] / upscale_[i] with any values,
// networks/vgg_osvos.py:45-46,68-69): forward, backward and the parameter gradients of the eight deconvolutions.
// The default path (tail.cu, side_conv.cu, side_bwd_folded.cu) folds side_prep o {score_dsn, fuse slice} into one
// 3x3 conv C -> 2, which needs the interp_surgery taps (diagonal, bilinear); this path keeps the 16 side features F_k.
//
// Scale k, stride s = 2^(k+1), kernel 2s, T = (2s)^2 taps t = ty * 2s + tx.  An output pixel (y, x) of the cropped map
// has the full-map coordinate (y + top, x + left) and exactly the source pixels (iy, ix) with ty = y + top - iy s and
// tx = x + left - ix s in [0, 2s): at most 2 x 2 of them (sources outside the map count as zero).
//   side_k(y, x) = sum_src A_k[t] p_k(src)                           A_k = upscale_[k].weight[0][0]
//   fused(y, x)  = b + sum_k sum_src sum_ci V_k[t][ci] F_k[ci](src)  V_k[t][ci] = sum_co f[16k + co] U_k[ci][co][t]
// Backward, with g_k / g_4 the gradients of side_k / fused:
//   dp_k(src)     = sum_t g_k(out(src, t)) A_k[t],   dF_k[ci](src) = sum_t g_4(out(src, t)) V_k[t][ci] + dp_k(src) sw_k[ci]
//   H_k[t][ci]    = sum_src g_4(out(src, t)) F_k[ci](src),   gA_k[t] = sum_src g_k(out(src, t)) p_k(src)
// and every parameter gradient of the tail is algebra on H, gA and three sums over the source pixels
// (upsampling_grads_finish_kernel).  Every reduction here is fixed-order by construction (per-block partial rows added
// by osvos_reduce_rows), so OSVOS_FLAG_DETERMINISTIC changes nothing in this file.
#include "objective.cuh"
#include "ptx.cuh"
#include "tail_scales.cuh"

namespace osvos {

constexpr int kGenTaps = OSVOS_UPSAMPLING_TAPS;   // 16 + 64 + 256 + 1024
static_assert(kGenTaps == 16 + 64 + 256 + 1024, "tap table layout");
__host__ __device__ __forceinline__ int gen_tap_offset(int k) { return k == 0 ? 0 : k == 1 ? 16 : k == 2 ? 80 : 336; }
__host__ __device__ __forceinline__ int gen_row_len(int taps) { return 17 * taps + 33; }   // H, gA, sum dp F, sum dp, sum dF

int reduce_rows_launch(const float* rows, int nrows, int ncols, int ld, float* scratch, float* out, int accumulate,
                       cudaStream_t stream);   // bwd_kernels.cu

struct GenScale {
  const float* feat;   // [n, hk, wk, 16]
  const float* pq;     // [n, hk, wk, 2], p_k in channel 0
  int hk, wk, s, log2s, top, left;
};

static void fill_gen_scales(GenScale* sc, const float* const* feat, const float* const* pq, int h, int w) {
  for (int k = 0; k < 4; ++k) {
    const TailGeometry g = tail_geometry(k, h, w);
    sc[k].feat = feat[k];
    sc[k].pq = pq[k];
    sc[k].hk = g.hk;
    sc[k].wk = g.wk;
    sc[k].s = g.s;
    sc[k].log2s = k + 1;
    sc[k].top = g.top;
    sc[k].left = g.left;
  }
}

// ------------------------------------------------------------------------------------------------------------ fold
struct GenFoldParams {
  const float* up_w[4];    // [16][16][T]
  const float* up1_w[4];   // [T]
  const float* fuse_w;     // [64]
  float* vtab;             // [kGenTaps][16]
  float* atab;             // [kGenTaps]
};

__global__ void __launch_bounds__(256) upsampling_fold_kernel(const __grid_constant__ GenFoldParams p) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= kGenTaps * 17) return;
  const int tg = i < kGenTaps * 16 ? i >> 4 : i - kGenTaps * 16;
  const int k = tg < 16 ? 0 : tg < 80 ? 1 : tg < 336 ? 2 : 3;
  const int taps = 16 << (2 * k), tap = tg - gen_tap_offset(k);
  if (i >= kGenTaps * 16) {
    p.atab[tg] = __ldg(p.up1_w[k] + tap);
    return;
  }
  const int ci = i & 15;
  float v = 0.f;
#pragma unroll
  for (int co = 0; co < 16; ++co)
    v = fmaf(__ldg(p.fuse_w + 16 * k + co), __ldg(p.up_w[k] + static_cast<size_t>(ci * 16 + co) * taps + tap), v);
  p.vtab[i] = v;
}

// --------------------------------------------------------------------------------------------------------- forward
struct GenFwdParams {
  GenScale sc[4];
  const float* vtab;
  const float* atab;
  const float* fuse_bias;
  float* out[5];
  const float* label;
  double* sums;           // kTailSums, then one row of kTailVals block partials per block
  float* losses;
  float loss_weights[5];
  float inv_divisor;
  int n, h, w;
};
constexpr int kGenThreads = 256;
constexpr int kGenTabFloats = kGenTaps * 17;   // V then A: 92,480 bytes of shared memory

// One block = one output row at a time, one thread = one pixel: per scale up to 2 x 2 sources, each a 16-channel dot
// product of the side features with the tap's V row (shared memory) plus one A tap on p.
__global__ void __launch_bounds__(kGenThreads) tail_general_fwd_kernel(const __grid_constant__ GenFwdParams p) {
  extern __shared__ float4 gen_tab4[];
  float* tab = reinterpret_cast<float*>(gen_tab4);
  const float* atab = tab + kGenTaps * 16;
  for (int i = threadIdx.x; i < kGenTabFloats / 4; i += kGenThreads)
    gen_tab4[i] = __ldg(reinterpret_cast<const float4*>(p.vtab) + i);   // vtab and atab are contiguous
  __syncthreads();
  const uint32_t total = static_cast<uint32_t>(p.n) * p.h * p.w;
  const float fb = p.fuse_bias ? __ldg(p.fuse_bias) : 0.f;
  CbceSums<5, true, false> acc;   // the maps' loss sums (objective.cuh)
  for (int row = blockIdx.x; row < p.n * p.h; row += gridDim.x) {
    const int img = row / p.h, y = row - img * p.h;
    for (int x = threadIdx.x; x < p.w; x += kGenThreads) {
      float o[5];
      float fused = fb;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const GenScale& sc = p.sc[k];
        const int fs = 2 * sc.s;
        const int oy = y + sc.top, ox = x + sc.left;
        const int ay = oy >> sc.log2s, ax = ox >> sc.log2s;
        const int ry = oy & (sc.s - 1), rx = ox & (sc.s - 1);
        const float* V = tab + gen_tap_offset(k) * 16;
        const float* A = atab + gen_tap_offset(k);
        float side = 0.f;
#pragma unroll
        for (int u = 0; u < 2; ++u) {          // u = 0: source row ay (ty = ry), u = 1: row ay - 1 (ty = ry + s)
          const int iy = ay - u;
          if (iy < 0 || iy >= sc.hk) continue;
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            const int ix = ax - v;
            if (ix < 0 || ix >= sc.wk) continue;
            const int tap = (ry + u * sc.s) * fs + rx + v * sc.s;
            const size_t src = (static_cast<size_t>(img) * sc.hk + iy) * sc.wk + ix;
            side = fmaf(A[tap], __ldg(sc.pq + 2 * src), side);
            const float4* f4 = reinterpret_cast<const float4*>(sc.feat + 16 * src);
            const float4* v4 = reinterpret_cast<const float4*>(V + 16 * tap);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 a = __ldg(f4 + j), b = v4[j];
              fused = fmaf(a.x, b.x, fused);
              fused = fmaf(a.y, b.y, fused);
              fused = fmaf(a.z, b.z, fused);
              fused = fmaf(a.w, b.w, fused);
            }
          }
        }
        o[k] = side;
      }
      o[4] = fused;
      const size_t e = static_cast<size_t>(row) * p.w + x;
#pragma unroll
      for (int k = 0; k < 5; ++k)
        if (p.out[k]) p.out[k][e] = o[k];
      if (p.label) acc.add(o, __ldg(p.label + e));
    }
  }
  if (!p.label) return;
  // block partials to this block's row, then the last block adds the rows in block order (tail.cu's deterministic form)
  // and turns the sums into the losses
  if (commit_block_sums<kGenThreads, kTailSums, true>(acc.v, p.sums, TailSlot()) && threadIdx.x == 0)
    tail_losses<false>(p.sums, total, p.losses, p.loss_weights, p.inv_divisor);
}

// -------------------------------------------------------------------------------------------------------- backward
// Work item = (scale, image, source row iy, segment of kGenSeg source columns).  The block stages the 2s x (seg + 1) s
// window of g_k and g_4 its sources reach (formed on the fly from logits and label in LOSS mode), then
//   phase 1: 16 lanes per source pixel, lane ci: dF[ci] over all T taps, dp split over the lanes and shuffle-reduced;
//            dF is written as a split-bf16 act of 64 channels (16..63 zero): the operand of the tensor-core weight and
//            data gradients of side_prep (osvos_conv3x3_wgrad / osvos_conv3x3 with transposed weights);
//   phase 2: one thread per (tap, ci) bin of H (and per tap of gA) sums over the segment's pixels;
// and writes its partial row [H (16 T) | gA (T) | sum dp F (16) | sum dp | sum dF (16)].
constexpr int kGenSeg = 16;
struct GenBwdScale {
  const float* feat;
  const float* pq;
  const float* score_w;       // [16]
  __nv_bfloat16* df_hi;       // [n, hk, wk, 64]
  __nv_bfloat16* df_lo;       // or NULL (fast)
  float* rows;                // [items][gen_row_len(T)]
  int hk, wk, s, top, left, segs, first_item;
};
struct GenBwdParams {
  GenBwdScale sc[4];
  const float* vtab;
  const float* atab;
  const float* src[5];
  const float* label;
  const double* sums;
  const float* upstream;
  float coeff[5];
  float inv_divisor;
  float* fuse_bias_grad;
  int n, h, w;
};

__host__ __device__ __forceinline__ int gen_bwd_smem_floats(int s) {
  return 2 * (2 * s) * ((kGenSeg + 1) * s) + kGenSeg * 16 * 2 + 2 * kGenSeg;
}

template <bool LOSS>
__global__ void __launch_bounds__(256) tail_general_bwd_kernel(const __grid_constant__ GenBwdParams p) {
  extern __shared__ float gen_bwd_smem[];
  const int tid = threadIdx.x;
  int k = 3;
  while (k > 0 && static_cast<int>(blockIdx.x) < p.sc[k].first_item) --k;
  const GenBwdScale& sc = p.sc[k];
  const int local = static_cast<int>(blockIdx.x) - sc.first_item;
  const int seg = local % sc.segs, rowi = local / sc.segs;
  const int iy = rowi % sc.hk, img = rowi / sc.hk;
  const int s = sc.s, fs = 2 * s, taps = fs * fs;
  const int ix0 = seg * kGenSeg;
  const int nout = min(kGenSeg, sc.wk - ix0);
  const int rw = (kGenSeg + 1) * s;          // window columns
  const int y0 = iy * s - sc.top, x0 = ix0 * s - sc.left;
  float* gk = gen_bwd_smem;                  // [2s][rw]
  float* g4 = gk + fs * rw;
  float* fseg = g4 + fs * rw;                // [kGenSeg][16] side features of the segment
  float* dfseg = fseg + kGenSeg * 16;        // [kGenSeg][16] their gradients
  float* pseg = dfseg + kGenSeg * 16;        // [kGenSeg]
  float* dpseg = pseg + kGenSeg;             // [kGenSeg]
  const float* V = p.vtab + gen_tap_offset(k) * 16;
  const float* A = p.atab + gen_tap_offset(k);

  float wpos = 0.f, wneg = 0.f, cp = 1.f, cq = 1.f;
  if (LOSS) tail_loss_coeffs<false>(p, k, wpos, wneg, cp, cq);
  const bool use_p = LOSS ? (p.coeff[k] != 0.f) : (p.src[k] != nullptr);
  const bool use_q = LOSS ? (p.coeff[4] != 0.f) : (p.src[4] != nullptr);
  for (int i = tid; i < fs * rw; i += 256) {
    const int r = i / rw, c = i - r * rw;
    const int y = y0 + r, x = x0 + c;
    float a = 0.f, b = 0.f;
    if (y >= 0 && y < p.h && x >= 0 && x < p.w) {
      const size_t o = (static_cast<size_t>(img) * p.h + y) * p.w + x;
      if (LOSS) {
        const bool pos = __ldg(p.label + o) >= 0.5f;
        const float wgt = pos ? wpos : wneg, yv = pos ? 1.f : 0.f;
        if (use_p) a = cp * wgt * (sigmoid(__ldg(p.src[k] + o)) - yv);
        if (use_q) b = cq * wgt * (sigmoid(__ldg(p.src[4] + o)) - yv);
      } else {
        if (use_p) a = __ldg(p.src[k] + o);
        if (use_q) b = __ldg(p.src[4] + o);
      }
    }
    gk[i] = a;
    g4[i] = b;
  }
  const size_t pix0 = (static_cast<size_t>(img) * sc.hk + iy) * sc.wk + ix0;
  for (int i = tid; i < kGenSeg * 16; i += 256) fseg[i] = (i >> 4) < nout ? __ldg(sc.feat + pix0 * 16 + i) : 0.f;
  if (tid < kGenSeg) pseg[tid] = tid < nout ? __ldg(sc.pq + 2 * (pix0 + tid)) : 0.f;
  __syncthreads();

  // phase 1
  {
    const int j = tid >> 4, ci = tid & 15;
    float dfv = 0.f, dpv = 0.f;
    if (j < nout) {
      const float* g4j = g4 + j * s;
      const float* gkj = gk + j * s;
      for (int ty = 0; ty < fs; ++ty)
        for (int tx = 0; tx < fs; ++tx) dfv = fmaf(g4j[ty * rw + tx], __ldg(V + (ty * fs + tx) * 16 + ci), dfv);
      for (int t = ci; t < taps; t += 16) dpv = fmaf(gkj[(t / fs) * rw + t % fs], __ldg(A + t), dpv);
    }
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) dpv += __shfl_xor_sync(0xffffffffu, dpv, off);   // within the 16-lane group
    if (j < nout) {
      dfv = fmaf(dpv, __ldg(sc.score_w + ci), dfv);
      dfseg[j * 16 + ci] = dfv;
      if (ci == 0) dpseg[j] = dpv;
      const size_t d = (pix0 + j) * 64;
      __nv_bfloat16 hi, lo;
      split_bf16(dfv, hi, lo);
      const __nv_bfloat16 z = __float2bfloat16_rn(0.f);
      sc.df_hi[d + ci] = hi;
      sc.df_hi[d + 16 + ci] = z;
      sc.df_hi[d + 32 + ci] = z;
      sc.df_hi[d + 48 + ci] = z;
      if (sc.df_lo) {
        sc.df_lo[d + ci] = lo;
        sc.df_lo[d + 16 + ci] = z;
        sc.df_lo[d + 32 + ci] = z;
        sc.df_lo[d + 48 + ci] = z;
      }
    } else if (j < kGenSeg) {
      dfseg[j * 16 + ci] = 0.f;
      if (ci == 0) dpseg[j] = 0.f;
    }
  }
  __syncthreads();

  // phase 2
  float* row = sc.rows + static_cast<size_t>(local) * gen_row_len(taps);
  for (int b = tid; b < 17 * taps; b += 256) {
    float acc = 0.f;
    if (b < 16 * taps) {
      const int t = b >> 4, ci = b & 15;
      const float* g = g4 + (t / fs) * rw + t % fs;
      for (int j = 0; j < nout; ++j) acc = fmaf(g[j * s], fseg[j * 16 + ci], acc);
    } else {
      const int t = b - 16 * taps;
      const float* g = gk + (t / fs) * rw + t % fs;
      for (int j = 0; j < nout; ++j) acc = fmaf(g[j * s], pseg[j], acc);
    }
    row[b] = acc;
  }
  if (tid < 33) {
    float acc = 0.f;
    for (int j = 0; j < nout; ++j) {
      if (tid < 16) acc = fmaf(dpseg[j], fseg[j * 16 + tid], acc);
      else if (tid == 16) acc += dpseg[j];
      else acc += dfseg[j * 16 + tid - 17];
    }
    row[17 * taps + tid] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------- finish
struct GenFinishScale {
  const float* red;    // [gen_row_len(T)]
  const float* up_w;   // [16][16][T]
  float* d_up;         // [16][16][T] or NULL
  float* d_up1;        // [T] or NULL
  float* d_score_w;    // [16] or NULL
  float* d_score_b;    // [1] or NULL
  float* d_side_b;     // [16] or NULL
};
struct GenFinishParams {
  GenFinishScale sc[4];
  const float* fuse_w;
  float* d_fuse_w;     // [64] or NULL
  int accumulate;
};

// One block per (scale, output channel co of upscale[k]):
//   d upscale[k][ci][co][t] = f[16k + co] H[t][ci],   d fuse.weight[16k + co] = sum_{ci,t} U[ci][co][t] H[t][ci]
// and block co == 0 also: d upscale_[k] = gA, d score_dsn[k] = (sum dp F, sum dp), d side_prep[k].bias = sum dF.
__global__ void __launch_bounds__(256) upsampling_grads_finish_kernel(const __grid_constant__ GenFinishParams p) {
  const int k = blockIdx.x >> 4, co = blockIdx.x & 15;
  const GenFinishScale& sc = p.sc[k];
  const int taps = 16 << (2 * k);
  const bool acc = p.accumulate != 0;
  const float f = __ldg(p.fuse_w + 16 * k + co);
  float dot = 0.f;
  for (int i = threadIdx.x; i < 16 * taps; i += 256) {
    const int ci = i / taps, t = i - ci * taps;
    const float hv = __ldg(sc.red + t * 16 + ci);
    const size_t e = static_cast<size_t>(ci * 16 + co) * taps + t;
    dot = fmaf(__ldg(sc.up_w + e), hv, dot);
    if (sc.d_up) sc.d_up[e] = acc ? sc.d_up[e] + f * hv : f * hv;
  }
  __shared__ float red[256];
  red[threadIdx.x] = dot;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  auto put = [&](float* dst, float v) { *dst = acc ? *dst + v : v; };
  if (threadIdx.x == 0 && p.d_fuse_w) put(p.d_fuse_w + 16 * k + co, red[0]);
  if (co != 0) return;
  for (int t = threadIdx.x; t < taps; t += 256)
    if (sc.d_up1) put(sc.d_up1 + t, __ldg(sc.red + 16 * taps + t));
  const float* sums = sc.red + 17 * taps;
  if (threadIdx.x < 16 && sc.d_score_w) put(sc.d_score_w + threadIdx.x, __ldg(sums + threadIdx.x));
  if (threadIdx.x == 16 && sc.d_score_b) put(sc.d_score_b, __ldg(sums + 16));
  if (threadIdx.x >= 17 && threadIdx.x < 33 && sc.d_side_b) put(sc.d_side_b + threadIdx.x - 17, __ldg(sums + threadIdx.x));
}

// work items of the backward per scale, and the floats of its partial rows
static int gen_bwd_plan(GenBwdParams* p, int n, int h, int w, size_t* row_floats) {
  int items = 0;
  size_t rows = 0;
  for (int k = 0; k < 4; ++k) {
    const TailGeometry g = tail_geometry(k, h, w);
    const int segs = (g.wk + kGenSeg - 1) / kGenSeg;
    if (p) {
      GenBwdScale& sc = p->sc[k];
      sc.hk = g.hk;
      sc.wk = g.wk;
      sc.s = g.s;
      sc.top = g.top;
      sc.left = g.left;
      sc.segs = segs;
      sc.first_item = items;
    }
    const int nk = n * g.hk * segs;
    if (row_floats) row_floats[k] = rows;
    rows += static_cast<size_t>(nk) * gen_row_len(4 * g.s * g.s);
    items += nk;
  }
  if (row_floats) row_floats[4] = rows;
  return items;
}

}  // namespace osvos

using namespace osvos;

extern "C" int osvos_upsampling_fold(const osvos_upsampling_fold_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->fuse_w != nullptr && a->vtab != nullptr && a->atab != nullptr);
  GenFoldParams p;
  for (int k = 0; k < 4; ++k) {
    OSVOS_CHECK_ARG(a->upscale_w[k] != nullptr && a->upscale1_w[k] != nullptr);
    p.up_w[k] = a->upscale_w[k];
    p.up1_w[k] = a->upscale1_w[k];
  }
  p.fuse_w = a->fuse_w;
  p.vtab = a->vtab;
  p.atab = a->atab;
  upsampling_fold_kernel<<<(kGenTaps * 17 + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream_)>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" size_t osvos_tail_general_fwd_sums(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return kTailSums + static_cast<size_t>(tail_fwd_blocks(n, h)) * kTailVals;
}

extern "C" int osvos_tail_general_fwd(const osvos_tail_general_fwd_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->n > 0 && a->h > 0 && a->w > 0);
  OSVOS_CHECK_ARG((a->flags & ~OSVOS_FLAG_DETERMINISTIC) == 0);
  OSVOS_CHECK_ARG(a->vtab != nullptr && a->atab == a->vtab + kGenTaps * 16);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->vtab) & 15) == 0);
  OSVOS_CHECK_ARG(a->label == nullptr || a->sums != nullptr);
  OSVOS_CHECK_ARG(a->losses == nullptr || (a->label != nullptr && a->divisor > 0.f));
  OSVOS_CHECK_ARG(static_cast<size_t>(a->n) * a->h * a->w < (1ull << 31));
  GenFwdParams p;
  memset(&p, 0, sizeof(p));
  for (int k = 0; k < 4; ++k) {
    OSVOS_CHECK_ARG(a->feat[k] != nullptr && a->pq[k] != nullptr && (reinterpret_cast<uintptr_t>(a->feat[k]) & 15) == 0);
  }
  fill_gen_scales(p.sc, a->feat, a->pq, a->h, a->w);
  p.vtab = a->vtab;
  p.atab = a->atab;
  p.fuse_bias = a->fuse_bias;
  for (int k = 0; k < 5; ++k) {
    p.out[k] = a->out[k];
    p.loss_weights[k] = a->loss_weights[k];
  }
  p.label = a->label;
  p.sums = a->label ? a->sums : nullptr;
  p.losses = a->losses;
  p.inv_divisor = a->divisor > 0.f ? 1.f / a->divisor : 1.f;
  p.n = a->n;
  p.h = a->h;
  p.w = a->w;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (p.sums) OSVOS_CHECK_CUDA(cudaMemsetAsync(p.sums, 0, kTailSums * sizeof(double), stream));
  const int smem = kGenTabFloats * static_cast<int>(sizeof(float));
  static uint64_t attr_done = 0;
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(tail_general_fwd_kernel, smem, &attr_done));
  tail_general_fwd_kernel<<<tail_fwd_blocks(a->n, a->h), kGenThreads, smem, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" size_t osvos_tail_general_bwd_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  GenBwdParams p;
  size_t off[5];
  gen_bwd_plan(&p, n, h, w, off);
  size_t scratch = 0;
  for (int k = 0; k < 4; ++k) {
    const int nrows = n * p.sc[k].hk * p.sc[k].segs;
    const size_t sk = osvos_reduce_rows_scratch_floats(nrows, gen_row_len(4 * p.sc[k].s * p.sc[k].s));
    scratch = sk > scratch ? sk : scratch;
  }
  return (off[4] + scratch) * sizeof(float);
}

extern "C" int osvos_tail_general_bwd(const osvos_tail_general_bwd_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->n > 0 && a->h > 0 && a->w > 0 && a->workspace != nullptr);
  OSVOS_CHECK_ARG((a->flags & ~OSVOS_FLAG_DETERMINISTIC) == 0);
  OSVOS_CHECK_ARG(a->vtab != nullptr && a->atab != nullptr);
  OSVOS_CHECK_ARG(static_cast<size_t>(a->n) * a->h * a->w < (1ull << 31));
  const bool loss = a->label != nullptr;
  OSVOS_CHECK_ARG(!loss || (a->sums != nullptr && a->divisor > 0.f));
  for (int k = 0; k < 5; ++k) OSVOS_CHECK_ARG(!loss || a->src[k] != nullptr || a->loss_weights[k] == 0.f);
  GenBwdParams p;
  memset(&p, 0, sizeof(p));
  size_t off[5];
  const int items = gen_bwd_plan(&p, a->n, a->h, a->w, off);
  float* ws = static_cast<float*>(a->workspace);
  for (int k = 0; k < 4; ++k) {
    OSVOS_CHECK_ARG(a->feat[k] != nullptr && a->pq[k] != nullptr && a->score_w[k] != nullptr && a->df_hi[k] != nullptr &&
                    a->red[k] != nullptr);
    GenBwdScale& sc = p.sc[k];
    sc.feat = a->feat[k];
    sc.pq = a->pq[k];
    sc.score_w = a->score_w[k];
    sc.df_hi = static_cast<__nv_bfloat16*>(a->df_hi[k]);
    sc.df_lo = static_cast<__nv_bfloat16*>(a->df_lo[k]);
    sc.rows = ws + off[k];
  }
  p.vtab = a->vtab;
  p.atab = a->atab;
  for (int k = 0; k < 5; ++k) {
    p.src[k] = a->src[k];
    p.coeff[k] = a->loss_weights[k];
  }
  p.label = a->label;
  p.sums = a->sums;
  p.upstream = a->upstream;
  p.inv_divisor = loss ? 1.f / a->divisor : 1.f;
  p.fuse_bias_grad = loss ? a->fuse_bias_grad : nullptr;
  p.n = a->n;
  p.h = a->h;
  p.w = a->w;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int smem = gen_bwd_smem_floats(16) * static_cast<int>(sizeof(float));
  static uint64_t attr_done[2] = {0, 0};
  if (loss) {
    OSVOS_CHECK_CUDA(ensure_dynamic_smem(tail_general_bwd_kernel<true>, smem, &attr_done[1]));
    tail_general_bwd_kernel<true><<<items, 256, smem, stream>>>(p);
  } else {
    OSVOS_CHECK_CUDA(ensure_dynamic_smem(tail_general_bwd_kernel<false>, smem, &attr_done[0]));
    tail_general_bwd_kernel<false><<<items, 256, smem, stream>>>(p);
  }
  OSVOS_CHECK_CUDA(cudaGetLastError());
  for (int k = 0; k < 4; ++k) {   // the partial rows in row order
    const int nrows = a->n * p.sc[k].hk * p.sc[k].segs;
    const int len = gen_row_len(4 * p.sc[k].s * p.sc[k].s);
    const int rc = reduce_rows_launch(ws + off[k], nrows, len, len, ws + off[4], a->red[k], 0, stream);
    if (rc) return rc;
  }
  return OSVOS_OK;
}

extern "C" int osvos_upsampling_grads_finish(const osvos_upsampling_grads_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->fuse_w != nullptr);
  GenFinishParams p;
  for (int k = 0; k < 4; ++k) {
    OSVOS_CHECK_ARG(a->red[k] != nullptr && a->upscale_w[k] != nullptr);
    GenFinishScale& sc = p.sc[k];
    sc.red = a->red[k];
    sc.up_w = a->upscale_w[k];
    sc.d_up = a->d_upscale_w[k];
    sc.d_up1 = a->d_upscale1_w[k];
    sc.d_score_w = a->d_score_w[k];
    sc.d_score_b = a->d_score_b[k];
    sc.d_side_b = a->d_side_b[k];
  }
  p.fuse_w = a->fuse_w;
  p.d_fuse_w = a->d_fuse_w;
  p.accumulate = a->accumulate ? 1 : 0;
  upsampling_grads_finish_kernel<<<64, 256, 0, static_cast<cudaStream_t>(stream_)>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

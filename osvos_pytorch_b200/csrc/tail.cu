// Side-branch tail, forward: zero-padded bilinear "deconvolution" of the four
// low-resolution score / fuse-slice maps, centre crop, fusion sum and (optional)
// the per-pixel class-balanced BCE terms with their spatial reductions - one
// bandwidth-bound pass.
//
// Reference ops replaced (see include/osvos_b200.h): ConvTranspose2d with
// interp_surgery weights (networks/vgg_osvos.py:45-46,68-69;
// layers/osvos_layers.py:59-85), center_crop (layers/osvos_layers.py:51-56),
// cat + fuse (networks/vgg_osvos.py:71-72), loss terms
// (layers/osvos_layers.py:28-41).
//
// Math: the deconvolution with kernel 2s / stride s and taps
// f[t] = 1 - |t - (s - .5)| / s touches at most two source rows and columns per
// output pixel: with o = y + crop_top, a = o / s, r = o % s the rows are
// a (weight (r + .5)/s, if a < h_k) and a - 1 (weight 1 - (r + .5)/s, if a >= 1);
// rows outside the source contribute zero (zero padding => attenuated border).
#include "objective.cuh"
#include "ptx.cuh"
#include "tail_scales.cuh"

namespace osvos {

struct TailScale {
  const float* pq;  // [n, hk, wk, 2]
  int hk, wk, s, log2s, top, left;
  float inv_s;      // 1 / s, exact (s is a power of two): the tap weights are multiples of 1 / (2 s)
};
struct TailParams {
  TailScale sc[4];
  const float* fuse_bias;
  float* out[5];
  const float* label;
  double* sums;
  float* losses;          // [6]: the five per-map losses and their weighted total (written by the last block), or NULL
  float loss_weights[5];
  float inv_divisor;
  int n, h, w;
  int vec_mask;  // bit k: out[k] is 16-byte aligned; bit 5: label is
};

constexpr int kTailThreads = 256;

// One block = one output row.  Phase 1 interpolates VERTICALLY once per row: for each scale the (at most two) source rows
// are blended into shared memory, v_k[c] = wy0 * pq_k[ay - 1][c] + wy1 * pq_k[ay][c] (806 float2 for a 854-pixel row).
// Phase 2: a thread takes four consecutive pixels (shifted so that the four are a 16-byte aligned group of the flat map
// whatever the row length) and blends HORIZONTALLY from shared memory: two LDS.64 and four FMAs per scale and pixel.
// (The full 2 x 2 gather with its index arithmetic per pixel and scale costs ~850 instructions per pixel group.)
// DET (OSVOS_FLAG_DETERMINISTIC): block partials go to rows behind the sums, added in a fixed order by the last block.
// VOID (OSVOS_FLAG_VOID_LABELS): pixels with y < 0 enter no sum; N is counted (sums[11]) and N == 0 gives losses of 0.
template <bool DET, bool VOID>
__device__ __forceinline__ void tail_fwd_body(const TailParams& p) {
  extern __shared__ float2 vbuf[];     // [scale 0 .. 3][wk_k] vertically blended (p, q)
  pdl_wait();               // side maps, biases and the accumulators all come from earlier kernels (ptx.cuh)
  pdl_launch_dependents();
  const uint32_t total = static_cast<uint32_t>(p.n) * p.h * p.w;
  const float fb = p.fuse_bias ? __ldg(p.fuse_bias) : 0.f;
  int voff[4];
  voff[0] = 0;
#pragma unroll
  for (int k = 1; k < 4; ++k) voff[k] = voff[k - 1] + p.sc[k - 1].wk;

  CbceSums<5, true, VOID> acc;   // the maps' loss sums (objective.cuh)

  for (int row = blockIdx.x; row < p.n * p.h; row += gridDim.x) {
    const int img = row / p.h, y = row - img * p.h;
    if (row != static_cast<int>(blockIdx.x)) __syncthreads();      // the previous row's readers are done with vbuf
    // ---- phase 1: vertical blend of the source rows of this output row
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const TailScale& sc = p.sc[k];
      const int oy = y + sc.top;
      const int ay = oy >> sc.log2s;
      const float fy1 = (static_cast<float>(oy & (sc.s - 1)) + 0.5f) * sc.inv_s;   // weight of row ay (s = 2^k: exact)
      const float w0 = ay >= 1 ? 1.f - fy1 : 0.f, w1 = ay < sc.hk ? fy1 : 0.f;
      const float2* r0 = reinterpret_cast<const float2*>(sc.pq) + (static_cast<size_t>(img) * sc.hk + (ay >= 1 ? ay - 1 : 0)) * sc.wk;
      const float2* r1 = reinterpret_cast<const float2*>(sc.pq) + (static_cast<size_t>(img) * sc.hk + (ay < sc.hk ? ay : sc.hk - 1)) * sc.wk;
      for (int c = threadIdx.x; c < sc.wk; c += kTailThreads) {
        float2 v = make_float2(0.f, 0.f);
        if (w0 != 0.f) {
          const float2 t = __ldg(r0 + c);
          v.x = w0 * t.x, v.y = w0 * t.y;
        }
        if (w1 != 0.f) {
          const float2 t = __ldg(r1 + c);
          v.x = fmaf(w1, t.x, v.x), v.y = fmaf(w1, t.y, v.y);
        }
        vbuf[voff[k] + c] = v;
      }
    }
    __syncthreads();
    // ---- phase 2: horizontal blend, four pixels per thread
    const uint32_t row_base = static_cast<uint32_t>(row) * p.w;
    const int shift = static_cast<int>(row_base & 3u);
    for (int g = threadIdx.x; g * 4 - shift < p.w; g += kTailThreads) {
      const int x_first = g * 4 - shift;
      const uint32_t e0 = row_base + x_first;          // multiple of 4 (may start before the row: those lanes are skipped)
      float o[4][5];   // [pixel][map]
      float lab[4] = {0, 0, 0, 0};
      const bool full = x_first >= 0 && x_first + 3 < p.w;
      if (p.label) {
        if (full && (p.vec_mask & 32)) {
          const float4 l4 = __ldg(reinterpret_cast<const float4*>(p.label + e0));
          lab[0] = l4.x, lab[1] = l4.y, lab[2] = l4.z, lab[3] = l4.w;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (x_first + j >= 0 && x_first + j < p.w) lab[j] = __ldg(p.label + e0 + j);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int x = x_first + j;
        const bool live = x >= 0 && x < p.w;
        float fused = fb;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const TailScale& sc = p.sc[k];
          const int ox = (live ? x : 0) + sc.left;
          const int ax = ox >> sc.log2s;
          const float fx1 = (static_cast<float>(ox & (sc.s - 1)) + 0.5f) * sc.inv_s;   // weight of col ax
          const float w0 = ax >= 1 ? 1.f - fx1 : 0.f, w1 = ax < sc.wk ? fx1 : 0.f;
          const float2 t0 = vbuf[voff[k] + (ax >= 1 ? ax - 1 : 0)];
          const float2 t1 = vbuf[voff[k] + (ax < sc.wk ? ax : sc.wk - 1)];
          o[j][k] = fmaf(w1, t1.x, w0 * t0.x);
          fused += fmaf(w1, t1.y, w0 * t0.y);
        }
        o[j][4] = fused;
        if (p.label && live) acc.add(o[j], lab[j]);
      }
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        if (!p.out[k]) continue;
        if (full && (p.vec_mask & (1 << k))) {
          *reinterpret_cast<float4*>(p.out[k] + e0) = make_float4(o[0][k], o[1][k], o[2][k], o[3][k]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (x_first + j >= 0 && x_first + j < p.w) p.out[k][e0 + j] = o[j][k];
        }
      }
    }
  }

  if (p.label && p.sums) {
    // the last block to arrive turns the sums into the five losses and their weighted total
    if (commit_block_sums<kTailThreads, kTailSums, DET>(acc.v, p.sums, TailSlot()) && threadIdx.x == 0)
      tail_losses<VOID>(p.sums, total, p.losses, p.loss_weights, p.inv_divisor);
  }
}

template <bool DET = false>
__global__ void __launch_bounds__(kTailThreads) tail_fwd_kernel(const TailParams p) {
  tail_fwd_body<DET, false>(p);
}

template <bool DET>
__global__ void __launch_bounds__(kTailThreads) tail_fwd_void_kernel(const TailParams p) {
  tail_fwd_body<DET, true>(p);
}

// ------------------------------------------------------------------------------------------------------------------
// Backward of the tail (and, in LOSS mode, of the class-balanced BCE on top of it) in ONE launch:
//   dpq[k][iy][ix] = sum_{ty,tx < 2s} f[ty] f[tx] * (g_k, g_4)[iy*s + ty - top][ix*s + tx - left]        (adjoint of the
//   zero-padded bilinear deconvolution + crop: networks/vgg_osvos.py:68-72, layers/osvos_layers.py:51-85)
// with g_k either given (LOSS = false: arbitrary upstream gradients of the five maps) or formed on the fly from the logit
// maps and the label (LOSS = true): g_k = c_k * w * (sigmoid(x_k) - y) / divisor, w = y Nn/N + (1-y) P/N
// (layers/osvos_layers.py:28-46) - the five dL/dlogit maps are never written to memory.
// Work item = (scale, image, low-res row iy, segment of low-res columns): the block first reduces its 2s source rows
// column-wise into shared memory (coalesced row reads, separable weights), then each low-res pixel of the segment sums
// its 2s columns (sub-warp shuffle reduction).  Segments are sized so that every item covers 2-4 k source pixels.
struct TailBwdScale {
  float* dpq;  // [n, hk, wk, 2]
  int hk, wk, s, top, left, seg_lo, segs, first_item;
};
struct TailBwdParams {
  TailBwdScale sc[4];
  const float* src[5];    // LOSS: the five logit maps; else the five upstream gradient maps (NULL = zero)
  const float* label;
  const double* sums;     // forward sums: P at [10], N at [11], A_pos / A_neg at [12] / [13]
  const float* upstream;  // device scalar d(total loss) or NULL (= 1)
  float coeff[5];         // loss weights
  float inv_divisor;
  float* fuse_bias_grad;  // [1] or NULL
  int n, h, w, total_items;
};
constexpr int kTailBwdCols = 512 + 32;

// DET: with several row groups per column, their column sums are added into shared memory in row-group order instead of
// with shared-memory atomics.
// VOID (LOSS only, OSVOS_FLAG_VOID_LABELS): pixels with y < 0 get weight 0, and N = sums[11] == 0 gives zero gradients.
template <bool LOSS, bool DET, bool VOID>
__device__ __forceinline__ void tail_bwd2_body(const TailBwdParams& p) {
  __shared__ float colp[kTailBwdCols], colq[kTailBwdCols];
  const int tid = threadIdx.x;
  int k = 3;
  while (k > 0 && static_cast<int>(blockIdx.x) < p.sc[k].first_item) --k;
  const TailBwdScale& sc = p.sc[k];
  const int local = static_cast<int>(blockIdx.x) - sc.first_item;
  const int seg = local % sc.segs, row = local / sc.segs;
  const int iy = row % sc.hk, img = row / sc.hk;
  const int s = sc.s, fs = 2 * s;
  const int ix0 = seg * sc.seg_lo;
  const int nout = min(sc.seg_lo, sc.wk - ix0);
  const int xlo = ix0 * s - sc.left;        // image column of shared-memory column 0 (may be negative)
  const int width = nout * s + s;
  const float inv_s = 1.f / static_cast<float>(s);

  float wpos = 0.f, wneg = 0.f, cp = 1.f, cq = 1.f;
  if (LOSS) tail_loss_coeffs<VOID>(p, k, wpos, wneg, cp, cq);
  const bool use_p = LOSS ? (p.coeff[k] != 0.f) : (p.src[k] != nullptr);
  const bool use_q = LOSS ? (p.coeff[4] != 0.f) : (p.src[4] != nullptr);

  for (int c = tid; c < width; c += 256) colp[c] = 0.f, colq[c] = 0.f;
  __syncthreads();
  // phase 1: column sums over the 2s source rows.  Threads = (row group r) x (column c0): wpad columns side by side,
  // 256 / wpad row groups striding the rows.
  const int wpad = min(256, (width + 31) & ~31);
  const int rgroups = 256 / wpad;
  const int r = tid / wpad, c0 = tid - r * wpad;
  float keep_p = 0.f, keep_q = 0.f;   // DET, rgroups > 1: this thread's (single) column sum
  bool kept = false;
  if (r < rgroups) {
    for (int c = c0; c < width; c += wpad) {
      const int x = xlo + c;
      const bool xin = x >= 0 && x < p.w;
      float ap = 0.f, aq = 0.f;
      // four source rows per step with all their loads issued before the first use: the row loop is a chain of
      // dependent global loads otherwise (16 round trips for s = 16)
      for (int t0 = r; t0 < fs; t0 += 4 * rgroups) {
        float fyv[4], lv[4], pv[4], qv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int ty = t0 + u * rgroups;
          const int y = iy * s + ty - sc.top;
          const bool ok = xin && ty < fs && y >= 0 && y < p.h;
          const size_t o = ok ? (static_cast<size_t>(img) * p.h + y) * p.w + x : 0;     // (index 0: a valid address)
          fyv[u] = ok ? 1.f - fabsf(static_cast<float>(ty) - (static_cast<float>(s) - 0.5f)) * inv_s : 0.f;
          lv[u] = LOSS ? __ldg(p.label + o) : 0.f;
          pv[u] = use_p ? __ldg(p.src[k] + o) : 0.f;
          qv[u] = use_q ? __ldg(p.src[4] + o) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (LOSS) {
            const bool pos = lv[u] >= 0.5f;
            float wgt = (pos ? wpos : wneg) * fyv[u];
            if constexpr (VOID) wgt = lv[u] < 0.f ? 0.f : wgt;
            const float yv = pos ? 1.f : 0.f;
            if (use_p) ap = fmaf(wgt, sigmoid(pv[u]) - yv, ap);
            if (use_q) aq = fmaf(wgt, sigmoid(qv[u]) - yv, aq);
          } else {
            ap = fmaf(fyv[u], pv[u], ap);
            aq = fmaf(fyv[u], qv[u], aq);
          }
        }
      }
      if (rgroups > 1) {
        if constexpr (DET) {
          keep_p = ap, keep_q = aq, kept = true;   // rgroups > 1 means width <= wpad: one column per thread
        } else {
          atomicAdd(&colp[c], ap);
          atomicAdd(&colq[c], aq);
        }
      } else {
        colp[c] = ap, colq[c] = aq;
      }
    }
  }
  __syncthreads();
  if constexpr (DET) {
    for (int rr = 0; rr < rgroups && rgroups > 1; ++rr) {
      if (kept && r == rr) colp[c0] += keep_p, colq[c0] += keep_q;
      __syncthreads();
    }
  }
  // phase 2: every low-res pixel of the segment sums its 2s columns; lw = min(32, 2s) lanes per pixel
  const int lw = fs < 32 ? fs : 32;
  const int per_pass = 256 / lw;
  const int sub = tid % lw, grp = tid / lw;
  for (int base = 0; base < nout; base += per_pass) {
    const int oi = base + grp;
    float dp = 0.f, dq = 0.f;
    if (oi < nout) {
      for (int tx = sub; tx < fs; tx += lw) {
        const float fx = 1.f - fabsf(static_cast<float>(tx) - (static_cast<float>(s) - 0.5f)) * inv_s;
        dp = fmaf(fx, colp[oi * s + tx], dp);
        dq = fmaf(fx, colq[oi * s + tx], dq);
      }
    }
    for (int off = lw >> 1; off > 0; off >>= 1) {
      dp += __shfl_xor_sync(0xffffffffu, dp, off);
      dq += __shfl_xor_sync(0xffffffffu, dq, off);
    }
    if (oi < nout && sub == 0) {
      float* dst = sc.dpq + ((static_cast<size_t>(img) * sc.hk + iy) * sc.wk + ix0 + oi) * 2;
      *reinterpret_cast<float2*>(dst) = make_float2(dp * cp, dq * cq);
    }
  }
}

template <bool LOSS, bool DET = false>
__global__ void __launch_bounds__(256) tail_bwd2_kernel(const __grid_constant__ TailBwdParams p) {
  tail_bwd2_body<LOSS, DET, false>(p);
}

template <bool DET>
__global__ void __launch_bounds__(256) tail_bwd2_void_kernel(const __grid_constant__ TailBwdParams p) {
  tail_bwd2_body<true, DET, true>(p);
}

}  // namespace osvos

using namespace osvos;

static void fill_tail_scales(TailParams& p, const float* const* pq, int h, int w) {
  for (int k = 0; k < 4; ++k) {
    const TailGeometry g = tail_geometry(k, h, w);
    TailScale& sc = p.sc[k];
    sc.pq = pq[k];
    sc.hk = g.hk;
    sc.wk = g.wk;
    sc.s = g.s;
    sc.log2s = k + 1;
    sc.inv_s = 1.f / static_cast<float>(g.s);
    sc.top = g.top;
    sc.left = g.left;
  }
}

extern "C" int osvos_tail_fwd(const osvos_tail_fwd_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->n > 0 && a->h > 0 && a->w > 0);
  OSVOS_CHECK_ARG((a->flags & ~(OSVOS_FLAG_DETERMINISTIC | OSVOS_FLAG_VOID_LABELS)) == 0);
  OSVOS_CHECK_ARG(a->label == nullptr || a->sums != nullptr);
  OSVOS_CHECK_ARG(!(a->flags & OSVOS_FLAG_VOID_LABELS) || a->label != nullptr);
  OSVOS_CHECK_ARG(a->losses == nullptr || (a->label != nullptr && a->divisor > 0.f));
  OSVOS_CHECK_ARG(static_cast<size_t>(a->n) * a->h * a->w < (1ull << 31));   // 32-bit element indices in the kernel
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TailParams p;
  for (int k = 0; k < 4; ++k) OSVOS_CHECK_ARG(a->pq[k] != nullptr);
  fill_tail_scales(p, a->pq, a->h, a->w);
  p.vec_mask = 0;
  for (int k = 0; k < 5; ++k) {
    p.out[k] = a->out[k];
    OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->out[k]) & 3) == 0);
    if ((reinterpret_cast<uintptr_t>(a->out[k]) & 15) == 0) p.vec_mask |= 1 << k;
    p.loss_weights[k] = a->loss_weights[k];
  }
  if ((reinterpret_cast<uintptr_t>(a->label) & 15) == 0) p.vec_mask |= 32;
  p.fuse_bias = a->fuse_bias;
  p.label = a->label;
  p.sums = a->sums;
  p.losses = a->losses;
  p.inv_divisor = a->divisor > 0.f ? 1.f / a->divisor : 1.f;
  p.n = a->n;
  p.h = a->h;
  p.w = a->w;
  if (a->sums) OSVOS_CHECK_CUDA(cudaMemsetAsync(a->sums, 0, kTailSums * sizeof(double), stream));
  const size_t blocks = static_cast<size_t>(tail_fwd_blocks(a->n, a->h));
  const size_t smem = sizeof(float2) * (p.sc[0].wk + p.sc[1].wk + p.sc[2].wk + p.sc[3].wk);
  OSVOS_CHECK_ARG(smem <= 48 * 1024);                               // rows up to ~13,000 pixels
  // (with a loss, the memset above is this kernel's stream predecessor: plain launch)
  if (a->flags & OSVOS_FLAG_VOID_LABELS) {
    if (a->flags & OSVOS_FLAG_DETERMINISTIC)
      tail_fwd_void_kernel<true><<<static_cast<int>(blocks), kTailThreads, smem, stream>>>(p);
    else
      tail_fwd_void_kernel<false><<<static_cast<int>(blocks), kTailThreads, smem, stream>>>(p);
  } else if (a->sums && (a->flags & OSVOS_FLAG_DETERMINISTIC))
    tail_fwd_kernel<true><<<static_cast<int>(blocks), kTailThreads, smem, stream>>>(p);
  else if (a->sums)
    tail_fwd_kernel<false><<<static_cast<int>(blocks), kTailThreads, smem, stream>>>(p);
  else
    OSVOS_CHECK_CUDA(launch_pdl(tail_fwd_kernel<false>, dim3(static_cast<unsigned>(blocks)), dim3(kTailThreads), smem,
                                stream, p));
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// segment sizes (low-res columns per work item) per scale: 2s rows x (seg_lo + 1) s columns = 2-4 k source pixels
static int fill_tail_bwd_scales(TailBwdParams& p, float* const* dpq, int n, int h, int w) {
  static const int kSegLo[4] = {255, 63, 15, 7};
  int items = 0;
  for (int k = 0; k < 4; ++k) {
    const TailGeometry g = tail_geometry(k, h, w);
    TailBwdScale& sc = p.sc[k];
    sc.dpq = dpq[k];
    sc.hk = g.hk;
    sc.wk = g.wk;
    sc.s = g.s;
    sc.top = g.top;
    sc.left = g.left;
    sc.seg_lo = kSegLo[k];
    sc.segs = (g.wk + sc.seg_lo - 1) / sc.seg_lo;
    sc.first_item = items;
    items += n * g.hk * sc.segs;
  }
  p.total_items = items;
  return items;
}

extern "C" int osvos_tail_bwd(const osvos_tail_bwd_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->n > 0 && a->h > 0 && a->w > 0);
  OSVOS_CHECK_ARG((a->flags & ~OSVOS_FLAG_DETERMINISTIC) == 0);
  for (int k = 0; k < 4; ++k) OSVOS_CHECK_ARG(a->dpq[k] != nullptr);
  TailBwdParams p;
  memset(&p, 0, sizeof(p));
  const int items = fill_tail_bwd_scales(p, a->dpq, a->n, a->h, a->w);
  for (int k = 0; k < 5; ++k) p.src[k] = a->grad_out[k];
  p.n = a->n, p.h = a->h, p.w = a->w;
  if (a->flags & OSVOS_FLAG_DETERMINISTIC)
    tail_bwd2_kernel<false, true><<<items, 256, 0, static_cast<cudaStream_t>(stream_)>>>(p);
  else
    tail_bwd2_kernel<false><<<items, 256, 0, static_cast<cudaStream_t>(stream_)>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_tail_loss_bwd(const osvos_tail_loss_bwd_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr && a->n > 0 && a->h > 0 && a->w > 0 && a->label != nullptr && a->sums != nullptr);
  OSVOS_CHECK_ARG(a->divisor > 0.f);
  OSVOS_CHECK_ARG((a->flags & ~(OSVOS_FLAG_DETERMINISTIC | OSVOS_FLAG_VOID_LABELS)) == 0);
  for (int k = 0; k < 4; ++k) OSVOS_CHECK_ARG(a->dpq[k] != nullptr);
  for (int k = 0; k < 5; ++k) OSVOS_CHECK_ARG(a->logits[k] != nullptr || a->loss_weights[k] == 0.f);
  TailBwdParams p;
  memset(&p, 0, sizeof(p));
  const int items = fill_tail_bwd_scales(p, a->dpq, a->n, a->h, a->w);
  for (int k = 0; k < 5; ++k) {
    p.src[k] = a->logits[k];
    p.coeff[k] = a->loss_weights[k];
  }
  p.label = a->label;
  p.sums = a->sums;
  p.upstream = a->upstream;
  p.inv_divisor = 1.f / a->divisor;
  p.fuse_bias_grad = a->fuse_bias_grad;
  p.n = a->n, p.h = a->h, p.w = a->w;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool det = (a->flags & OSVOS_FLAG_DETERMINISTIC) != 0;
  if (a->flags & OSVOS_FLAG_VOID_LABELS) {
    if (det)
      tail_bwd2_void_kernel<true><<<items, 256, 0, stream>>>(p);
    else
      tail_bwd2_void_kernel<false><<<items, 256, 0, stream>>>(p);
  } else if (det) {
    tail_bwd2_kernel<true, true><<<items, 256, 0, stream>>>(p);
  } else {
    tail_bwd2_kernel<true><<<items, 256, 0, stream>>>(p);
  }
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" size_t osvos_tail_fwd_deterministic_sums(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return kTailSums + static_cast<size_t>(tail_fwd_blocks(n, h)) * kTailVals;
}

extern "C" size_t osvos_tail_fwd_sums(int n, int h, int w, int flags) {
  if (n <= 0 || h <= 0 || w <= 0 || (flags & ~(OSVOS_FLAG_DETERMINISTIC | OSVOS_FLAG_VOID_LABELS)) != 0) return 0;
  if (!(flags & OSVOS_FLAG_DETERMINISTIC)) return kTailSums;
  const int vals = (flags & OSVOS_FLAG_VOID_LABELS) ? kTailVoidVals : kTailVals;
  return kTailSums + static_cast<size_t>(tail_fwd_blocks(n, h)) * vals;
}

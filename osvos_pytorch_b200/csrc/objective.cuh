// class_balanced_cross_entropy_loss (layers/osvos_layers.py:19-48 of the reference) on the device, one definition for
// the plain objective (loss.cu) and the two side-branch tails that compute it on the fly (tail.cu, tail_general.cu):
//   forward : S_pos = sum_{y=1} (softplus(x) - x), S_neg = sum_{y=0} softplus(x), P = #(y=1), N = #pixels
//             loss = (Nn/N * S_pos + P/N * S_neg) / divisor,  Nn = N - P      (:38-46)
//   backward: dx = w * (sigmoid(x) - y) / divisor, w = y*Nn/N + (1-y)*P/N
// VOID (OSVOS_FLAG_VOID_LABELS): a label y < 0 marks a void pixel, counted in neither class and in no sum; N = #(y >= 0)
// is then counted like P instead of taken from the element count.
// The helpers return numerators and class weights; each caller keeps its own scaling (loss.cu divides by a double
// divisor and folds the upstream gradient into its weights, the tails multiply by a float 1 / divisor).
#pragma once
#include "common.cuh"

namespace osvos {

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + __expf(-x)); }

// A tail's sums (doubles): [2k] / [2k+1] = S_pos / S_neg of map k (the four side maps, then the fused one), [10] = P,
// [11] = N, [12] / [13] = A_pos / A_neg of the fused map (sum_{y=1} (sigmoid(x) - 1), sum_{y=0} sigmoid(x): d fuse.bias
// without another pass), [14] = arrival counter; the deterministic forms put one row of block partials per block behind.
constexpr int kTailSums = OSVOS_TAIL_SUMS;
static_assert(kTailSums == 15, "tail sums layout");
constexpr int kTailVals = 13;       // block partials: sums[0..10], [12], [13]
constexpr int kTailVoidVals = 14;   // the void form also counts N into sums[11]

// where block partial i goes: in order, except that N (the void form's last partial) sits before the A sums
struct TailSlot {
  __device__ __forceinline__ int operator()(int i) const { return i < 11 ? i : i < 13 ? i + 1 : 11; }
};
struct IdentitySlot {
  __device__ __forceinline__ int operator()(int i) const { return i; }
};

// One thread's partial sums over its pixels, in the order of a block's partial row: S_pos / S_neg of each of the M
// logit maps, P, then with FUSED_A the A sums of map M - 1, then with VOID N.
template <int M, bool FUSED_A, bool VOID>
struct CbceSums {
  static constexpr int kVals = 2 * M + 1 + (FUSED_A ? 2 : 0) + (VOID ? 1 : 0);
  float v[kVals] = {};

  // the pixel with the logits x[0..M) and the label y
  __device__ __forceinline__ void add(const float (&x)[M], float y) {
    if constexpr (VOID) {
      if (y < 0.f) return;
      v[kVals - 1] += 1.f;
    }
    const bool pos = y >= 0.5f;
    v[2 * M] += pos ? 1.f : 0.f;
#pragma unroll
    for (int k = 0; k < M; ++k) {
      const float sp = softplus(x[k]);
      if (pos) v[2 * k] += sp - x[k];
      else v[2 * k + 1] += sp;
    }
    if constexpr (FUSED_A) {
      const float sg = sigmoid(x[M - 1]);
      if (pos) v[2 * M + 1] += sg - 1.f;
      else v[2 * M + 2] += sg;
    }
  }
};
static_assert(CbceSums<5, true, false>::kVals == kTailVals && CbceSums<5, true, true>::kVals == kTailVoidVals,
              "a tail's block partials");

// Adds every thread's vals into the grid's sums: shuffles within each warp, then the block's warps in fp64, then either
// one fp64 atomic per value into sums[slot(i)] (zeroed before the launch) or, with DET, a row of kVals doubles per block
// behind the kHeader leading values, which the last block to arrive adds in block order into sums[slot(i)].  The
// arrival counter is sums[kHeader - 1].  Every thread of the kThreads-thread block calls it; it returns true in the last
// block, where the final sums are then readable (with DET, by thread 0 that wrote them).
template <int kThreads, int kHeader, bool DET, int kVals, typename Slot>
__device__ __forceinline__ bool commit_block_sums(float (&vals)[kVals], double* sums, Slot slot) {
  __shared__ float red[kThreads / 32][kVals];
#pragma unroll
  for (int i = 0; i < kVals; ++i)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) vals[i] += __shfl_xor_sync(0xffffffffu, vals[i], off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kVals; ++i) red[warp][i] = vals[i];
  }
  __syncthreads();
  if (threadIdx.x < kVals) {
    double acc = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) acc += static_cast<double>(red[w][threadIdx.x]);
    if constexpr (DET)
      sums[kHeader + kVals * static_cast<size_t>(blockIdx.x) + threadIdx.x] = acc;
    else
      atomicAdd(sums + slot(threadIdx.x), acc);
  }
  const bool last = last_block_arrives(reinterpret_cast<unsigned int*>(sums + kHeader - 1));
  if constexpr (DET) {
    if (last) {
      __shared__ double dred[kThreads];
      for (int i = 0; i < kVals; ++i) {
        const double t = block_ordered_sum(sums + kHeader + i, static_cast<int>(gridDim.x), kVals, dred);
        if (threadIdx.x == 0) sums[slot(i)] = t;
      }
    }
  }
  return last;
}

// Nn/N * S_pos + P/N * S_neg: a map's loss before the division by the divisor
__device__ __forceinline__ double cbce_numerator(double s_pos, double s_neg, double p, double n) {
  return (n - p) / n * s_pos + p / n * s_neg;
}

// the backward's class weights: Nn/N of a positive pixel, P/N of a negative one
__device__ __forceinline__ float cbce_pos_weight(double p, double n) { return static_cast<float>((n - p) / n); }
__device__ __forceinline__ float cbce_neg_weight(double p, double n) { return static_cast<float>(p / n); }

// A tail's forward finish, by thread 0 of the last block after commit_block_sums: N into sums[11] (unless VOID counted
// it), and with `losses` the five maps' losses L_k = numerator_k / divisor (0 when N == 0) and their weighted total.
template <bool VOID>
__device__ __forceinline__ void tail_losses(double* sums, uint32_t total, float* losses, const float* loss_weights,
                                            float inv_divisor) {
  const double tot = VOID ? __ldcg(sums + 11) : static_cast<double>(total);
  const double pcount = __ldcg(sums + 10);
  if constexpr (!VOID) sums[11] = tot;
  if (losses) {
    double wsum = 0.0;
    for (int k = 0; k < 5; ++k) {
      double lk = cbce_numerator(__ldcg(sums + 2 * k), __ldcg(sums + 2 * k + 1), pcount, tot) *
                  static_cast<double>(inv_divisor);
      if constexpr (VOID) lk = tot > 0.0 ? lk : 0.0;
      losses[k] = static_cast<float>(lk);
      wsum += static_cast<double>(loss_weights[k]) * lk;
    }
    losses[5] = static_cast<float>(wsum);
  }
}

// A tail backward's LOSS-mode coefficients for scale k: the class weights, and cp / cq = the loss weight of side map k /
// of the fused map times d(total loss) / divisor (all 0 when VOID and N == 0).  Block 0 also writes d fuse.bias =
// sum_px g_4 from the forward's A sums.  P is a TailBwdParams or a GenBwdParams.
template <bool VOID, typename P>
__device__ __forceinline__ void tail_loss_coeffs(const P& p, int k, float& wpos, float& wneg, float& cp, float& cq) {
  const double pc = p.sums[10], nt = p.sums[11];
  wpos = cbce_pos_weight(pc, nt);
  wneg = cbce_neg_weight(pc, nt);
  const float up = (p.upstream ? __ldg(p.upstream) : 1.f) * p.inv_divisor;
  cp = p.coeff[k] * up;
  cq = p.coeff[4] * up;
  if constexpr (VOID) {
    if (!(nt > 0.0)) wpos = wneg = cp = cq = 0.f;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && p.fuse_bias_grad) {
    if (VOID && !(nt > 0.0))
      p.fuse_bias_grad[0] = 0.f;
    else
      p.fuse_bias_grad[0] = cq * static_cast<float>(cbce_numerator(p.sums[12], p.sums[13], pc, nt));
  }
}

}  // namespace osvos

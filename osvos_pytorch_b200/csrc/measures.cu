// DAVIS-2016 region (J) and boundary (F) measures of fused logit maps against uint8 annotations, as integer counts
// (DESIGN.md §14).  Three launches over bit-packed masks, 32 pixels per word, bit j of word k of a row = column 32k+j;
// bits past the last column are zero in every map, which is what "zeros shifted in" means at the right edge:
//   1. pack:     P = logit > 0, G = byte != 0 -> workspace bit maps; |P∧G| and |P∨G| with popc.  A warp covers one word:
//                every lane reads one pixel and __ballot_sync forms the word, so any mask byte alignment works.
//   2. boundary: B(P), B(G) from four words each (the word, its right neighbour, the two below); |B(P)| and |B(G)|.
//   3. match:    for every word where B(P) (B(G)) has bits, dilate B(G) (B(P)) by the disk at that word and popc the AND;
//                two threads per word, one per direction, so that a 480p frame alone spreads over every SM.
//                Dilation distributes over OR, so rows y-d and y+d (same half-width) are ORed first and dilated once.
//                The loop runs from d = 0 outwards and stops once every boundary bit of the word is matched.
// Counts are reduced per block (warp shuffles, then shared memory) and added with one atomicAdd per block and count.
#include "common.cuh"
#include "merge.cuh"

namespace osvos {

constexpr int kMeasureThreads = 128;
constexpr int kMeasureWarps = kMeasureThreads / 32;

struct MeasureMaps {
  uint32_t* p;    // [n][h][wwords] predicted mask
  uint32_t* g;    // [n][h][wwords] ground truth
  uint32_t* bp;   // [n][h][wwords] boundary of p
  uint32_t* bg;   // [n][h][wwords] boundary of g
};

__host__ __device__ inline int measure_words(int w) { return (w + 31) >> 5; }

// Adds v0 / v1 of every thread of the block into dst[0] / dst[1]; one atomicAdd per block and value.
__device__ __forceinline__ void block_add2(int v0, int v1, int* dst) {
  __shared__ int part[2][kMeasureWarps];
  v0 = __reduce_add_sync(0xffffffffu, v0);
  v1 = __reduce_add_sync(0xffffffffu, v1);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    part[0][warp] = v0;
    part[1][warp] = v1;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    int a = threadIdx.x < kMeasureWarps ? part[0][threadIdx.x] : 0;
    int b = threadIdx.x < kMeasureWarps ? part[1][threadIdx.x] : 0;
    a = __reduce_add_sync(0xffffffffu, a);
    b = __reduce_add_sync(0xffffffffu, b);
    if (threadIdx.x == 0) {
      if (a) atomicAdd(dst, a);
      if (b) atomicAdd(dst + 1, b);
    }
  }
}

// blockIdx.y = frame; warps stride over the frame's h * wwords words.
__global__ void __launch_bounds__(kMeasureThreads)
measures_pack_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ masks, MeasureMaps maps,
                     int* __restrict__ counts, int h, int w) {
  const int f = blockIdx.y;
  const int ww = measure_words(w);
  const int words = h * ww;
  const size_t hw = static_cast<size_t>(h) * w;
  const float* lf = logits + f * hw;
  const uint8_t* mf = masks + f * hw;
  const size_t base = static_cast<size_t>(f) * words;
  const int lane = threadIdx.x & 31;
  int inter = 0, uni = 0;
  for (int i = blockIdx.x * kMeasureWarps + (threadIdx.x >> 5); i < words; i += gridDim.x * kMeasureWarps) {
    const int y = i / ww;
    const int x = ((i - y * ww) << 5) + lane;
    bool p = false, g = false;
    if (x < w) {
      const size_t o = static_cast<size_t>(y) * w + x;
      p = __ldg(lf + o) > 0.f;                    // +0.0 and -0.0 are background
      g = __ldg(mf + o) != 0;
    }
    const uint32_t pw = __ballot_sync(0xffffffffu, p);
    const uint32_t gw = __ballot_sync(0xffffffffu, g);
    if (lane == 0) {
      maps.p[base + i] = pw;
      maps.g[base + i] = gw;
      inter += __popc(pw & gw);
      uni += __popc(pw | gw);
    }
  }
  block_add2(inter, uni, counts + 6 * f);
}

// b = seg^E | seg^S | seg^SE; last row seg^E; last column seg^S; b[h-1][w-1] = 0.
__device__ __forceinline__ uint32_t boundary_word(const uint32_t* __restrict__ seg, int y, int k, int h, int ww,
                                                  uint32_t last_col) {
  const uint32_t* row = seg + static_cast<size_t>(y) * ww;
  const uint32_t c = row[k];
  const uint32_t c1 = k + 1 < ww ? row[k + 1] : 0u;
  const uint32_t e = __funnelshift_r(c, c1, 1);
  if (y == h - 1) return (c ^ e) & ~last_col;
  const uint32_t s = row[ww + k];
  const uint32_t s1 = k + 1 < ww ? row[ww + k + 1] : 0u;
  const uint32_t se = __funnelshift_r(s, s1, 1);
  const uint32_t b = (c ^ e) | (c ^ s) | (c ^ se);
  return (b & ~last_col) | ((c ^ s) & last_col);
}

__global__ void __launch_bounds__(kMeasureThreads)
measures_boundary_kernel(MeasureMaps maps, int* __restrict__ counts, int h, int w) {
  const int f = blockIdx.y;
  const int ww = measure_words(w);
  const int words = h * ww;
  const size_t base = static_cast<size_t>(f) * words;
  const int last_k = ww - 1;
  const uint32_t last_bit = 1u << ((w - 1) & 31);
  int nfg = 0, ngt = 0;
  for (int i = blockIdx.x * kMeasureThreads + threadIdx.x; i < words; i += gridDim.x * kMeasureThreads) {
    const int y = i / ww;
    const int k = i - y * ww;
    const uint32_t last_col = k == last_k ? last_bit : 0u;
    const uint32_t bp = boundary_word(maps.p + base, y, k, h, ww, last_col);
    const uint32_t bg = boundary_word(maps.g + base, y, k, h, ww, last_col);
    maps.bp[base + i] = bp;
    maps.bg[base + i] = bg;
    nfg += __popc(bp);
    ngt += __popc(bg);
  }
  block_add2(nfg, ngt, counts + 6 * f + 2);
}

// OR over dx in [-a, a] of the row shifted so that bit j sees column 32k + j + dx (a < 32: three words suffice).
__device__ __forceinline__ uint32_t hdilate(uint32_t prev, uint32_t cur, uint32_t next, int a) {
  uint64_t right = (static_cast<uint64_t>(next) << 32) | cur;   // >> d: bit j sees j + d
  uint64_t left = (static_cast<uint64_t>(cur) << 32) | prev;    // << d, high word: bit j sees j - d
  int span = 1;                                                 // both cover shifts 0 .. span-1
  while (2 * span <= a + 1) {
    right |= right >> span;
    left |= left << span;
    span *= 2;
  }
  if (span < a + 1) {
    right |= right >> (a + 1 - span);
    left |= left << (a + 1 - span);
  }
  return static_cast<uint32_t>(right) | static_cast<uint32_t>(left >> 32);
}

// Bits of `target` (word k of row y) that the disk-dilated `other` map covers.
__device__ __forceinline__ uint32_t matched_bits(const uint32_t* __restrict__ other, uint32_t target, int y, int k, int h,
                                                 int ww, int r) {
  uint32_t hit = 0;
  int a = r;                                       // half-width of the disk row at distance d: max a with a²+d² <= r²
  for (int d = 0; d <= r; ++d) {
    while (a * a + d * d > r * r) --a;
    uint32_t p = 0, c = 0, n = 0;
#pragma unroll
    for (int sgn = 0; sgn < 2; ++sgn) {
      const int yy = sgn ? y + d : y - d;
      if ((sgn && d == 0) || yy < 0 || yy >= h) continue;
      const uint32_t* row = other + static_cast<size_t>(yy) * ww;
      c |= row[k];
      if (k > 0) p |= row[k - 1];
      if (k + 1 < ww) n |= row[k + 1];
    }
    hit |= hdilate(p, c, n, a) & target;
    if (hit == target) break;
  }
  return hit;
}

__global__ void __launch_bounds__(kMeasureThreads)
measures_match_kernel(MeasureMaps maps, int* __restrict__ counts, int h, int w, int r) {
  const int f = blockIdx.y;
  const int ww = measure_words(w);
  const int words = h * ww;
  const size_t base = static_cast<size_t>(f) * words;
  int fg_match = 0, gt_match = 0;
  for (int t = blockIdx.x * kMeasureThreads + threadIdx.x; t < 2 * words; t += gridDim.x * kMeasureThreads) {
    const int i = t >> 1;
    const int side = t & 1;
    const int y = i / ww;
    const int k = i - y * ww;
    const uint32_t target = (side ? maps.bg : maps.bp)[base + i];
    if (target) {
      const int m = __popc(matched_bits((side ? maps.bp : maps.bg) + base, target, y, k, h, ww, r));
      fg_match += side ? 0 : m;
      gt_match += side ? m : 0;
    }
  }
  block_add2(fg_match, gt_match, counts + 6 * f + 4);
}

// Per-object form (DESIGN.md §24): blockIdx.y = frame f of n; every lane reads its label and annotation byte once and
// the warp forms the K (P, G) words of object k = 1..K, P = label == k, G = gt == k, both cleared where gt == 255
// (void).  Plane f * K + (k - 1) of each map, so the boundary and match kernels run over n * K planes unchanged and
// their counts land in [n][K][6].  |P∧G| and |P∨G| are summed per object in shared memory, one atomicAdd per block,
// object and count.
__global__ void __launch_bounds__(kMeasureThreads)
measures_pack_objects_kernel(const uint8_t* __restrict__ labels, const uint8_t* __restrict__ gt, MeasureMaps maps,
                             int* __restrict__ counts, int nobj, int h, int w) {
  __shared__ int part[2 * OSVOS_DAVIS_MAX_OBJECTS];
  const int f = blockIdx.y;
  const int ww = measure_words(w);
  const int words = h * ww;
  const size_t hw = static_cast<size_t>(h) * w;
  const uint8_t* lf = labels + f * hw;
  const uint8_t* gf = gt + f * hw;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 2 * nobj; i += kMeasureThreads) part[i] = 0;
  __syncthreads();
  for (int i = blockIdx.x * kMeasureWarps + (threadIdx.x >> 5); i < words; i += gridDim.x * kMeasureWarps) {
    const int y = i / ww;
    const int x = ((i - y * ww) << 5) + lane;
    int lab = 0, g = 0;
    if (x < w) {
      const size_t o = static_cast<size_t>(y) * w + x;
      lab = __ldg(lf + o);
      g = __ldg(gf + o);
      if (g == 255) lab = g = 0;                    // void: in neither mask
    }
    // objects present in this word: skip the ballots of the others, their words are zero
    const uint32_t any = __reduce_or_sync(0xffffffffu, (lab <= nobj ? 1u << (lab & 31) : 0u) |
                                                             (g <= nobj ? 1u << (g & 31) : 0u));
    for (int k = 1; k <= nobj; ++k) {
      uint32_t pw = 0, gw = 0;
      if (k >= 32 || (any >> k) & 1u) {
        pw = __ballot_sync(0xffffffffu, lab == k);
        gw = __ballot_sync(0xffffffffu, g == k);
      }
      if (lane == 0) {
        const size_t plane = static_cast<size_t>(f) * nobj + (k - 1);
        maps.p[plane * words + i] = pw;
        maps.g[plane * words + i] = gw;
        const int in = __popc(pw & gw), un = __popc(pw | gw);
        if (in) atomicAdd(&part[2 * (k - 1)], in);
        if (un) atomicAdd(&part[2 * (k - 1) + 1], un);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * nobj; i += kMeasureThreads)
    if (part[i]) atomicAdd(counts + 6 * (static_cast<size_t>(f) * nobj + (i >> 1)) + (i & 1), part[i]);
}

}  // namespace osvos

using namespace osvos;

extern "C" size_t osvos_davis_measures_objects_workspace_bytes(int n, int k, int h, int w) {
  if (n <= 0 || k <= 0 || h <= 0 || w <= 0) return 0;
  return 4 * sizeof(uint32_t) * static_cast<size_t>(n) * k * h * measure_words(w);
}

extern "C" int osvos_davis_measures_objects(const uint8_t* labels, const uint8_t* gt, int* counts, void* workspace,
                                            int n, int k, int h, int w, int r, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(labels != nullptr && gt != nullptr && counts != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(k >= 1 && k <= OSVOS_DAVIS_MAX_OBJECTS);
  OSVOS_CHECK_ARG(n > 0 && static_cast<long long>(n) * k < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768);
  OSVOS_CHECK_ARG(r >= 1 && r <= OSVOS_DAVIS_MAX_RADIUS);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 3) == 0 && (reinterpret_cast<uintptr_t>(counts) & 3) == 0);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int planes = n * k;
  const size_t plane = static_cast<size_t>(planes) * h * measure_words(w);
  uint32_t* ws = static_cast<uint32_t*>(workspace);
  const MeasureMaps maps{ws, ws + plane, ws + 2 * plane, ws + 3 * plane};
  const int words = h * measure_words(w);
  const int sms = device_sm_count();
  const int per_frame = max(1, (8 * sms + n - 1) / n);
  const int per_plane = max(1, (8 * sms + planes - 1) / planes);
  const dim3 grid_pack(min(per_frame, (words + kMeasureWarps - 1) / kMeasureWarps), n);
  const dim3 grid_word(min(per_plane, (words + kMeasureThreads - 1) / kMeasureThreads), planes);
  const dim3 grid_match(min(per_plane, (2 * words + kMeasureThreads - 1) / kMeasureThreads), planes);
  OSVOS_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 6 * static_cast<size_t>(planes), stream));
  measures_pack_objects_kernel<<<grid_pack, kMeasureThreads, 0, stream>>>(labels, gt, maps, counts, k, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  measures_boundary_kernel<<<grid_word, kMeasureThreads, 0, stream>>>(maps, counts, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  measures_match_kernel<<<grid_match, kMeasureThreads, 0, stream>>>(maps, counts, h, w, r);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// ---- merge of per-object fused maps (DESIGN.md §24) ------------------------------------------------------------------

namespace osvos {

// label = 1 + the first k of the largest logit if that logit is > 0, else 0: `best` starts at +0 and only a strictly
// larger value replaces it, so ±0 and NaN never win and ties go to the lowest k.  Four pixels per thread; float4 loads
// when every map is 16-byte aligned (vec), one 32-bit store when out is 4-byte aligned too.
template <bool VEC>
__global__ void __launch_bounds__(256) merge_objects_kernel(MergeMaps maps, int nobj, uint8_t* __restrict__ out,
                                                            long long pixels) {
  const long long quads = (pixels + 3) >> 2;
  const bool out_aligned = (reinterpret_cast<uintptr_t>(out) & 3) == 0;
  for (long long q = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; q < quads;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long i0 = q << 2;
    float best[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t lab[4] = {0, 0, 0, 0};
    const bool full = i0 + 4 <= pixels;
    for (int k = 0; k < nobj; ++k) {
      float v[4];
      if (VEC && full) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(maps.map[k] + i0));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = i0 + j < pixels ? __ldg(maps.map[k] + i0 + j) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (v[j] > best[j]) {
          best[j] = v[j];
          lab[j] = k + 1;
        }
      }
    }
    if (full && out_aligned) {
      *reinterpret_cast<uint32_t*>(out + i0) = lab[0] | (lab[1] << 8) | (lab[2] << 16) | (lab[3] << 24);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (i0 + j < pixels) out[i0 + j] = static_cast<uint8_t>(lab[j]);
    }
  }
}

}  // namespace osvos

extern "C" int osvos_merge_objects(const float* const* maps, int k, uint8_t* out, size_t pixels,
                                   osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(maps != nullptr && out != nullptr && pixels > 0);
  OSVOS_CHECK_ARG(k >= 1 && k <= OSVOS_MERGE_MAX_OBJECTS);
  MergeMaps m{};
  bool vec = true;
  for (int i = 0; i < k; ++i) {
    OSVOS_CHECK_ARG(maps[i] != nullptr && (reinterpret_cast<uintptr_t>(maps[i]) & 3) == 0);
    vec = vec && (reinterpret_cast<uintptr_t>(maps[i]) & 15) == 0;
    m.map[i] = maps[i];
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long quads = (static_cast<long long>(pixels) + 3) >> 2;
  const unsigned blocks = static_cast<unsigned>(min(static_cast<long long>(16 * device_sm_count()), (quads + 255) / 256));
  if (vec)
    merge_objects_kernel<true><<<blocks, 256, 0, stream>>>(m, k, out, static_cast<long long>(pixels));
  else
    merge_objects_kernel<false><<<blocks, 256, 0, stream>>>(m, k, out, static_cast<long long>(pixels));
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" size_t osvos_davis_measures_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return 4 * sizeof(uint32_t) * static_cast<size_t>(n) * h * measure_words(w);
}

extern "C" int osvos_davis_measures(const float* logits, const uint8_t* masks, int* counts, void* workspace, int n,
                                    int h, int w, int r, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(logits != nullptr && masks != nullptr && counts != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(n > 0 && n < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768);
  OSVOS_CHECK_ARG(r >= 1 && r <= OSVOS_DAVIS_MAX_RADIUS);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 3) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 3) == 0);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t plane = static_cast<size_t>(n) * h * measure_words(w);
  uint32_t* ws = static_cast<uint32_t*>(workspace);
  const MeasureMaps maps{ws, ws + plane, ws + 2 * plane, ws + 3 * plane};
  const int words = h * measure_words(w);
  // about eight blocks per SM over the whole batch, and no more blocks per frame than the frame has work for
  const int per_frame = max(1, (8 * device_sm_count() + n - 1) / n);
  const dim3 grid_pack(min(per_frame, (words + kMeasureWarps - 1) / kMeasureWarps), n);
  const dim3 grid_word(min(per_frame, (words + kMeasureThreads - 1) / kMeasureThreads), n);
  OSVOS_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 6 * n, stream));
  measures_pack_kernel<<<grid_pack, kMeasureThreads, 0, stream>>>(logits, masks, maps, counts, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  measures_boundary_kernel<<<grid_word, kMeasureThreads, 0, stream>>>(maps, counts, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  const dim3 grid_match(min(per_frame, (2 * words + kMeasureThreads - 1) / kMeasureThreads), n);
  measures_match_kernel<<<grid_match, kMeasureThreads, 0, stream>>>(maps, counts, h, w, r);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// Fully connected CRF (Krähenbühl & Koltun 2011) with Potts labels, mean-field on the device (DESIGN.md §29).
//
// One call, every frame of the batch:
//   1. crf_elevate_kernel: each pixel's feature (x, y, R, G, B) scaled and elevated onto the permutohedral lattice in R⁶
//      (Adams, Baek & Davis 2010), its enclosing simplex's 6 vertices as packed 64-bit keys (frame in the top bits, so
//      no vertex is shared between frames) and the barycentric weights.  Float64, unfused, in the order of DESIGN §29,
//      so tests/crf_ref.py reproduces keys and weights bit for bit.
//   2. CUB radix sort of the 6·P (key, entry) pairs (stable), a mark of each new key, an inclusive scan: the vertex of
//      every entry, the sorted unique keys and each vertex's segment of entries.  Nothing depends on insertion order.
//   3. crf_neighbours_kernel: each vertex's 12 blur neighbours, by binary search in the unique keys; found once, used by
//      every splat/blur/slice of the call.
//   4. The normaliser F(1) (splat of the weights, blur, slice), then T mean-field iterations of: splat the K+1 label
//      probabilities (a fixed-order sum over each vertex's sorted segment), 6 blur passes, slice, the exact truncated
//      Gaussian (rows, then columns fused with the update and the softmax).
// The vertex count is data dependent: buffers are sized by 6 vertices per pixel and the kernels read the count from the
// workspace (grid-stride loops), so nothing is read back to the host.  There are no atomics: every output element is
// one thread's fixed-order sum, whatever the launch configuration.
#include <math.h>

#include <cub/cub.cuh>

#include "common.cuh"
#include "merge.cuh"

namespace osvos {
namespace {

constexpr int kD = 5;               // feature dimensions (x, y, R, G, B)
constexpr int kD1 = kD + 1;         // lattice coordinates, simplex vertices per pixel
constexpr int kQBits = 10;          // bits per packed coordinate quotient
constexpr int kQBias = 1 << (kQBits - 1);
constexpr int kQMax = (1 << kQBits) - 1;
constexpr int kKeyBits = kD * kQBits + 3;   // 5 quotients + the remainder class (0..5)
constexpr int kFrameBits = 64 - kKeyBits;   // 11: up to 2048 frames per call
constexpr int kThreads = 256;
constexpr int kMaxBlocks = 4096;
constexpr int kSplatBlocks = 2048;  // block-per-vertex loop

struct Scales {
  double s[kD];       // sqrt(2/3)·(d+1) / sqrt((j+1)(j+2)) / θ_j, computed on the host
  double down;        // 1 / (d+1)
};

// Coordinate key[i] ≡ r (mod 6) for every i of a vertex of remainder class r: key = 6·q_i + r; the 6th coordinate is
// minus the sum of the other five, so (frame, r, q_0..q_4) identify the vertex.
__host__ __device__ inline uint64_t pack_key(uint64_t frame, int r, const int* q) {
  uint64_t k = frame << kKeyBits | static_cast<uint64_t>(r) << (kD * kQBits);
  for (int i = 0; i < kD; ++i) k |= static_cast<uint64_t>(q[i] + kQBias) << (i * kQBits);
  return k;
}

__device__ __forceinline__ int floor_div6(int a) { return a >= 0 ? a / 6 : -((5 - a) / 6); }

// Grid-stride bound helpers.
__device__ __forceinline__ size_t gtid() { return static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; }
__device__ __forceinline__ size_t gstride() { return static_cast<size_t>(gridDim.x) * blockDim.x; }

// 1. one thread per pixel: keys_in / vals_in / wts at entries 6p .. 6p+5.
__global__ void __launch_bounds__(kThreads)
crf_elevate_kernel(const uint8_t* __restrict__ frames, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                   float* __restrict__ wts, int h, int w, size_t pixels, Scales sc) {
  const size_t hw = static_cast<size_t>(h) * w;
  for (size_t p = gtid(); p < pixels; p += gstride()) {
    const size_t f = p / hw, o = p - f * hw;
    const int y = static_cast<int>(o / w), x = static_cast<int>(o - static_cast<size_t>(y) * w);
    const uint8_t* px = frames + 3 * p;                 // BGR
    const double v[kD] = {static_cast<double>(x), static_cast<double>(y), static_cast<double>(px[2]),
                          static_cast<double>(px[1]), static_cast<double>(px[0])};
    double e[kD1];
    double sm = 0.0;
#pragma unroll
    for (int j = kD; j > 0; --j) {
      const double cf = __dmul_rn(v[j - 1], sc.s[j - 1]);
      e[j] = __dadd_rn(sm, -__dmul_rn(static_cast<double>(j), cf));
      sm = __dadd_rn(sm, cf);
    }
    e[0] = sm;
    // the closest remainder-0 point
    int rem0[kD1], rank[kD1];
    int sum = 0;
#pragma unroll
    for (int i = 0; i < kD1; ++i) {
      const double t = __dmul_rn(e[i], sc.down);
      const double up = ceil(t) * kD1, dn = floor(t) * kD1;      // exact: small integers
      rem0[i] = static_cast<int>(__dadd_rn(up, -e[i]) < __dadd_rn(e[i], -dn) ? up : dn);
      sum += rem0[i];
      rank[i] = 0;
    }
    sum /= kD1;
    double dif[kD1];
#pragma unroll
    for (int i = 0; i < kD1; ++i) dif[i] = __dadd_rn(e[i], -static_cast<double>(rem0[i]));
#pragma unroll
    for (int i = 0; i < kD; ++i)
#pragma unroll
      for (int j = i + 1; j < kD1; ++j) {
        if (dif[i] < dif[j]) ++rank[i];
        else ++rank[j];
      }
#pragma unroll
    for (int i = 0; i < kD1; ++i) {
      if (sum > 0) {
        if (rank[i] >= kD1 - sum) { rem0[i] -= kD1; rank[i] += sum - kD1; }
        else rank[i] += sum;
      } else if (sum < 0) {
        if (rank[i] < -sum) { rem0[i] += kD1; rank[i] += kD1 + sum; }
        else rank[i] += sum;
      }
    }
    // barycentric weights: slot s gets +v_i from the i of rank d - s and -v_i from the i of rank d + 1 - s
    double vi[kD1];
#pragma unroll
    for (int i = 0; i < kD1; ++i) vi[i] = __dmul_rn(__dadd_rn(e[i], -static_cast<double>(rem0[i])), sc.down);
    double bary[kD1 + 1];
#pragma unroll
    for (int s = 0; s <= kD1; ++s) {
      double plus = 0.0, minus = 0.0;
#pragma unroll
      for (int i = 0; i < kD1; ++i) {
        if (rank[i] == kD - s) plus = vi[i];
        if (rank[i] == kD1 - s) minus = vi[i];
      }
      bary[s] = __dadd_rn(plus, -minus);
    }
    bary[0] = __dadd_rn(bary[0], __dadd_rn(1.0, bary[kD1]));
#pragma unroll
    for (int r = 0; r < kD1; ++r) {
      int q[kD];
#pragma unroll
      for (int i = 0; i < kD; ++i) {
        const int k = rem0[i] + r - (rank[i] > kD - r ? kD1 : 0);
        q[i] = floor_div6(k - r);
      }
      const size_t ent = kD1 * p + r;
      keys[ent] = pack_key(f, r, q);
      vals[ent] = static_cast<uint32_t>(ent);
      wts[ent] = static_cast<float>(bary[r]);
    }
  }
}

// 2a. flag[e] = 1 where the sorted key differs from its predecessor.
__global__ void __launch_bounds__(kThreads)
crf_mark_kernel(const uint64_t* __restrict__ keys, int* __restrict__ flag, size_t entries) {
  for (size_t e = gtid(); e < entries; e += gstride()) flag[e] = e == 0 || keys[e] != keys[e - 1];
}

// 2b. vid = inclusive scan of the flags: vertex vid[e] - 1 of sorted entry e.  Unique keys, segment starts, the vertex
// of every original entry, each frame's first vertex, and the vertex total at counts[n].
__global__ void __launch_bounds__(kThreads)
crf_compact_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const int* __restrict__ vid,
                   uint64_t* __restrict__ ukey, uint32_t* __restrict__ seg, int* __restrict__ pv,
                   int* __restrict__ counts, int* __restrict__ fstart, size_t entries, int n) {
  for (size_t e = gtid(); e < entries; e += gstride()) {
    const int v = vid[e] - 1;
    pv[vals[e]] = v;
    if (e == 0 || vid[e - 1] != vid[e]) {
      ukey[v] = keys[e];
      seg[v] = static_cast<uint32_t>(e);
      const int fr = static_cast<int>(keys[e] >> kKeyBits);
      if (e == 0 || static_cast<int>(keys[e - 1] >> kKeyBits) != fr) fstart[fr] = v;
    }
    if (e == entries - 1) {
      counts[n] = v + 1;
      seg[v + 1] = static_cast<uint32_t>(entries);
    }
  }
}

__device__ __forceinline__ int find_key(const uint64_t* __restrict__ ukey, int m, uint64_t key) {
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ukey[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo < m && ukey[lo] == key ? lo : -1;
}

// 3. nbr[(2j + s) * cap + v], s = 0: key - 1 with coordinate j + (d+1); s = 1: key + 1 with coordinate j - (d+1)
// (direction j = d moves the five stored coordinates only).  -1: absent.  Also each frame's vertex count.
__global__ void __launch_bounds__(kThreads)
crf_neighbours_kernel(const uint64_t* __restrict__ ukey, int* __restrict__ nbr, int* __restrict__ counts,
                      const int* __restrict__ fstart, size_t cap, int n) {
  const int m = counts[n];
  for (size_t vv = gtid(); vv < static_cast<size_t>(m); vv += gstride()) {
    const int v = static_cast<int>(vv);
    const uint64_t key = ukey[v];
    const uint64_t fr = key >> kKeyBits;
    if (v == m - 1 || (ukey[v + 1] >> kKeyBits) != fr) counts[fr] = v + 1 - fstart[fr];
    const int r = static_cast<int>((key >> (kD * kQBits)) & 7);
    int k[kD];
#pragma unroll
    for (int i = 0; i < kD; ++i) k[i] = 6 * (static_cast<int>((key >> (i * kQBits)) & kQMax) - kQBias) + r;
#pragma unroll
    for (int j = 0; j < kD1; ++j) {
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int step = s == 0 ? -1 : 1;
        const int r2 = (r + step + kD1) % kD1;
        int q[kD];
        bool inside = true;
#pragma unroll
        for (int i = 0; i < kD; ++i) {
          const int c = k[i] + step - (i == j ? step * kD1 : 0);
          q[i] = floor_div6(c - r2);
          inside = inside && q[i] + kQBias >= 0 && q[i] + kQBias <= kQMax;
        }
        nbr[(2 * j + s) * cap + v] = inside ? find_key(ukey, m, pack_key(fr, r2, q)) : -1;
      }
    }
  }
}

// 4a. splat: val[c][v] = Σ over v's sorted segment of w_e · Q[c][pixel(e)] (Q == nullptr: the weights alone).  One
// block per vertex (a vertex of a flat region can hold most of a frame's pixels): thread t adds entries t, t + 256, ...
// in order, then a fixed shuffle tree per warp and warp 0 adds the 8 warp sums in order.
__global__ void __launch_bounds__(kThreads)
crf_splat_kernel(const float* __restrict__ q, const float* __restrict__ wts, const uint32_t* __restrict__ vals,
                 const uint32_t* __restrict__ seg, const int* __restrict__ counts, float* __restrict__ val, int channels,
                 size_t pixels, size_t cap, int n) {
  __shared__ float part[kThreads / 32];
  const int m = counts[n];
  for (int v = blockIdx.x; v < m; v += gridDim.x) {
    const uint32_t b = seg[v], e = seg[v + 1];
    for (int c = 0; c < channels; ++c) {
      float s = 0.f;
      for (uint32_t i = b + threadIdx.x; i < e; i += kThreads) {
        const uint32_t ent = vals[i];
        const float wv = wts[ent];
        s += q == nullptr ? wv : wv * q[c * pixels + ent / kD1];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      __syncthreads();                                   // `part` may still be read for the previous channel
      if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
      __syncthreads();
      if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < kThreads / 32; ++i) t += part[i];
        val[c * cap + v] = t;
      }
    }
  }
}

// 4b. blur along direction j: ½ v + ¼ (v⁻ + v⁺), absent neighbours 0.
__global__ void __launch_bounds__(kThreads)
crf_blur_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ nbr,
                const int* __restrict__ counts, int channels, size_t cap, int n) {
  const int m = counts[n];
  for (size_t v = gtid(); v < static_cast<size_t>(m); v += gstride()) {
    const int a = nbr[v], b = nbr[cap + v];
    for (int c = 0; c < channels; ++c) {
      const float* x = in + c * cap;
      const float na = a >= 0 ? x[a] : 0.f, nb = b >= 0 ? x[b] : 0.f;
      out[c * cap + v] = 0.5f * x[v] + 0.25f * (na + nb);
    }
  }
}

// 4c. slice: F[c][p] = Σ_r w_{6p+r} · val[c][vertex(6p+r)], r ascending; norm == nullptr: store F (the F(1) pass), else
// store F / norm[p].
__global__ void __launch_bounds__(kThreads)
crf_slice_kernel(const float* __restrict__ val, const float* __restrict__ wts, const int* __restrict__ pv,
                 const float* __restrict__ norm, float* __restrict__ out, int channels, size_t pixels, size_t cap) {
  for (size_t p = gtid(); p < pixels; p += gstride()) {
    int vtx[kD1];
    float wr[kD1];
#pragma unroll
    for (int r = 0; r < kD1; ++r) {
      vtx[r] = pv[kD1 * p + r];
      wr[r] = wts[kD1 * p + r];
    }
    const float inv = norm == nullptr ? 1.f : 1.f / norm[p];
    for (int c = 0; c < channels; ++c) {
      const float* x = val + c * cap;
      float s = 0.f;
#pragma unroll
      for (int r = 0; r < kD1; ++r) s += wr[r] * x[vtx[r]];
      out[c * pixels + p] = norm == nullptr ? s : s * inv;
    }
  }
}

// Gaussian taps g[0..R] = exp(-d² / (2θγ²)), in float64 rounded to fp32.
__global__ void __launch_bounds__(kThreads)
crf_taps_kernel(float* __restrict__ g, int radius, double inv2s2) {
  for (size_t d = gtid(); d <= static_cast<size_t>(radius); d += gstride())
    g[d] = static_cast<float>(exp(-static_cast<double>(d) * static_cast<double>(d) * inv2s2));
}

// 4d. rows: t[c][p] = Σ_{dx ascending, inside the row} g[|dx|] · Q[c][p + dx].
__global__ void __launch_bounds__(kThreads)
crf_gauss_rows_kernel(const float* __restrict__ q, const float* __restrict__ g, float* __restrict__ t, int channels,
                      int w, size_t pixels, int radius) {
  for (size_t p = gtid(); p < pixels; p += gstride()) {
    const int x = static_cast<int>(p % w);
    const int lo = max(-radius, -x), hi = min(radius, w - 1 - x);
    for (int c = 0; c < channels; ++c) {
      const float* row = q + c * pixels + p;
      float s = 0.f;
      for (int dx = lo; dx <= hi; ++dx) s += g[abs(dx)] * row[dx];
      t[c * pixels + p] = s;
    }
  }
}

// 4e. columns of t (the smoothness message S after dividing by the in-frame tap sums), the update
// a_l = a⁰_l + w_α·B_l + w_γ·S_l with a⁰ = (0, z_1..z_K), and either Q = softmax(a) or, in the last iteration,
// out[k-1] = a_k - a_0.  INIT: a = a⁰ (no messages are read).
template <bool INIT, bool LAST>
__global__ void __launch_bounds__(kThreads)
crf_update_kernel(const MergeMaps maps, const float* __restrict__ bmsg, const float* __restrict__ g,
                  float* __restrict__ a, const float* __restrict__ t, float* __restrict__ q, float* __restrict__ out,
                  int k, int h, int w, size_t pixels, int radius, float w_a, float w_g) {
  const size_t hw = static_cast<size_t>(h) * w;
  const int channels = k + 1;
  for (size_t p = gtid(); p < pixels; p += gstride()) {
    float inv = 0.f;
    int lo = 0, hi = 0;
    if (!INIT) {
      const size_t o = p % hw;
      const int y = static_cast<int>(o / w), x = static_cast<int>(o % w);
      const int xl = max(-radius, -x), xh = min(radius, w - 1 - x);
      lo = max(-radius, -y);
      hi = min(radius, h - 1 - y);
      float nx = 0.f, ny = 0.f;
      for (int d = xl; d <= xh; ++d) nx += g[abs(d)];
      for (int d = lo; d <= hi; ++d) ny += g[abs(d)];
      inv = 1.f / (nx * ny);
    }
    float mx = -INFINITY;
    for (int c = 0; c < channels; ++c) {
      float v = c == 0 ? 0.f : maps.map[c - 1][p];
      if (!INIT) {
        const float* col = t + c * pixels + p;
        float s = 0.f;
        for (int dy = lo; dy <= hi; ++dy) s += g[abs(dy)] * col[static_cast<ptrdiff_t>(dy) * w];
        v = v + w_a * bmsg[c * pixels + p] + w_g * (s * inv);
      }
      a[c * pixels + p] = v;
      mx = fmaxf(mx, v);
    }
    if (LAST) {
      const float a0 = a[p];
      for (int c = 1; c < channels; ++c) out[(c - 1) * pixels + p] = a[c * pixels + p] - a0;
    } else {
      float z = 0.f;
      for (int c = 0; c < channels; ++c) z += expf(a[c * pixels + p] - mx);
      const float iz = 1.f / z;
      for (int c = 0; c < channels; ++c) q[c * pixels + p] = expf(a[c * pixels + p] - mx) * iz;
    }
  }
}

// Workspace layout; every region 256-byte aligned.
struct Layout {
  size_t counts, fstart, keys_in, keys_out, vals_in, vals_out, wts, vid, ukey, seg, pv, nbr, val0, val1, norm, q, bmsg,
      a, t, taps, cub, cub_bytes, total;
};

size_t align256(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

// Host-side limits: the packed keys' range, index widths, frames per call.  Returns false when refused.
bool crf_fits(int n, int k, int h, int w, double theta_a, double theta_b, Scales* sc) {
  if (n <= 0 || n > (1 << kFrameBits) || h <= 0 || w <= 0 || h >= 32768 || w >= 32768) return false;
  if (k < 1 || k > OSVOS_MERGE_MAX_OBJECTS) return false;
  if (!(theta_a > 0.0) || !(theta_b > 0.0) || !isfinite(theta_a) || !isfinite(theta_b)) return false;
  const size_t entries = static_cast<size_t>(kD1) * n * h * w;
  if (entries >= (static_cast<size_t>(1) << 31) - 1) return false;
  const double inv_std = sqrt(2.0 / 3.0) * kD1;
  const double theta[kD] = {theta_a, theta_a, theta_b, theta_b, theta_b};
  const double vmax[kD] = {static_cast<double>(w - 1), static_cast<double>(h - 1), 255.0, 255.0, 255.0};
  double cfmax[kD];
  for (int j = 0; j < kD; ++j) {
    sc->s[j] = inv_std / sqrt(static_cast<double>((j + 1) * (j + 2))) / theta[j];
    cfmax[j] = vmax[j] * sc->s[j];
  }
  sc->down = 1.0 / kD1;
  // elevated[j] lies in [-j·cf_{j-1}, Σ_{i>=j} cf_i] (cf >= 0); a key coordinate is within 3 + 6 + 5 of it
  double bound = 0.0;
  for (int j = 0; j <= kD; ++j) {
    double hi = 0.0;
    for (int i = j; i < kD; ++i) hi += cfmax[i];
    const double lo = j > 0 ? j * cfmax[j - 1] : 0.0;
    bound = fmax(bound, fmax(hi, lo));
  }
  // |q| = |(key - r) / 6| <= (bound + 1 + 14 + 5) / 6 must stay below kQBias (one step to spare for the neighbours)
  return isfinite(bound) && (bound + 20.0) / kD1 + 1.0 < kQBias - 1;
}

Layout crf_layout(int n, int k, int h, int w, size_t cub_bytes) {
  const size_t pixels = static_cast<size_t>(n) * h * w, cap = kD1 * pixels, ch = static_cast<size_t>(k) + 1;
  Layout l;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o = align256(o + bytes); return at; };
  l.counts = take(sizeof(int) * (n + 1));
  l.fstart = take(sizeof(int) * n);
  l.keys_in = take(sizeof(uint64_t) * cap);
  l.keys_out = take(sizeof(uint64_t) * cap);
  l.vals_in = take(sizeof(uint32_t) * cap);
  l.vals_out = take(sizeof(uint32_t) * cap);
  l.wts = take(sizeof(float) * cap);
  l.vid = take(sizeof(int) * cap);
  l.ukey = take(sizeof(uint64_t) * cap);
  l.seg = take(sizeof(uint32_t) * (cap + 1));
  l.pv = take(sizeof(int) * cap);
  l.nbr = take(sizeof(int) * 2 * kD1 * cap);
  l.val0 = take(sizeof(float) * ch * cap);
  l.val1 = take(sizeof(float) * ch * cap);
  l.norm = take(sizeof(float) * pixels);
  l.q = take(sizeof(float) * ch * pixels);
  l.bmsg = take(sizeof(float) * ch * pixels);
  l.a = take(sizeof(float) * ch * pixels);
  l.t = take(sizeof(float) * ch * pixels);
  l.taps = take(sizeof(float) * (h > w ? h : w));
  l.cub = take(cub_bytes);
  l.cub_bytes = cub_bytes;
  l.total = o;
  return l;
}

int key_end_bit(int n) {
  int b = 0;
  while ((1 << b) < n) ++b;
  return kKeyBits + b;
}

// Temporary storage of the sort and the scan (host query; CUB launches nothing when asked for sizes).
cudaError_t crf_cub_bytes(int n, size_t entries, size_t* bytes) {
  size_t sort = 0, scan = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort, static_cast<const uint64_t*>(nullptr),
                                                  static_cast<uint64_t*>(nullptr), static_cast<const uint32_t*>(nullptr),
                                                  static_cast<uint32_t*>(nullptr), static_cast<int>(entries), 0,
                                                  key_end_bit(n));
  if (e != cudaSuccess) return e;
  e = cub::DeviceScan::InclusiveSum(nullptr, scan, static_cast<const int*>(nullptr), static_cast<int*>(nullptr),
                                    static_cast<int>(entries));
  *bytes = sort > scan ? sort : scan;
  return e;
}

int grid_for(size_t items) {
  const size_t b = (items + kThreads - 1) / kThreads;
  return static_cast<int>(b < kMaxBlocks ? (b > 0 ? b : 1) : kMaxBlocks);
}

}  // namespace
}  // namespace osvos

using namespace osvos;

extern "C" size_t osvos_dense_crf_workspace_bytes(int n, int k, int h, int w) {
  Scales sc;
  if (!crf_fits(n, k, h, w, 1e30, 1e30, &sc)) return 0;    // sizes only; the key range is checked by the call
  size_t cub_bytes = 0;
  if (crf_cub_bytes(n, static_cast<size_t>(kD1) * n * h * w, &cub_bytes) != cudaSuccess) return 0;
  return crf_layout(n, k, h, w, cub_bytes).total;
}

extern "C" int osvos_dense_crf(const uint8_t* frames, const float* const* maps, float* out, void* workspace, int n,
                               int k, int h, int w, int iterations, float w_a, double theta_a, double theta_b,
                               float w_g, double theta_g, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(frames != nullptr && maps != nullptr && out != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(n > 0 && k >= 1 && k <= OSVOS_MERGE_MAX_OBJECTS && h > 0 && w > 0 && h < 32768 && w < 32768);
  OSVOS_CHECK_ARG(n <= (1 << kFrameBits));
  OSVOS_CHECK_ARG(iterations >= 0);
  OSVOS_CHECK_ARG(isfinite(w_a) && w_a >= 0.f && isfinite(w_g) && w_g >= 0.f);
  OSVOS_CHECK_ARG(isfinite(theta_a) && theta_a > 0.0 && isfinite(theta_b) && theta_b > 0.0 && isfinite(theta_g) &&
                  theta_g > 0.0);
  for (int i = 0; i < k; ++i)
    OSVOS_CHECK_ARG(maps[i] != nullptr && (reinterpret_cast<uintptr_t>(maps[i]) & 3) == 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 3) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0);
  Scales sc;
  OSVOS_CHECK_ARG(crf_fits(n, k, h, w, theta_a, theta_b, &sc));     // the packed keys hold every coordinate
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t pixels = static_cast<size_t>(n) * h * w, cap = kD1 * pixels;
  if (iterations == 0) {                                             // r_k = z_k, bit for bit
    for (int i = 0; i < k; ++i)
      OSVOS_CHECK_CUDA(cudaMemcpyAsync(out + i * pixels, maps[i], sizeof(float) * pixels, cudaMemcpyDeviceToDevice,
                                       stream));
    return OSVOS_OK;
  }
  size_t cub_bytes = 0;
  OSVOS_CHECK_CUDA(crf_cub_bytes(n, cap, &cub_bytes));
  const Layout l = crf_layout(n, k, h, w, cub_bytes);
  char* ws = static_cast<char*>(workspace);
  auto at = [&](size_t off) { return static_cast<void*>(ws + off); };
  int* counts = static_cast<int*>(at(l.counts));
  int* fstart = static_cast<int*>(at(l.fstart));
  uint64_t* keys_in = static_cast<uint64_t*>(at(l.keys_in));
  uint64_t* keys_out = static_cast<uint64_t*>(at(l.keys_out));
  uint32_t* vals_in = static_cast<uint32_t*>(at(l.vals_in));
  uint32_t* vals_out = static_cast<uint32_t*>(at(l.vals_out));
  float* wts = static_cast<float*>(at(l.wts));
  int* vid = static_cast<int*>(at(l.vid));
  int* flag = reinterpret_cast<int*>(vals_in);                       // free once the sort has run
  uint64_t* ukey = static_cast<uint64_t*>(at(l.ukey));
  uint32_t* seg = static_cast<uint32_t*>(at(l.seg));
  int* pv = static_cast<int*>(at(l.pv));
  int* nbr = static_cast<int*>(at(l.nbr));
  float* val[2] = {static_cast<float*>(at(l.val0)), static_cast<float*>(at(l.val1))};
  float* norm = static_cast<float*>(at(l.norm));
  float* q = static_cast<float*>(at(l.q));
  float* bmsg = static_cast<float*>(at(l.bmsg));
  float* a = static_cast<float*>(at(l.a));
  float* t = static_cast<float*>(at(l.t));
  float* taps = static_cast<float*>(at(l.taps));
  MergeMaps zmaps;
  for (int i = 0; i < k; ++i) zmaps.map[i] = maps[i];
  // taps beyond the frame are never read
  const int radius = static_cast<int>(fmin(ceil(3.0 * theta_g), static_cast<double>((h > w ? h : w) - 1)));
  const double inv2s2 = 1.0 / (2.0 * theta_g * theta_g);

  const int gp = grid_for(pixels), ge = grid_for(cap);
  // 1-3: the lattice
  crf_elevate_kernel<<<gp, kThreads, 0, stream>>>(frames, keys_in, vals_in, wts, h, w, pixels, sc);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  size_t tb = l.cub_bytes;
  OSVOS_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(at(l.cub), tb, keys_in, keys_out, vals_in, vals_out,
                                                   static_cast<int>(cap), 0, key_end_bit(n), stream));
  crf_mark_kernel<<<ge, kThreads, 0, stream>>>(keys_out, flag, cap);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  tb = l.cub_bytes;
  OSVOS_CHECK_CUDA(cub::DeviceScan::InclusiveSum(at(l.cub), tb, flag, vid, static_cast<int>(cap), stream));
  crf_compact_kernel<<<ge, kThreads, 0, stream>>>(keys_out, vals_out, vid, ukey, seg, pv, counts, fstart, cap, n);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  crf_neighbours_kernel<<<ge, kThreads, 0, stream>>>(ukey, nbr, counts, fstart, cap, n);
  OSVOS_CHECK_CUDA(cudaGetLastError());

  const int ch = k + 1;
  // splat -> 6 blur passes -> slice; the result is in val[0] after an even number of passes
  auto filter = [&](const float* src, int channels, const float* nrm, float* dst) -> cudaError_t {
    crf_splat_kernel<<<kSplatBlocks, kThreads, 0, stream>>>(src, wts, vals_out, seg, counts, val[0], channels, pixels, cap, n);
    for (int j = 0; j < kD1; ++j)
      crf_blur_kernel<<<ge, kThreads, 0, stream>>>(val[j & 1], val[(j + 1) & 1], nbr + 2 * j * cap, counts, channels,
                                                   cap, n);
    crf_slice_kernel<<<gp, kThreads, 0, stream>>>(val[kD1 & 1], wts, pv, nrm, dst, channels, pixels, cap);
    return cudaGetLastError();
  };
  OSVOS_CHECK_CUDA(filter(nullptr, 1, nullptr, norm));              // F(1)

  crf_taps_kernel<<<grid_for(radius + 1), kThreads, 0, stream>>>(taps, radius, inv2s2);
  crf_update_kernel<true, false><<<gp, kThreads, 0, stream>>>(zmaps, nullptr, taps, a, nullptr, q, nullptr, k, h, w,
                                                               pixels, radius, w_a, w_g);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  for (int it = 0; it < iterations; ++it) {
    OSVOS_CHECK_CUDA(filter(q, ch, norm, bmsg));
    crf_gauss_rows_kernel<<<gp, kThreads, 0, stream>>>(q, taps, t, ch, w, pixels, radius);
    if (it + 1 < iterations)
      crf_update_kernel<false, false><<<gp, kThreads, 0, stream>>>(zmaps, bmsg, taps, a, t, q, nullptr, k, h, w, pixels,
                                                                   radius, w_a, w_g);
    else
      crf_update_kernel<false, true><<<gp, kThreads, 0, stream>>>(zmaps, bmsg, taps, a, t, q, out, k, h, w, pixels,
                                                                  radius, w_a, w_g);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  return OSVOS_OK;
}

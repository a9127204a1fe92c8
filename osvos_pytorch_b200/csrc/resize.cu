// Resize of decoded uint8 frames and masks (the reference's DAVIS2016(inputRes=...), dataloaders/davis_2016.py:96-99,
// which calls scipy.misc.imresize: for uint8 input that is PIL.Image.fromarray(arr).resize((w, h), resample)).  The
// kernels restate Pillow's 8-bit resampler (libImaging/Resample.c, Geometry.c ImagingScaleAffine) bit for bit
// (DESIGN.md §17):
//   BILINEAR: separable, horizontal pass first into a uint8 intermediate that holds only the source rows the vertical
//             pass reads, then the vertical pass; an axis that keeps its size has no pass.  Per axis and output o a
//             table holds {xmin, count, k[0..ksize)}: triangle-filter weights widened by the downscale factor (Pillow's
//             antialias), normalised by their sum and rounded to 22-bit fixed point.  Pixels are integer sums
//             2^21 + sum(src * k), clipped to 8 bits, so only the tables need care: they are computed here in double
//             with explicitly rounded operations (__dmul_rn / __dadd_rn / __ddiv_rn), which nvcc cannot contract into
//             FMAs, in Pillow's operation order.
//   NEAREST:  index tables from Pillow's sequential accumulation xo = scale / 2, xo += scale (one thread per axis: the
//             running double sum is what Pillow rounds, a closed form is not the same), then one gather.
// Identical sizes are a copy.  Bandwidth-bound: one thread per output byte, so both passes read and write rows with
// consecutive bytes across a warp whatever the source alignment.
// The fp32 resize (osvos_resize_f32, DESIGN.md §18) upsamples fused logit maps to the annotations' stored size: Pillow's
// BILINEAR resize of an 'F' image (scipy 1.0's imresize(mode='F')), the same tables kept in double and accumulated in
// double, with an fp32 intermediate between the passes.
#include "common.cuh"

namespace osvos {

constexpr int kResizeThreads = 256;
constexpr int kPrecisionBits = 22;                 // Pillow's PRECISION_BITS = 32 - 8 - 2

struct ResizeAxis {
  int* tab;       // bilinear: [out][2 + ksize] = {xmin, count, k...}; nearest: [out] source index
  int in, out;    // out == 0: no table for this axis
  int ksize;
};

inline int resize_ksize(int in, int out) {
  const double scale = static_cast<double>(in) / out;
  return static_cast<int>(ceil(scale < 1.0 ? 1.0 : scale)) * 2 + 1;
}

__device__ __forceinline__ double triangle(double x) {
  if (x < 0.0) x = -x;
  return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// precompute_coeffs of Resample.c for output o of one axis of `in` -> `out` samples: emit(x, k) receives each weight k,
// normalised by the weights' sum, for x in [0, count); returns {xmin, count}.  Both emitters below share it, so the 8-bit
// and the fp32 resize use one table arithmetic.
template <class Emit>
__device__ __forceinline__ int2 bilinear_coeffs(int in, int out, int ksize, int o, Emit emit) {
  const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
  const double fs = scale < 1.0 ? 1.0 : scale;                 // support = 1.0 * fs
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn(static_cast<double>(o), 0.5), scale);
  int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, fs), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, fs), 0.5));
  if (xmax > in) xmax = in;
  const int cnt = min(max(xmax - xmin, 0), ksize);
  double ww = 0.0;
  for (int x = 0; x < cnt; ++x)
    ww = __dadd_rn(ww, triangle(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss)));
  for (int x = 0; x < cnt; ++x) {
    double k = triangle(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
    if (ww != 0.0) k = __ddiv_rn(k, ww);
    emit(x, k);
  }
  return make_int2(xmin, cnt);
}

// The 8-bit emitter (normalize_coeffs_8bpc): each weight rounded to 22-bit fixed point, in the row after {xmin, count}.
__device__ void bilinear_row(const ResizeAxis& a, int o) {
  int* row = a.tab + static_cast<size_t>(o) * (a.ksize + 2);
  const int2 b = bilinear_coeffs(a.in, a.out, a.ksize, o, [row](int x, double k) {
    const double scaled = __dmul_rn(k, static_cast<double>(1 << kPrecisionBits));   // exact: a power of two
    row[2 + x] = static_cast<int>(k < 0.0 ? __dsub_rn(scaled, 0.5) : __dadd_rn(scaled, 0.5));
  });
  row[0] = b.x;
  row[1] = b.y;
}

// Bilinear: one thread per output of either axis (x first, then y).
__global__ void __launch_bounds__(128) resize_bilinear_tables_kernel(ResizeAxis ax, ResizeAxis ay) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < ax.out) {
    bilinear_row(ax, t);
  } else if (t - ax.out < ay.out) {
    bilinear_row(ay, t - ax.out);
  }
}

// Nearest: thread 0 walks the x axis, thread 1 the y axis (ImagingScaleAffine's running sums).
__global__ void resize_nearest_tables_kernel(ResizeAxis ax, ResizeAxis ay) {
  if (threadIdx.x > 1) return;
  const ResizeAxis a = threadIdx.x == 0 ? ax : ay;
  const double scale = __ddiv_rn(static_cast<double>(a.in), static_cast<double>(a.out));
  double xo = __dmul_rn(scale, 0.5);
  for (int o = 0; o < a.out; ++o) {
    const int idx = xo < 0.0 ? 0 : static_cast<int>(xo);
    a.tab[o] = min(idx, a.in - 1);               // never reached for a resize; keeps the gather inside the frame
    xo = __dadd_rn(xo, scale);
  }
}

__device__ __forceinline__ uint8_t clip8(int acc) {
  if (acc <= 0) return 0;
  if (acc >= (1 << kPrecisionBits << 8)) return 255;
  return static_cast<uint8_t>(acc >> kPrecisionBits);
}

// Horizontal pass: src [n][h][w][C] -> dst [n][h][out_w][C] (frame stride h rows).  With `vtab` only the rows
// [vtab first xmin, last xmin + count) are resampled, written from dst row 0 (Pillow's ybox_first / ybox_last);
// without it every row is.
template <int C>
__global__ void __launch_bounds__(kResizeThreads)
resize_horizontal_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const int* __restrict__ htab,
                         const int* __restrict__ vtab, int h, int w, int out_w, int hstride, int out_h, int vstride) {
  const int f = blockIdx.z;
  int first = 0, rows = h;
  if (vtab != nullptr) {
    const int* last = vtab + static_cast<size_t>(out_h - 1) * vstride;
    first = __ldg(vtab);
    rows = __ldg(last) + __ldg(last + 1) - first;
  }
  const int r = blockIdx.y;
  const int row_bytes = out_w * C;
  const int b = blockIdx.x * kResizeThreads + threadIdx.x;
  if (r >= rows || b >= row_bytes) return;
  const int xo = b / C;
  const int ch = b - xo * C;
  const int* k = htab + static_cast<size_t>(xo) * hstride;
  const int xmin = __ldg(k), cnt = __ldg(k + 1);
  const uint8_t* s = src + (static_cast<size_t>(f) * h + first + r) * w * C + xmin * C + ch;
  int acc = 1 << (kPrecisionBits - 1);
  for (int t = 0; t < cnt; ++t) acc += static_cast<int>(__ldg(s + t * C)) * __ldg(k + 2 + t);
  dst[(static_cast<size_t>(f) * h + r) * row_bytes + b] = clip8(acc);
}

// Vertical pass: src [n][src_rows][row_bytes] -> dst [n][out_h][row_bytes]; output row yo reads source rows from
// vtab's xmin, less vtab's first xmin when `shift` (the horizontal pass dropped the rows above it).
__global__ void __launch_bounds__(kResizeThreads)
resize_vertical_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const int* __restrict__ vtab,
                       int vstride, int src_rows, int row_bytes, int out_h, int shift) {
  const int f = blockIdx.z;
  const int yo = blockIdx.y;
  const int b = blockIdx.x * kResizeThreads + threadIdx.x;
  if (b >= row_bytes) return;
  const int* k = vtab + static_cast<size_t>(yo) * vstride;
  const int ymin = __ldg(k) - (shift ? __ldg(vtab) : 0);
  const int cnt = __ldg(k + 1);
  const uint8_t* s = src + (static_cast<size_t>(f) * src_rows + ymin) * row_bytes + b;
  int acc = 1 << (kPrecisionBits - 1);
  for (int t = 0; t < cnt; ++t) acc += static_cast<int>(__ldg(s + static_cast<size_t>(t) * row_bytes)) * __ldg(k + 2 + t);
  dst[(static_cast<size_t>(f) * out_h + yo) * row_bytes + b] = clip8(acc);
}

// Nearest: dst[f][yo][xo][ch] = src[f][ytab[yo]][xtab[xo]][ch].
template <int C>
__global__ void __launch_bounds__(kResizeThreads)
resize_nearest_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const int* __restrict__ xtab,
                      const int* __restrict__ ytab, int h, int w, int out_h, int out_w) {
  const int f = blockIdx.z;
  const int yo = blockIdx.y;
  const int row_bytes = out_w * C;
  const int b = blockIdx.x * kResizeThreads + threadIdx.x;
  if (b >= row_bytes) return;
  const int xo = b / C;
  const int ch = b - xo * C;
  const uint8_t* s = src + (static_cast<size_t>(f) * h + __ldg(ytab + yo)) * w * C;
  dst[(static_cast<size_t>(f) * out_h + yo) * row_bytes + b] = __ldg(s + __ldg(xtab + xo) * C + ch);
}

struct ResizePlan {
  size_t htab_off, vtab_off, tmp_off, bytes;
  bool need_h, need_v;
  int kh, kv;
};

inline size_t align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

ResizePlan resize_plan(int n, int h, int w, int c, int out_h, int out_w, int mode) {
  ResizePlan p{};
  p.need_h = w != out_w;
  p.need_v = h != out_h;
  if (!p.need_h && !p.need_v) return p;          // a copy
  if (mode == OSVOS_RESIZE_NEAREST) {            // one gather; both index tables
    p.vtab_off = align16(sizeof(int) * out_w);
    p.bytes = p.vtab_off + align16(sizeof(int) * out_h);
    return p;
  }
  p.kh = p.need_h ? resize_ksize(w, out_w) : 0;
  p.kv = p.need_v ? resize_ksize(h, out_h) : 0;
  p.vtab_off = p.need_h ? align16(sizeof(int) * static_cast<size_t>(out_w) * (p.kh + 2)) : 0;
  p.tmp_off = p.vtab_off + (p.need_v ? align16(sizeof(int) * static_cast<size_t>(out_h) * (p.kv + 2)) : 0);
  p.bytes = p.tmp_off + (p.need_h && p.need_v ? static_cast<size_t>(n) * h * out_w * c : 0);
  return p;
}

template <int C>
int launch_resize(const uint8_t* src, uint8_t* dst, uint8_t* ws, const ResizePlan& p, int n, int h, int w, int out_h,
                  int out_w, int mode, cudaStream_t stream) {
  int* htab = reinterpret_cast<int*>(ws + p.htab_off);
  int* vtab = reinterpret_cast<int*>(ws + p.vtab_off);
  if (mode == OSVOS_RESIZE_NEAREST) {
    resize_nearest_tables_kernel<<<1, 32, 0, stream>>>(ResizeAxis{htab, w, out_w, 0}, ResizeAxis{vtab, h, out_h, 0});
    OSVOS_CHECK_CUDA(cudaGetLastError());
    const dim3 grid((out_w * C + kResizeThreads - 1) / kResizeThreads, out_h, n);
    resize_nearest_kernel<C><<<grid, kResizeThreads, 0, stream>>>(src, dst, htab, vtab, h, w, out_h, out_w);
    OSVOS_CHECK_CUDA(cudaGetLastError());
    return OSVOS_OK;
  }
  const ResizeAxis ax{htab, w, p.need_h ? out_w : 0, p.kh};
  const ResizeAxis ay{vtab, h, p.need_v ? out_h : 0, p.kv};
  resize_bilinear_tables_kernel<<<(ax.out + ay.out + 127) / 128, 128, 0, stream>>>(ax, ay);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  uint8_t* tmp = ws + p.tmp_off;
  if (p.need_h) {
    const dim3 grid((out_w * C + kResizeThreads - 1) / kResizeThreads, h, n);
    resize_horizontal_kernel<C><<<grid, kResizeThreads, 0, stream>>>(src, p.need_v ? tmp : dst, htab,
                                                                      p.need_v ? vtab : nullptr, h, w, out_w, p.kh + 2,
                                                                      out_h, p.kv + 2);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  if (p.need_v) {
    const dim3 grid((out_w * C + kResizeThreads - 1) / kResizeThreads, out_h, n);
    resize_vertical_kernel<<<grid, kResizeThreads, 0, stream>>>(p.need_h ? tmp : src, dst, vtab, p.kv + 2, h, out_w * C,
                                                                out_h, p.need_h ? 1 : 0);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  return OSVOS_OK;
}

// ---- fp32 bilinear (Pillow's 'F' image: ImagingResampleHorizontal_32bpc / Vertical_32bpc; DESIGN.md §18) ----------
// The same tables as above without the 8-bit rounding: bounds {xmin, count} per output and the normalised double
// weights.  Each pass accumulates ss = 0.0; ss += (double)src * k in double, one rounding per operation, and stores
// (float)ss, so the horizontal pass's intermediate is fp32 as Pillow's is.

struct ResizeAxisF64 {
  int* bounds;    // [out][2] = {xmin, count}
  double* k;      // [out][ksize]
  int in, out;    // out == 0: no table for this axis
  int ksize;
};

__device__ void bilinear_row_f64(const ResizeAxisF64& a, int o) {
  double* row = a.k + static_cast<size_t>(o) * a.ksize;
  const int2 b = bilinear_coeffs(a.in, a.out, a.ksize, o, [row](int x, double k) { row[x] = k; });
  a.bounds[2 * o] = b.x;
  a.bounds[2 * o + 1] = b.y;
}

__global__ void __launch_bounds__(128) resize_f32_tables_kernel(ResizeAxisF64 ax, ResizeAxisF64 ay) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < ax.out) {
    bilinear_row_f64(ax, t);
  } else if (t - ax.out < ay.out) {
    bilinear_row_f64(ay, t - ax.out);
  }
}

// Horizontal pass: src [n][h][w] -> dst [n][h][out_w] (frame stride h rows); with `vbounds` only the rows the vertical
// pass reads, written from dst row 0, as resize_horizontal_kernel.
__global__ void __launch_bounds__(kResizeThreads)
resize_f32_horizontal_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ hbounds,
                             const double* __restrict__ hk, const int* __restrict__ vbounds, int h, int w, int out_w,
                             int ksize, int out_h) {
  const int f = blockIdx.z;
  int first = 0, rows = h;
  if (vbounds != nullptr) {
    first = __ldg(vbounds);
    rows = __ldg(vbounds + 2 * (out_h - 1)) + __ldg(vbounds + 2 * (out_h - 1) + 1) - first;
  }
  const int r = blockIdx.y;
  const int xo = blockIdx.x * kResizeThreads + threadIdx.x;
  if (r >= rows || xo >= out_w) return;
  const int xmin = __ldg(hbounds + 2 * xo), cnt = __ldg(hbounds + 2 * xo + 1);
  const double* k = hk + static_cast<size_t>(xo) * ksize;
  const float* s = src + (static_cast<size_t>(f) * h + first + r) * w + xmin;
  double ss = 0.0;
  for (int t = 0; t < cnt; ++t) ss = __dadd_rn(ss, __dmul_rn(static_cast<double>(__ldg(s + t)), __ldg(k + t)));
  dst[(static_cast<size_t>(f) * h + r) * out_w + xo] = __double2float_rn(ss);
}

// Vertical pass: src [n][src_rows][w] -> dst [n][out_h][w]; source rows from vbounds' xmin, less the first xmin when
// `shift`.
__global__ void __launch_bounds__(kResizeThreads)
resize_f32_vertical_kernel(const float* __restrict__ src, float* __restrict__ dst, const int* __restrict__ vbounds,
                           const double* __restrict__ vk, int ksize, int src_rows, int w, int out_h, int shift) {
  const int f = blockIdx.z;
  const int yo = blockIdx.y;
  const int x = blockIdx.x * kResizeThreads + threadIdx.x;
  if (x >= w) return;
  const int ymin = __ldg(vbounds + 2 * yo) - (shift ? __ldg(vbounds) : 0);
  const int cnt = __ldg(vbounds + 2 * yo + 1);
  const double* k = vk + static_cast<size_t>(yo) * ksize;
  const float* s = src + (static_cast<size_t>(f) * src_rows + ymin) * w + x;
  double ss = 0.0;
  for (int t = 0; t < cnt; ++t)
    ss = __dadd_rn(ss, __dmul_rn(static_cast<double>(__ldg(s + static_cast<size_t>(t) * w)), __ldg(k + t)));
  dst[(static_cast<size_t>(f) * out_h + yo) * w + x] = __double2float_rn(ss);
}

// Workspace: hbounds, vbounds (int), hk, vk (double), then the fp32 intermediate [n][h][out_w] when both axes change;
// every part starts 16-byte aligned.
struct ResizeF32Plan {
  size_t vbounds_off, hk_off, vk_off, tmp_off, bytes;
  bool need_h, need_v;
  int kh, kv;
};

ResizeF32Plan resize_f32_plan(int n, int h, int w, int out_h, int out_w) {
  ResizeF32Plan p{};
  p.need_h = w != out_w;
  p.need_v = h != out_h;
  if (!p.need_h && !p.need_v) return p;          // a copy
  p.kh = p.need_h ? resize_ksize(w, out_w) : 0;
  p.kv = p.need_v ? resize_ksize(h, out_h) : 0;
  p.vbounds_off = p.need_h ? align16(sizeof(int) * 2 * static_cast<size_t>(out_w)) : 0;
  p.hk_off = p.vbounds_off + (p.need_v ? align16(sizeof(int) * 2 * static_cast<size_t>(out_h)) : 0);
  p.vk_off = p.hk_off + (p.need_h ? align16(sizeof(double) * static_cast<size_t>(out_w) * p.kh) : 0);
  p.tmp_off = p.vk_off + (p.need_v ? align16(sizeof(double) * static_cast<size_t>(out_h) * p.kv) : 0);
  p.bytes = p.tmp_off + (p.need_h && p.need_v ? sizeof(float) * static_cast<size_t>(n) * h * out_w : 0);
  return p;
}

int launch_resize_f32(const float* src, float* dst, uint8_t* ws, const ResizeF32Plan& p, int n, int h, int w,
                      int out_h, int out_w, cudaStream_t stream) {
  int* hbounds = reinterpret_cast<int*>(ws);
  int* vbounds = reinterpret_cast<int*>(ws + p.vbounds_off);
  double* hk = reinterpret_cast<double*>(ws + p.hk_off);
  double* vk = reinterpret_cast<double*>(ws + p.vk_off);
  const ResizeAxisF64 ax{hbounds, hk, w, p.need_h ? out_w : 0, p.kh};
  const ResizeAxisF64 ay{vbounds, vk, h, p.need_v ? out_h : 0, p.kv};
  resize_f32_tables_kernel<<<(ax.out + ay.out + 127) / 128, 128, 0, stream>>>(ax, ay);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  float* tmp = reinterpret_cast<float*>(ws + p.tmp_off);
  if (p.need_h) {
    const dim3 grid((out_w + kResizeThreads - 1) / kResizeThreads, h, n);
    resize_f32_horizontal_kernel<<<grid, kResizeThreads, 0, stream>>>(src, p.need_v ? tmp : dst, hbounds, hk,
                                                                       p.need_v ? vbounds : nullptr, h, w, out_w, p.kh,
                                                                       out_h);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  if (p.need_v) {
    const dim3 grid((out_w + kResizeThreads - 1) / kResizeThreads, out_h, n);
    resize_f32_vertical_kernel<<<grid, kResizeThreads, 0, stream>>>(p.need_h ? tmp : src, dst, vbounds, vk, p.kv, h,
                                                                     out_w, out_h, p.need_h ? 1 : 0);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  return OSVOS_OK;
}

}  // namespace osvos

using namespace osvos;

static bool resize_dims_ok(int n, int h, int w, int c, int out_h, int out_w, int mode) {
  return n > 0 && n < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768 && out_h > 0 && out_w > 0 && out_h < 32768 &&
         out_w < 32768 && (c == 1 || c == 3) && (mode == OSVOS_RESIZE_BILINEAR || mode == OSVOS_RESIZE_NEAREST);
}

extern "C" size_t osvos_resize_u8_workspace_bytes(int n, int h, int w, int c, int out_h, int out_w, int mode) {
  if (!resize_dims_ok(n, h, w, c, out_h, out_w, mode)) return 0;
  return resize_plan(n, h, w, c, out_h, out_w, mode).bytes;
}

extern "C" int osvos_resize_u8(const uint8_t* src, uint8_t* dst, void* workspace, int n, int h, int w, int c, int out_h,
                               int out_w, int mode, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && dst != nullptr);
  OSVOS_CHECK_ARG(resize_dims_ok(n, h, w, c, out_h, out_w, mode));
  const ResizePlan p = resize_plan(n, h, w, c, out_h, out_w, mode);
  OSVOS_CHECK_ARG(p.bytes == 0 || (workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 3) == 0));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p.need_h && !p.need_v) {
    OSVOS_CHECK_CUDA(cudaMemcpyAsync(dst, src, static_cast<size_t>(n) * h * w * c, cudaMemcpyDeviceToDevice, stream));
    return OSVOS_OK;
  }
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  return c == 1 ? launch_resize<1>(src, dst, ws, p, n, h, w, out_h, out_w, mode, stream)
                : launch_resize<3>(src, dst, ws, p, n, h, w, out_h, out_w, mode, stream);
}

extern "C" size_t osvos_resize_f32_workspace_bytes(int n, int h, int w, int out_h, int out_w) {
  if (!resize_dims_ok(n, h, w, 1, out_h, out_w, OSVOS_RESIZE_BILINEAR)) return 0;
  return resize_f32_plan(n, h, w, out_h, out_w).bytes;
}

extern "C" int osvos_resize_f32(const float* src, float* dst, void* workspace, int n, int h, int w, int out_h,
                                int out_w, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && dst != nullptr);
  OSVOS_CHECK_ARG(resize_dims_ok(n, h, w, 1, out_h, out_w, OSVOS_RESIZE_BILINEAR));
  const ResizeF32Plan p = resize_f32_plan(n, h, w, out_h, out_w);
  OSVOS_CHECK_ARG(p.bytes == 0 || (workspace != nullptr && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!p.need_h && !p.need_v) {
    OSVOS_CHECK_CUDA(cudaMemcpyAsync(dst, src, sizeof(float) * n * h * w, cudaMemcpyDeviceToDevice, stream));
    return OSVOS_OK;
  }
  return launch_resize_f32(src, dst, static_cast<uint8_t*>(workspace), p, n, h, w, out_h, out_w, stream);
}

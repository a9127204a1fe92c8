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

// precompute_coeffs + normalize_coeffs_8bpc of Resample.c for output o of one axis.
__device__ void bilinear_row(const ResizeAxis& a, int o) {
  const double scale = __ddiv_rn(static_cast<double>(a.in), static_cast<double>(a.out));
  const double fs = scale < 1.0 ? 1.0 : scale;                 // support = 1.0 * fs
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn(static_cast<double>(o), 0.5), scale);
  int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, fs), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, fs), 0.5));
  if (xmax > a.in) xmax = a.in;
  const int cnt = min(max(xmax - xmin, 0), a.ksize);
  int* row = a.tab + static_cast<size_t>(o) * (a.ksize + 2);
  double ww = 0.0;
  for (int x = 0; x < cnt; ++x)
    ww = __dadd_rn(ww, triangle(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss)));
  for (int x = 0; x < cnt; ++x) {
    double k = triangle(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
    if (ww != 0.0) k = __ddiv_rn(k, ww);
    const double scaled = __dmul_rn(k, static_cast<double>(1 << kPrecisionBits));   // exact: a power of two
    row[2 + x] = static_cast<int>(k < 0.0 ? __dsub_rn(scaled, 0.5) : __dadd_rn(scaled, 0.5));
  }
  row[0] = xmin;
  row[1] = cnt;
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

// Baseline JPEG encoder for BGR frames: the bytes cv2.imencode('.jpg', frame, [IMWRITE_JPEG_QUALITY, q]) writes
// (libjpeg-turbo: JFIF, 4:2:0, ISLOW FDCT, the Annex K Huffman tables, no restart interval; DESIGN.md §23).
// tests/jpeg_encode_ref.py restates it in numpy and names the libjpeg-turbo routine behind each rule.  Everything is
// integer, so a frame's bytes do not depend on its batch mates, the stream or the run.
// Seven launches:
//   jpeg_fdct_kernel     8 threads per block of the scan (MCU order Y0 Y1 Y2 Y3 Cb Cr): edge-replicated samples,
//                        colour conversion, 2x2 chroma downsampling, FDCT (rows, then columns through shared memory),
//                        quantisation; int16 coefficients in zig-zag order.  A dummy block takes the DCT of the block
//                        whose DC it copies and zeroes its AC;
//   jpeg_count_kernel    one thread per block: its exact coded bit count (its DC difference needs the previous block
//                        of the same component in the scan);
//   jpeg_scan_kernel     one CTA per frame: bit offsets, the zeroed word buffer, the 1-bit padding of the last byte;
//   jpeg_write_kernel    one thread per block: ORs its bits into the word buffer (whole words inside its range are
//                        stored, the two shared ones ORed atomically; ranges never overlap, so order does not matter);
//   jpeg_ff_count_kernel one CTA per 4 KB chunk of scan bytes: its 0xFF bytes;
//   jpeg_place_kernel    one CTA per frame: each chunk's output offset, the header, EOI and the file's length;
//   jpeg_stuff_kernel    one CTA per chunk: the bytes copied to their place with 00 after every FF.
// overlay_mask_kernel (end of file) draws the picture these files usually hold: the mask over the frame;
// overlay_labels_kernel draws a label map of K objects the same way, each in its own colour (DESIGN.md §25).
#include "common.cuh"

namespace osvos {

constexpr int kJpegHeaderBytes = 623;
constexpr int kJpegBlockBitsMax = 22 + 63 * 26;      // DC: 11-bit code + 11 bits; 63 AC of 16-bit code + 10 bits
constexpr int kJpegChunk = 4096;                     // scan bytes per stuffing CTA: 256 threads x 16
constexpr int kJpegScanThreads = 1024;

__constant__ uint8_t kZigzagOfNatural[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42,
                                             3,  8,  12, 17, 25, 30, 41, 43, 9,  11, 18, 24, 31, 40, 44, 53,
                                             10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60,
                                             21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};

static const uint8_t kStdLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                      14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                      18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                      49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t kStdChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                        24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                        99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                        99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
static const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// Annex K.3: counts of codes of length 1..16, then the symbols
static const uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
static const uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
static const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D};
static const uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7, 0xA8, 0xA9,
    0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA,
    0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA,
    0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA};
static const uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
static const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16,
    0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26, 0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7,
    0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5, 0xC6, 0xC7, 0xC8,
    0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9,
    0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8, 0xF9, 0xFA};

struct JpegQuant {
  uint16_t div[2][64];                               // 8 q, natural order: luma, chroma
};

struct JpegCodes {
  uint32_t dc[2][12];                                // (length << 16) | code: luma, chroma
  uint32_t ac[2][256];
};

struct JpegHeader {
  uint8_t b[kJpegHeaderBytes + 1];
};

struct JpegPlan {
  int mx, my;                                        // MCU columns, rows
  int units;                                         // blocks per frame (6 per MCU)
  int chunks;                                        // stuffing chunks per frame at capacity
  size_t words;                                      // 32-bit words of the bit buffer per frame
  size_t coef_off, bits_off, offs_off, word_off, ff_off, place_off, total_off, bytes;
};

inline size_t jpeg_align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

inline bool jpeg_dims_ok(int h, int w) { return h >= 1 && w >= 1 && h <= 65500 && w <= 65500; }

inline size_t jpeg_scan_bytes_max(int h, int w) {
  const size_t units = 6 * static_cast<size_t>((h + 15) / 16) * ((w + 15) / 16);
  return (units * kJpegBlockBitsMax + 7) / 8;
}

inline size_t jpeg_max_bytes(int h, int w) { return kJpegHeaderBytes + 2 + 2 * jpeg_scan_bytes_max(h, w); }

JpegPlan jpeg_plan(int n, int h, int w) {
  JpegPlan p{};
  p.mx = (w + 15) / 16;
  p.my = (h + 15) / 16;
  p.units = 6 * p.mx * p.my;
  const size_t sb = jpeg_scan_bytes_max(h, w);
  p.chunks = static_cast<int>((sb + kJpegChunk - 1) / kJpegChunk);
  p.words = (sb + 3) / 4 + 1;
  const size_t nu = static_cast<size_t>(n) * p.units;
  p.coef_off = 0;
  p.bits_off = jpeg_align16(p.coef_off + nu * 64 * sizeof(int16_t));
  p.offs_off = jpeg_align16(p.bits_off + nu * sizeof(uint32_t));
  p.word_off = jpeg_align16(p.offs_off + nu * sizeof(unsigned long long));
  p.ff_off = jpeg_align16(p.word_off + static_cast<size_t>(n) * p.words * sizeof(uint32_t));
  p.place_off = jpeg_align16(p.ff_off + static_cast<size_t>(n) * p.chunks * sizeof(uint32_t));
  p.total_off = jpeg_align16(p.place_off + static_cast<size_t>(n) * p.chunks * sizeof(unsigned long long));
  p.bytes = p.total_off + static_cast<size_t>(n) * sizeof(unsigned long long);
  return p;
}

// ---- coefficients ---------------------------------------------------------------------------------------------------

// jfdctint.c: one 1-D pass.  `final`: the column pass (descale by CONST_BITS + PASS1_BITS, DC terms by PASS1_BITS);
// otherwise the row pass (scale the DC terms up by PASS1_BITS, descale the rest by CONST_BITS - PASS1_BITS).
__device__ __forceinline__ void fdct_1d(const int* d, int* o, bool final) {
  const int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
  const int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  const int sh = final ? 15 : 11;
  const int rnd = 1 << (sh - 1);
  if (final) {
    o[0] = (t10 + t11 + 2) >> 2;
    o[4] = (t10 - t11 + 2) >> 2;
  } else {
    o[0] = (t10 + t11) * 4;
    o[4] = (t10 - t11) * 4;
  }
  const int z1 = (t12 + t13) * 4433;
  o[2] = (z1 + t13 * 6270 + rnd) >> sh;
  o[6] = (z1 - t12 * 15137 + rnd) >> sh;
  const int z5 = (t4 + t6 + t5 + t7) * 9633;
  const int a1 = (t4 + t7) * -7373, a2 = (t5 + t6) * -20995;
  const int a3 = (t4 + t6) * -16069 + z5, a4 = (t5 + t7) * -3196 + z5;
  o[7] = (t4 * 2446 + a1 + a3 + rnd) >> sh;
  o[5] = (t5 * 16819 + a2 + a4 + rnd) >> sh;
  o[3] = (t6 * 25172 + a2 + a3 + rnd) >> sh;
  o[1] = (t7 * 12299 + a1 + a4 + rnd) >> sh;
}

// jccolor.c rgb_ycc_convert, 16 fractional bits; comp 0 Y, 1 Cb, 2 Cr
__device__ __forceinline__ int ycc_of(const uint8_t* px, int comp) {
  const int b = px[0], g = px[1], r = px[2];
  if (comp == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (comp == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

constexpr int kFdctThreads = 256;                    // 32 blocks per CTA, 8 threads (one row, then one column) each

__global__ void __launch_bounds__(kFdctThreads) jpeg_fdct_kernel(const uint8_t* __restrict__ src, int16_t* __restrict__ coef,
                                                                 JpegQuant quant, int n, int h, int w, int mx, int units) {
  __shared__ int ws[kFdctThreads / 8][8][9];
  const long long g = static_cast<long long>(blockIdx.x) * kFdctThreads + threadIdx.x;
  const long long unit = g >> 3;
  const int r = static_cast<int>(g & 7);
  const bool valid = unit < static_cast<long long>(n) * units;
  int (*sw)[9] = ws[threadIdx.x >> 3];
  int f = 0, j = 0, comp = 0;
  if (valid) {
    f = static_cast<int>(unit / units);
    const int u = static_cast<int>(unit % units);
    const int m = u / 6;
    j = u % 6;
    const int mi = m / mx, mj = m % mx;
    const uint8_t* frame = src + static_cast<size_t>(f) * h * w * 3;
    int d[8], o[8];
    if (j < 4) {
      const int wib = (w + 7) / 8, hib = (h + 7) / 8;
      int by = 2 * mi + (j >> 1), bx = 2 * mj + (j & 1);
      if (by >= hib) {                                           // bottom dummy: the DC of block 1 of its MCU
        by = 2 * mi;
        bx = 2 * mj + 1;
      }
      if (bx >= wib) bx -= 1;                                    // right dummy: the DC of the block to its left
      const int y = min(by * 8 + r, h - 1);
      for (int k = 0; k < 8; ++k) {
        const int x = min(bx * 8 + k, w - 1);
        d[k] = ycc_of(frame + (static_cast<size_t>(y) * w + x) * 3, 0) - 128;
      }
    } else {
      comp = j - 3;
      const int dr = min(mi * 8 + r, (h + 1) / 2 - 1);          // downsampled rows past the image repeat the last
      const int y0 = 2 * dr, y1 = min(2 * dr + 1, h - 1);
      for (int k = 0; k < 8; ++k) {
        const int oc = mj * 8 + k;
        const int x0 = min(2 * oc, w - 1), x1 = min(2 * oc + 1, w - 1);
        const int s = ycc_of(frame + (static_cast<size_t>(y0) * w + x0) * 3, comp) +
                      ycc_of(frame + (static_cast<size_t>(y0) * w + x1) * 3, comp) +
                      ycc_of(frame + (static_cast<size_t>(y1) * w + x0) * 3, comp) +
                      ycc_of(frame + (static_cast<size_t>(y1) * w + x1) * 3, comp);
        d[k] = ((s + 1 + (k & 1)) >> 2) - 128;                   // h2v2_downsample's bias 1, 2, 1, 2, ...
      }
    }
    fdct_1d(d, o, false);
    for (int k = 0; k < 8; ++k) sw[r][k] = o[k];
  }
  __syncwarp();
  if (!valid) return;
  int d[8], o[8];
  for (int k = 0; k < 8; ++k) d[k] = sw[k][r];
  fdct_1d(d, o, true);
  const int wib = (w + 7) / 8, hib = (h + 7) / 8;
  const int m = static_cast<int>(unit % units) / 6;
  const bool dummy = j < 4 && (2 * (m % mx) + (j & 1) >= wib || 2 * (m / mx) + (j >> 1) >= hib);
  int16_t* out = coef + static_cast<size_t>(unit) * 64;
  const uint16_t* div = quant.div[comp > 0 ? 1 : 0];
  for (int v = 0; v < 8; ++v) {
    const int nat = v * 8 + r;
    const int q = div[nat];
    const int a = abs(o[v]);
    int c = (a + (q >> 1)) / q;                                  // jcdctmgr.c: round half away from zero
    c = o[v] < 0 ? -c : c;
    if (dummy && nat != 0) c = 0;
    out[kZigzagOfNatural[nat]] = static_cast<int16_t>(c);
  }
}

// ---- entropy coding -------------------------------------------------------------------------------------------------

__device__ __forceinline__ int nbits_of(int v) { return v == 0 ? 0 : 32 - __clz(abs(v)); }

__device__ __forceinline__ int prev_dc(const int16_t* coef, long long unit, int units) {
  const int u = static_cast<int>(unit % units), j = u % 6;
  long long p;
  if (j >= 4) p = u >= 6 ? unit - 6 : -1;                        // Cb, Cr: the previous MCU's
  else if (j > 0) p = unit - 1;
  else p = u >= 6 ? unit - 3 : -1;                               // Y0: the previous MCU's Y3
  return p < 0 ? 0 : coef[static_cast<size_t>(p) * 64];
}

// Walks one block's symbols (jchuff.c encode_one_block) and hands each (code, length) to emit.
template <class Emit>
__device__ __forceinline__ void code_block(const int16_t* blk, int dc_prev, const uint32_t* dc, const uint32_t* ac,
                                           Emit&& emit) {
  const int diff = blk[0] - dc_prev;
  int s = nbits_of(diff);
  emit(static_cast<uint32_t>(((dc[s] & 0xFFFF) << s) | ((diff < 0 ? diff - 1 : diff) & ((1 << s) - 1))),
       static_cast<int>(dc[s] >> 16) + s);
  int run = 0;
  const int4* b4 = reinterpret_cast<const int4*>(blk);
#pragma unroll 1
  for (int q = 0; q < 8; ++q) {
    const int4 v4 = b4[q];
    const int16_t* v = reinterpret_cast<const int16_t*>(&v4);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (q == 0 && i == 0) continue;
      const int c = v[i];
      if (c == 0) {
        ++run;
        continue;
      }
      while (run > 15) {
        emit(ac[0xF0] & 0xFFFF, static_cast<int>(ac[0xF0] >> 16));
        run -= 16;
      }
      s = nbits_of(c);
      const uint32_t e = ac[(run << 4) | s];
      emit(((e & 0xFFFF) << s) | ((c < 0 ? c - 1 : c) & ((1 << s) - 1)), static_cast<int>(e >> 16) + s);
      run = 0;
    }
  }
  if (run > 0) emit(ac[0] & 0xFFFF, static_cast<int>(ac[0] >> 16));
}

__device__ __forceinline__ void load_codes(const JpegCodes& codes, JpegCodes& sm) {
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&codes);
  uint32_t* d = reinterpret_cast<uint32_t*>(&sm);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(JpegCodes) / 4); i += blockDim.x) d[i] = s[i];
  __syncthreads();
}

__global__ void __launch_bounds__(256) jpeg_count_kernel(const int16_t* __restrict__ coef, uint32_t* __restrict__ bits,
                                                         JpegCodes codes, long long total_units, int units) {
  __shared__ JpegCodes sm;
  load_codes(codes, sm);
  const long long unit = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (unit >= total_units) return;
  const int t = static_cast<int>(unit % units) % 6 >= 4 ? 1 : 0;
  uint32_t nb = 0;
  code_block(coef + static_cast<size_t>(unit) * 64, prev_dc(coef, unit, units), sm.dc[t], sm.ac[t],
             [&](uint32_t, int len) { nb += len; });
  bits[unit] = nb;
}

// One CTA per frame: exclusive scan of the block bit counts, the frame's total, the zeroed words it will use and the
// 1 bits that pad its last byte.
__global__ void __launch_bounds__(kJpegScanThreads) jpeg_scan_kernel(const uint32_t* __restrict__ bits,
                                                                     unsigned long long* __restrict__ offs,
                                                                     uint32_t* __restrict__ words,
                                                                     unsigned long long* __restrict__ totals, int units,
                                                                     size_t words_per_frame) {
  __shared__ unsigned long long warp_sums[32];
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5, f = blockIdx.x;
  const uint32_t* b = bits + static_cast<size_t>(f) * units;
  unsigned long long* o = offs + static_cast<size_t>(f) * units;
  const int per = (units + kJpegScanThreads - 1) / kJpegScanThreads;
  const int lo = min(units, t * per), hi = min(units, lo + per);
  unsigned long long mine = 0;
  for (int i = lo; i < hi; ++i) mine += b[i];
  unsigned long long x = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    unsigned long long s = warp_sums[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  unsigned long long run = x - mine + (wid > 0 ? warp_sums[wid - 1] : 0);
  for (int i = lo; i < hi; ++i) {
    o[i] = run;
    run += b[i];
  }
  const unsigned long long total = warp_sums[31];
  uint32_t* wf = words + static_cast<size_t>(f) * words_per_frame;
  const unsigned long long nw = (total + 31) / 32;
  for (unsigned long long i = t; i < nw; i += kJpegScanThreads) wf[i] = 0;
  __syncthreads();
  if (t == 0) {
    totals[f] = total;
    const int pad = static_cast<int>((8 - (total & 7)) & 7);
    if (pad) {                                                   // jchuff.c flush_bits: the byte is filled with 1s
      const int o32 = static_cast<int>(total & 31);
      wf[total >> 5] |= ((1u << pad) - 1) << (32 - o32 - pad);
    }
  }
}

// Bit buffer: word i holds scan bytes 4i .. 4i+3, the first in its top byte.
__global__ void __launch_bounds__(256) jpeg_write_kernel(const int16_t* __restrict__ coef,
                                                         const unsigned long long* __restrict__ offs,
                                                         uint32_t* __restrict__ words, JpegCodes codes,
                                                         long long total_units, int units, size_t words_per_frame) {
  __shared__ JpegCodes sm;
  load_codes(codes, sm);
  const long long unit = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (unit >= total_units) return;
  const int f = static_cast<int>(unit / units);
  const int t = static_cast<int>(unit % units) % 6 >= 4 ? 1 : 0;
  uint32_t* wf = words + static_cast<size_t>(f) * words_per_frame;
  const unsigned long long p0 = offs[unit];
  size_t wi = p0 >> 5;
  int nb = static_cast<int>(p0 & 31);                            // bits held in acc, counted from the word's start
  unsigned long long acc = 0;
  bool first = true;
  code_block(coef + static_cast<size_t>(unit) * 64, prev_dc(coef, unit, units), sm.dc[t], sm.ac[t],
             [&](uint32_t v, int len) {
               acc = (acc << len) | v;
               nb += len;
               if (nb >= 32) {
                 const uint32_t word = static_cast<uint32_t>(acc >> (nb - 32));
                 if (first) atomicOr(wf + wi, word);             // shared with the previous block
                 else wf[wi] = word;
                 first = false;
                 ++wi;
                 nb -= 32;
                 acc &= (1ull << nb) - 1;
               }
             });
  if (nb > 0) atomicOr(wf + wi, static_cast<uint32_t>(acc << (32 - nb)));   // shared with the next block
}

__device__ __forceinline__ uint8_t scan_byte(const uint32_t* wf, unsigned long long k) {
  return static_cast<uint8_t>(wf[k >> 2] >> (24 - 8 * (k & 3)));
}

__device__ __forceinline__ int block_sum_256(int v, int* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[wid] = v;
  __syncthreads();
  int s = 0;
  for (int k = 0; k < 8; ++k) s += red[k];
  return s;
}

__global__ void __launch_bounds__(256) jpeg_ff_count_kernel(const uint32_t* __restrict__ words,
                                                            const unsigned long long* __restrict__ totals,
                                                            uint32_t* __restrict__ ff, int chunks,
                                                            size_t words_per_frame) {
  __shared__ int red[8];
  const int f = blockIdx.y, c = blockIdx.x;
  const unsigned long long nbytes = (totals[f] + 7) / 8;
  const unsigned long long base = static_cast<unsigned long long>(c) * kJpegChunk;
  if (base >= nbytes) return;
  const uint32_t* wf = words + static_cast<size_t>(f) * words_per_frame;
  int cnt = 0;
  for (int i = 0; i < 16; ++i) {
    const unsigned long long k = base + threadIdx.x * 16 + i;
    cnt += k < nbytes && scan_byte(wf, k) == 0xFF;
  }
  cnt = block_sum_256(cnt, red);
  if (threadIdx.x == 0) ff[static_cast<size_t>(f) * chunks + c] = cnt;
}

__global__ void __launch_bounds__(kJpegScanThreads) jpeg_place_kernel(const uint32_t* __restrict__ ff,
                                                                      const unsigned long long* __restrict__ totals,
                                                                      unsigned long long* __restrict__ place,
                                                                      uint8_t* __restrict__ out,
                                                                      long long* __restrict__ lengths, JpegHeader hdr,
                                                                      int chunks, size_t max_bytes) {
  __shared__ unsigned long long warp_sums[32];
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5, f = blockIdx.x;
  const unsigned long long nbytes = (totals[f] + 7) / 8;
  const int used = static_cast<int>((nbytes + kJpegChunk - 1) / kJpegChunk);
  const uint32_t* fc = ff + static_cast<size_t>(f) * chunks;
  unsigned long long* pl = place + static_cast<size_t>(f) * chunks;
  const int per = (used + kJpegScanThreads - 1) / kJpegScanThreads;
  const int lo = min(used, t * per), hi = min(used, lo + per);
  unsigned long long mine = 0;
  for (int i = lo; i < hi; ++i) mine += fc[i];
  unsigned long long x = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    unsigned long long s = warp_sums[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  unsigned long long run = x - mine + (wid > 0 ? warp_sums[wid - 1] : 0);
  for (int i = lo; i < hi; ++i) {
    pl[i] = static_cast<unsigned long long>(i) * kJpegChunk + run;
    run += fc[i];
  }
  uint8_t* file = out + static_cast<size_t>(f) * max_bytes;
  for (int i = t; i < kJpegHeaderBytes; i += kJpegScanThreads) file[i] = hdr.b[i];
  if (t == 0) {
    const unsigned long long end = kJpegHeaderBytes + nbytes + warp_sums[31];
    file[end] = 0xFF;
    file[end + 1] = 0xD9;
    lengths[f] = static_cast<long long>(end + 2);
  }
}

__global__ void __launch_bounds__(256) jpeg_stuff_kernel(const uint32_t* __restrict__ words,
                                                         const unsigned long long* __restrict__ totals,
                                                         const unsigned long long* __restrict__ place,
                                                         uint8_t* __restrict__ out, int chunks, size_t words_per_frame,
                                                         size_t max_bytes) {
  __shared__ int warp_sums[8];
  const int f = blockIdx.y, c = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const unsigned long long nbytes = (totals[f] + 7) / 8;
  const unsigned long long base = static_cast<unsigned long long>(c) * kJpegChunk;
  if (base >= nbytes) return;
  const uint32_t* wf = words + static_cast<size_t>(f) * words_per_frame;
  uint8_t v[16];
  int cnt = 0;
  const unsigned long long k0 = base + t * 16;
  for (int i = 0; i < 16; ++i) {
    v[i] = k0 + i < nbytes ? scan_byte(wf, k0 + i) : 0;
    cnt += k0 + i < nbytes && v[i] == 0xFF;
  }
  int x = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  int before = x - cnt;
  for (int k = 0; k < wid; ++k) before += warp_sums[k];
  uint8_t* dst = out + static_cast<size_t>(f) * max_bytes + kJpegHeaderBytes + place[static_cast<size_t>(f) * chunks + c] +
                 (k0 - base) + before;
  for (int i = 0; i < 16 && k0 + i < nbytes; ++i) {
    *dst++ = v[i];
    if (v[i] == 0xFF) *dst++ = 0;
  }
}

// ---- host tables ----------------------------------------------------------------------------------------------------

int jpeg_quality_table(const uint8_t* base, int quality, int i) {           // jcparam.c with force_baseline
  const int q = quality < 1 ? 1 : (quality > 100 ? 100 : quality);
  const int scale = q < 50 ? 5000 / q : 200 - 2 * q;
  const int v = (base[i] * scale + 50) / 100;
  return v < 1 ? 1 : (v > 255 ? 255 : v);
}

void jpeg_huff(const uint8_t* counts, const uint8_t* syms, uint32_t* table) {
  int code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < counts[len - 1]; ++i, ++k, ++code) table[syms[k]] = (static_cast<uint32_t>(len) << 16) | code;
    code <<= 1;
  }
}

const JpegCodes& jpeg_codes() {
  static JpegCodes c = [] {
    JpegCodes t{};
    jpeg_huff(kDcLumaBits, kDcVals, t.dc[0]);
    jpeg_huff(kDcChromaBits, kDcVals, t.dc[1]);
    jpeg_huff(kAcLumaBits, kAcLumaVals, t.ac[0]);
    jpeg_huff(kAcChromaBits, kAcChromaVals, t.ac[1]);
    return t;
  }();
  return c;
}

JpegHeader jpeg_header(int h, int w, int quality) {
  JpegHeader hd{};
  uint8_t* p = hd.b;
  const uint8_t soi_app0[20] = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  memcpy(p, soi_app0, 20);
  p += 20;
  for (int t = 0; t < 2; ++t) {
    const uint8_t dqt[5] = {0xFF, 0xDB, 0, 67, static_cast<uint8_t>(t)};
    memcpy(p, dqt, 5);
    p += 5;
    for (int i = 0; i < 64; ++i) *p++ = static_cast<uint8_t>(jpeg_quality_table(t ? kStdChromaQ : kStdLumaQ, quality, kZigzag[i]));
  }
  const uint8_t sof[19] = {0xFF, 0xC0, 0, 17, 8, static_cast<uint8_t>(h >> 8), static_cast<uint8_t>(h),
                           static_cast<uint8_t>(w >> 8), static_cast<uint8_t>(w), 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1};
  memcpy(p, sof, 19);
  p += 19;
  const uint8_t* bits[4] = {kDcLumaBits, kAcLumaBits, kDcChromaBits, kAcChromaBits};
  const uint8_t* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
  const uint8_t ids[4] = {0x00, 0x10, 0x01, 0x11};
  for (int k = 0; k < 4; ++k) {
    int nsym = 0;
    for (int i = 0; i < 16; ++i) nsym += bits[k][i];
    const int len = 19 + nsym;
    const uint8_t dht[5] = {0xFF, 0xC4, static_cast<uint8_t>(len >> 8), static_cast<uint8_t>(len), ids[k]};
    memcpy(p, dht, 5);
    memcpy(p + 5, bits[k], 16);
    memcpy(p + 21, vals[k], nsym);
    p += 21 + nsym;
  }
  const uint8_t sos[14] = {0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
  memcpy(p, sos, 14);
  return hd;
}

}  // namespace osvos

using namespace osvos;

extern "C" size_t osvos_jpeg_max_bytes(int h, int w) { return jpeg_dims_ok(h, w) ? jpeg_max_bytes(h, w) : 0; }

extern "C" size_t osvos_jpeg_encode_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || n >= 65536 || !jpeg_dims_ok(h, w)) return 0;
  return jpeg_plan(n, h, w).bytes;
}

extern "C" int osvos_jpeg_encode(const uint8_t* src, uint8_t* out, int64_t* lengths, void* workspace, int n, int h, int w,
                                 int quality, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && out != nullptr && lengths != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(n > 0 && n < 65536 && jpeg_dims_ok(h, w) && quality >= 1 && quality <= 100);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(lengths) & 7) == 0);
  const JpegPlan p = jpeg_plan(n, h, w);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  int16_t* coef = reinterpret_cast<int16_t*>(ws + p.coef_off);
  uint32_t* bits = reinterpret_cast<uint32_t*>(ws + p.bits_off);
  unsigned long long* offs = reinterpret_cast<unsigned long long*>(ws + p.offs_off);
  uint32_t* words = reinterpret_cast<uint32_t*>(ws + p.word_off);
  uint32_t* ff = reinterpret_cast<uint32_t*>(ws + p.ff_off);
  unsigned long long* place = reinterpret_cast<unsigned long long*>(ws + p.place_off);
  unsigned long long* totals = reinterpret_cast<unsigned long long*>(ws + p.total_off);
  JpegQuant quant{};
  for (int i = 0; i < 64; ++i) {
    quant.div[0][i] = static_cast<uint16_t>(8 * jpeg_quality_table(kStdLumaQ, quality, i));
    quant.div[1][i] = static_cast<uint16_t>(8 * jpeg_quality_table(kStdChromaQ, quality, i));
  }
  const long long total_units = static_cast<long long>(n) * p.units;
  const size_t max_bytes = jpeg_max_bytes(h, w);
  jpeg_fdct_kernel<<<static_cast<unsigned>((total_units * 8 + kFdctThreads - 1) / kFdctThreads), kFdctThreads, 0,
                     stream>>>(src, coef, quant, n, h, w, p.mx, p.units);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  const unsigned ublocks = static_cast<unsigned>((total_units + 255) / 256);
  jpeg_count_kernel<<<ublocks, 256, 0, stream>>>(coef, bits, jpeg_codes(), total_units, p.units);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_scan_kernel<<<n, kJpegScanThreads, 0, stream>>>(bits, offs, words, totals, p.units, p.words);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_write_kernel<<<ublocks, 256, 0, stream>>>(coef, offs, words, jpeg_codes(), total_units, p.units, p.words);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_ff_count_kernel<<<dim3(p.chunks, n), 256, 0, stream>>>(words, totals, ff, p.chunks, p.words);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_place_kernel<<<n, kJpegScanThreads, 0, stream>>>(ff, totals, place, out, reinterpret_cast<long long*>(lengths),
                                                        jpeg_header(h, w, quality), p.chunks, max_bytes);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_stuff_kernel<<<dim3(p.chunks, n), 256, 0, stream>>>(words, totals, place, out, p.chunks, p.words, max_bytes);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// ---- overlay --------------------------------------------------------------------------------------------------------

namespace osvos {

__device__ __forceinline__ bool fg_at(const float* l, int y, int x, int h, int w) {
  return y >= 0 && x >= 0 && y < h && x < w && l[static_cast<size_t>(y) * w + x] > 0.f;
}

// One thread per pixel: black on the mask's edge (foreground with a 4-neighbour in the background or outside the
// frame), (v + c + 1) >> 1 on the rest of the foreground, v elsewhere.
__global__ void __launch_bounds__(256) overlay_mask_kernel(const uint8_t* __restrict__ frames,
                                                           const float* __restrict__ logits, uint8_t* out, int n, int h,
                                                           int w, int c0, int c1, int c2) {
  const long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const long long hw = static_cast<long long>(h) * w;
  if (i >= n * hw) return;
  const int f = static_cast<int>(i / hw);
  const int y = static_cast<int>((i % hw) / w), x = static_cast<int>(i % w);
  const float* l = logits + static_cast<size_t>(f) * hw;
  const uint8_t* s = frames + static_cast<size_t>(i) * 3;
  uint8_t* d = out + static_cast<size_t>(i) * 3;
  uint8_t v0 = s[0], v1 = s[1], v2 = s[2];
  if (fg_at(l, y, x, h, w)) {
    const bool edge = !fg_at(l, y - 1, x, h, w) || !fg_at(l, y + 1, x, h, w) || !fg_at(l, y, x - 1, h, w) ||
                      !fg_at(l, y, x + 1, h, w);
    v0 = edge ? 0 : static_cast<uint8_t>((v0 + c0 + 1) >> 1);
    v1 = edge ? 0 : static_cast<uint8_t>((v1 + c1 + 1) >> 1);
    v2 = edge ? 0 : static_cast<uint8_t>((v2 + c2 + 1) >> 1);
  }
  d[0] = v0;
  d[1] = v1;
  d[2] = v2;
}

__device__ __forceinline__ bool same_at(const uint8_t* l, int y, int x, int h, int w, uint8_t k) {
  return y >= 0 && x >= 0 && y < h && x < w && l[static_cast<size_t>(y) * w + x] == k;
}

// One CTA per row of one frame, its threads striding along the row, one pixel each per step: 3 frame bytes in, 3 out,
// the label and its four neighbours (the neighbours come from L1 / L2; DRAM sees each label byte about once).  A CTA
// per row costs one 32-bit division per CTA where a flat pixel index costs 64-bit divisions per pixel, which bound
// the flat layout's throughput.  Object k != 0: black where a 4-neighbour holds another id or lies outside the frame,
// else (v + c_k + 1) >> 1 with c_k = colors.bgr[k] (black for k >= n_colors).  The table is a __grid_constant__ kernel
// parameter, so the per-pixel lookup reads the constant bank.  Each thread reads only its own pixel's frame bytes, so
// out may be frames itself.
constexpr int kOverlayRowThreads = 128;

__global__ void __launch_bounds__(kOverlayRowThreads) overlay_labels_kernel(
    const uint8_t* frames, const uint8_t* __restrict__ labels, uint8_t* out, int h, int w,
    const __grid_constant__ osvos_overlay_colors colors, int n_colors) {
  const int row = blockIdx.x;                          // f * h + y
  const int f = row / h, y = row - f * h;
  const uint8_t* l = labels + static_cast<size_t>(f) * h * w;
  const size_t base = static_cast<size_t>(row) * w;
  for (int x = threadIdx.x; x < w; x += kOverlayRowThreads) {
    const uint8_t k = __ldg(labels + base + x);
    const uint8_t* s = frames + (base + x) * 3;
    uint8_t* d = out + (base + x) * 3;
    uint8_t v0 = s[0], v1 = s[1], v2 = s[2];
    if (k != 0) {
      const bool edge = !same_at(l, y - 1, x, h, w, k) || !same_at(l, y + 1, x, h, w, k) ||
                        !same_at(l, y, x - 1, h, w, k) || !same_at(l, y, x + 1, h, w, k);
      const bool known = k < n_colors;
      const int c0 = known ? colors.bgr[k][0] : 0, c1 = known ? colors.bgr[k][1] : 0;
      const int c2 = known ? colors.bgr[k][2] : 0;
      v0 = edge ? 0 : static_cast<uint8_t>((v0 + c0 + 1) >> 1);
      v1 = edge ? 0 : static_cast<uint8_t>((v1 + c1 + 1) >> 1);
      v2 = edge ? 0 : static_cast<uint8_t>((v2 + c2 + 1) >> 1);
    }
    d[0] = v0;
    d[1] = v1;
    d[2] = v2;
  }
}

}  // namespace osvos

extern "C" int osvos_overlay_mask(const uint8_t* frames, const float* logits, uint8_t* out, int n, int h, int w, int c0,
                                  int c1, int c2, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(frames != nullptr && logits != nullptr && out != nullptr);
  OSVOS_CHECK_ARG(n > 0 && h > 0 && w > 0 && static_cast<long long>(n) * h * w < (1ll << 40));
  OSVOS_CHECK_ARG(c0 >= 0 && c0 <= 255 && c1 >= 0 && c1 <= 255 && c2 >= 0 && c2 <= 255);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 3) == 0);
  const long long total = static_cast<long long>(n) * h * w;
  overlay_mask_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
      frames, logits, out, n, h, w, c0, c1, c2);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_overlay_labels(const uint8_t* frames, const uint8_t* labels, uint8_t* out, int n, int h, int w,
                                    const osvos_overlay_colors* colors, int n_colors, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(frames != nullptr && labels != nullptr && out != nullptr && colors != nullptr);
  OSVOS_CHECK_ARG(n > 0 && h > 0 && w > 0 && static_cast<long long>(n) * h < (1ll << 31));
  OSVOS_CHECK_ARG(static_cast<long long>(n) * h * w < (1ll << 40));
  OSVOS_CHECK_ARG(n_colors >= 0 && n_colors <= OSVOS_OVERLAY_MAX_COLORS);
  overlay_labels_kernel<<<static_cast<unsigned>(n * h), kOverlayRowThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
      frames, labels, out, h, w, *colors, n_colors);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

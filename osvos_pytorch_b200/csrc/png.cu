// PNG encoder for 8-bit grayscale maps (the files the reference writes with sm.imsave, train_online.py:187; DESIGN.md
// §21), and for 8-bit palette maps (DAVIS-2017 label files, §24: IHDR colour type 3 and a PLTE chunk, everything
// after the header identical to the grayscale file of the same bytes).  The format is restricted so that every part
// is parallel and the bytes are a function of the frame alone:
//   filter:   per row the type 0-4 of least sum(min(v, 256 - v)) over the filtered bytes, ties to the lower type;
//   segments: R = max(1, kPngSegmentBytes / (w + 1)) filtered rows each, one IDAT chunk per segment, compressed on
//             their own (no match crosses a segment start) into one dynamic-Huffman block or one stored block,
//             whichever is smaller (stored on a tie), BFINAL 0, then an empty stored block (zlib's full flush), so
//             every segment starts and ends on a byte; the first one carries the zlib header 78 01;
//   tokens:   literals and distance-1 matches only: a run of n >= 4 equal bytes is one literal, matches of 258, then
//             a remainder of 3..257 as one more match or 1..2 as literals;
//   codes:    two-queue Huffman over the used symbols sorted by (count, symbol), per-length counts limited to 15
//             (7 for the code-length code) by moving codes down from the longest length, lengths handed out in that
//             order from the longest, canonical codes (RFC 1951), one one-bit distance code;
//   trailer:  an IDAT with a final empty fixed-Huffman block (03 00) and the big-endian Adler-32, then IEND.
// tests/png_ref.py restates it in numpy byte for byte.
// Three launches: png_filter_kernel (one warp per row), png_segment_kernel (one CTA per (frame, segment): runs,
// histogram, codes, exact bit counts, bits written at scanned offsets, the chunk's CRC from per-thread slices combined
// with x^(8n) shift operators, the segment's Adler-32 partial sums), png_assemble_kernel (one CTA per (frame,
// segment): the chunk copied to its scanned offset; the first CTA writes signature and IHDR, the last the trailer,
// IEND and the file's length).
#include "common.cuh"

namespace osvos {

constexpr int kPngSegmentBytes = 16384;
constexpr int kPngThreads = 512;
constexpr int kPngWarps = kPngThreads / 32;
constexpr int kPngLitSyms = 286;
constexpr uint32_t kCrcPoly = 0xEDB88320u;
constexpr uint32_t kAdlerMod = 65521u;
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct PngPlan {
  int rows, nseg, seg_cap;       // rows per segment, segments per frame, bytes of one segment's slot
  size_t filt_off, slot_off, size_off, adler_off, bytes;
};

inline size_t png_align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

inline bool png_dims_ok(int h, int w) { return h > 0 && w > 0 && h < 32768 && w < 32768; }

PngPlan png_plan(int n, int h, int w) {
  PngPlan p{};
  p.rows = max(1, kPngSegmentBytes / (w + 1));
  p.nseg = (h + p.rows - 1) / p.rows;
  p.seg_cap = static_cast<int>(png_align16(static_cast<size_t>(p.rows) * (w + 1) + 24));
  p.filt_off = 0;
  p.slot_off = png_align16(static_cast<size_t>(n) * h * (w + 1));
  p.size_off = p.slot_off + static_cast<size_t>(n) * p.nseg * p.seg_cap;
  p.adler_off = png_align16(p.size_off + sizeof(int) * static_cast<size_t>(n) * p.nseg);
  p.bytes = p.adler_off + 2 * sizeof(uint32_t) * static_cast<size_t>(n) * p.nseg;
  return p;
}

// signature 8, IHDR 25, zlib header 2, trailer IDAT 18, IEND 12, and per segment 12 (chunk) + 10 (the stored block's
// header and the flush) + its bytes
inline size_t png_max_bytes(int h, int w) {
  const PngPlan p = png_plan(1, h, w);
  return 65 + 22 * static_cast<size_t>(p.nseg) + static_cast<size_t>(h) * (w + 1);
}

// ---- filter ---------------------------------------------------------------------------------------------------------

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__device__ __forceinline__ int filter_cost(int v) { v &= 255; return min(v, 256 - v); }

// src [n][h][w] (any alignment) -> filt [n][h][w + 1]: the chosen type, then the filtered bytes.  One warp per row.
__global__ void __launch_bounds__(256) png_filter_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ filt,
                                                         int n, int h, int w) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= static_cast<long long>(n) * h) return;
  const int y = static_cast<int>(row % h);
  const uint8_t* x = src + row * w;
  const uint8_t* up = y > 0 ? x - w : nullptr;
  int cost[5] = {0, 0, 0, 0, 0};
  for (int i = lane; i < w; i += 32) {
    const int v = __ldg(x + i);
    const int a = i > 0 ? __ldg(x + i - 1) : 0;
    const int b = up ? __ldg(up + i) : 0;
    const int c = (up && i > 0) ? __ldg(up + i - 1) : 0;
    cost[0] += filter_cost(v);
    cost[1] += filter_cost(v - a);
    cost[2] += filter_cost(v - b);
    cost[3] += filter_cost(v - ((a + b) >> 1));
    cost[4] += filter_cost(v - paeth(a, b, c));
  }
  int best = 0, best_cost = 0;
#pragma unroll
  for (int t = 0; t < 5; ++t) {
    int s = cost[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (t == 0 || s < best_cost) { best = t; best_cost = s; }
  }
  uint8_t* out = filt + row * (w + 1);
  if (lane == 0) out[0] = static_cast<uint8_t>(best);
  for (int i = lane; i < w; i += 32) {
    const int v = __ldg(x + i);
    const int a = i > 0 ? __ldg(x + i - 1) : 0;
    const int b = up ? __ldg(up + i) : 0;
    const int c = (up && i > 0) ? __ldg(up + i - 1) : 0;
    const int pred = best == 0 ? 0 : best == 1 ? a : best == 2 ? b : best == 3 ? ((a + b) >> 1) : paeth(a, b, c);
    out[1 + i] = static_cast<uint8_t>(v - pred);
  }
}

// ---- segment --------------------------------------------------------------------------------------------------------

// GF(2) product of two CRC-32 polynomials modulo the CRC polynomial (reflected bit order), zlib's multmodp.
__device__ uint32_t crc_multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}

// x^(8 * nbytes) modulo the CRC polynomial: the operator that appends nbytes zero bytes to a CRC register.
__device__ uint32_t crc_shift_op(uint32_t nbytes, const uint32_t* x2n) {
  uint32_t p = 1u << 31;                           // x^0
  int k = 3;
  while (nbytes) {
    if (nbytes & 1) p = crc_multmodp(x2n[k & 31], p);
    nbytes >>= 1;
    ++k;
  }
  return p;
}

__device__ __forceinline__ void length_symbol(int r, int& sym, int& eb, int& ev) {
  if (r <= 10) { sym = 254 + r; eb = 0; ev = 0; return; }
  if (r == 258) { sym = 285; eb = 0; ev = 0; return; }
  const int x = r - 3;
  eb = 29 - __clz(x);                              // bit_length(x) - 3
  sym = 257 + 4 * (eb + 1) + (x >> eb) - 4;
  ev = x & ((1 << eb) - 1);
}

struct HuffScratch {
  uint16_t order[kPngLitSyms];    // used symbols by (count, symbol)
  uint32_t iw[kPngLitSyms];       // internal node weights
  int16_t ipar[kPngLitSyms], lpar[kPngLitSyms];
  uint8_t idepth[kPngLitSyms];
  int count[16];
  int nused;
};

struct SegShared {
  uint32_t crc_table[256];
  uint32_t x2n[32];
  uint32_t freq[kPngLitSyms];
  uint8_t len[kPngLitSyms];
  uint16_t code[kPngLitSyms];
  uint32_t clfreq[19];
  uint8_t cllen[19];
  uint16_t clcode[19];
  uint16_t rle[kPngLitSyms + 2];  // per item: symbol | extra value << 5
  HuffScratch hs;
  int warp_i[kPngWarps];
  unsigned long long adler1, adler2;
  uint32_t crc;
  int header_bits, nlit, ncl, nrle;
  uint32_t data_pos;               // bit position of the first data token
};

// Code lengths for freq[0..nsym) limited to maxlen, by the whole block (see the file comment).  Ends synchronised.
__device__ void huffman_lengths(const uint32_t* freq, int nsym, int maxlen, uint8_t* len, HuffScratch& s) {
  const int t = threadIdx.x;
  if (t == 0) s.nused = 0;
  __syncthreads();
  if (t < nsym) {
    len[t] = 0;
    const uint32_t f = freq[t];
    if (f) {
      int rank = 0;
      for (int j = 0; j < nsym; ++j) {
        const uint32_t g = freq[j];
        rank += g && (g < f || (g == f && j < t));
      }
      s.order[rank] = static_cast<uint16_t>(t);
      atomicAdd(&s.nused, 1);
    }
  }
  __syncthreads();
  if (t == 0) {
    const int nu = s.nused;
    int li = 0, ii = 0;
    for (int k = 0; k < nu - 1; ++k) {
      uint32_t w = 0;
      for (int pick = 0; pick < 2; ++pick) {
        if (li < nu && (ii >= k || freq[s.order[li]] <= s.iw[ii])) {
          w += freq[s.order[li]];
          s.lpar[li++] = static_cast<int16_t>(k);
        } else {
          w += s.iw[ii];
          s.ipar[ii++] = static_cast<int16_t>(k);
        }
      }
      s.iw[k] = w;
    }
    if (nu >= 2) s.idepth[nu - 2] = 0;
    for (int k = nu - 3; k >= 0; --k) s.idepth[k] = s.idepth[s.ipar[k]] + 1;
    for (int l = 0; l <= maxlen; ++l) s.count[l] = 0;
    for (int k = 0; k < nu; ++k) s.count[min(nu >= 2 ? s.idepth[s.lpar[k]] + 1 : 1, maxlen)] += 1;
    uint32_t total = 0;
    for (int l = 1; l <= maxlen; ++l) total += static_cast<uint32_t>(s.count[l]) << (maxlen - l);
    while (total > (1u << maxlen)) {
      s.count[maxlen] -= 1;
      for (int l = maxlen - 1; l > 0; --l) {
        if (s.count[l]) {
          s.count[l] -= 1;
          s.count[l + 1] += 2;
          break;
        }
      }
      --total;
    }
    int pos = 0;
    for (int l = maxlen; l > 0; --l)
      for (int c = 0; c < s.count[l]; ++c) len[s.order[pos++]] = static_cast<uint8_t>(l);
  }
  __syncthreads();
}

// Canonical codes (bit-reversed for LSB-first packing) from lengths; one thread.
__device__ void canonical_codes(const uint8_t* len, int nsym, uint16_t* code) {
  int count[16] = {0}, next[16];
  for (int s = 0; s < nsym; ++s) count[len[s]] += 1;
  count[0] = 0;
  int c = 0;
  for (int b = 1; b < 16; ++b) {
    c = (c + count[b - 1]) << 1;
    next[b] = c;
  }
  for (int s = 0; s < nsym; ++s) {
    const int l = len[s];
    if (l) code[s] = static_cast<uint16_t>(__brev(static_cast<unsigned>(next[l]++)) >> (32 - l));
  }
}

// ORs a field of nbits <= 32 into the LSB-first bit stream at bit `pos`.
__device__ __forceinline__ void put_bits(uint32_t* words, uint32_t pos, uint32_t value, int nbits) {
  if (nbits == 0) return;
  const uint32_t wi = pos >> 5, sh = pos & 31;
  atomicOr(words + wi, value << sh);
  if (sh + nbits > 32) atomicOr(words + wi + 1, value >> (32 - sh));
}

__device__ __forceinline__ int block_exclusive_sum(int v, int* warp_tot, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  __syncthreads();
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  int before = 0;
  total = 0;
  for (int k = 0; k < kPngWarps; ++k) {
    before += k < wid ? warp_tot[k] : 0;
    total += warp_tot[k];
  }
  return before + incl - v;
}

// first run start at or after the end of this thread's chunk: suffix minimum over the threads' first starts
__device__ __forceinline__ int block_next_start(int first, int* warp_min, int L) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int m = first;                                   // inclusive suffix minimum within the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_down_sync(0xffffffffu, m, o);
    if (lane + o < 32) m = min(m, u);
  }
  int excl = __shfl_down_sync(0xffffffffu, m, 1);
  if (lane == 31) excl = L;
  __syncthreads();
  if (lane == 0) warp_min[wid] = m;
  __syncthreads();
  for (int k = wid + 1; k < kPngWarps; ++k) excl = min(excl, warp_min[k]);
  return excl;
}

// Calls f(value, length) for every run of equal bytes that starts in [beg, end); `next` is the first run start at or
// after end.
template <class F>
__device__ __forceinline__ void for_each_run(const uint8_t* d, int beg, int end, int next, F f) {
  int rs = -1;
  for (int i = beg; i < end; ++i) {
    if (i == 0 || d[i] != d[i - 1]) {
      if (rs >= 0) f(d[rs], i - rs);
      rs = i;
    }
  }
  if (rs >= 0) f(d[rs], next - rs);
}

// Calls emit(symbol, extra bits, extra value, is_match) for the tokens of one run, in stream order.
template <class E>
__device__ __forceinline__ void run_tokens(int v, int n, E emit) {
  if (n < 4) {
    for (int k = 0; k < n; ++k) emit(v, 0, 0, 0);
    return;
  }
  emit(v, 0, 0, 0);
  const int m = n - 1, q = m / 258, r = m - q * 258;
  for (int k = 0; k < q; ++k) emit(285, 0, 0, 1);
  if (r >= 3) {
    int sym, eb, ev;
    length_symbol(r, sym, eb, ev);
    emit(sym, eb, ev, 1);
  } else {
    for (int k = 0; k < r; ++k) emit(v, 0, 0, 0);
  }
}

// One CTA per (segment, frame).  Dynamic shared memory: the segment's filtered bytes (seg_bytes_cap), then the chunk
// being built as 32-bit words: "IDAT", the deflate bytes (with the zlib header in segment 0).
__global__ void __launch_bounds__(kPngThreads) png_segment_kernel(const uint8_t* __restrict__ filt, uint8_t* slots,
                                                                  int* sizes, uint32_t* adler, int h, int w, int rows,
                                                                  int nseg, int seg_cap, int seg_bytes_cap) {
  extern __shared__ __align__(16) uint8_t dyn_smem[];
  __shared__ SegShared sh;
  const int t = threadIdx.x;
  const int seg = blockIdx.x, f = blockIdx.y;
  const int row_bytes = w + 1;
  const int y0 = seg * rows;
  const int L = min(rows, h - y0) * row_bytes;
  uint8_t* d = dyn_smem;
  uint32_t* words = reinterpret_cast<uint32_t*>(dyn_smem + ((seg_bytes_cap + 15) & ~15));
  uint8_t* obytes = reinterpret_cast<uint8_t*>(words);
  const uint8_t* src = filt + (static_cast<size_t>(f) * h + y0) * row_bytes;

  // tables, histogram, bytes and the Adler-32 partial sums (sum d, sum (L - i) d)
  if (t < 256) {
    uint32_t c = t;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
    sh.crc_table[t] = c;
  }
  if (t < kPngLitSyms) sh.freq[t] = t == 256 ? 1 : 0;
  if (t < 19) sh.clfreq[t] = 0;
  if (t == 0) {
    sh.adler1 = sh.adler2 = 0;
    uint32_t p = 1u << 30;                         // x^1
    sh.x2n[0] = p;
    for (int k = 1; k < 32; ++k) sh.x2n[k] = p = crc_multmodp(p, p);
  }
  unsigned long long a1 = 0, a2 = 0;
  for (int i = t; i < L; i += kPngThreads) {
    const uint8_t v = src[i];
    d[i] = v;
    a1 += v;
    a2 += static_cast<unsigned long long>(L - i) * v;
  }
  __syncthreads();
  atomicAdd(&sh.adler1, a1);
  atomicAdd(&sh.adler2, a2);

  // this thread's chunk of run starts, and the first start after it
  const int chunk = (L + kPngThreads - 1) / kPngThreads;
  const int beg = min(L, t * chunk), end = min(L, beg + chunk);
  int first = L;
  for (int i = beg; i < end; ++i) {
    if (i == 0 || d[i] != d[i - 1]) { first = i; break; }
  }
  const int next = block_next_start(first, sh.warp_i, L);
  for_each_run(d, beg, end, next, [&](int v, int n) {
    run_tokens(v, n, [&](int sym, int, int, int) { atomicAdd(&sh.freq[sym], 1u); });
  });
  __syncthreads();

  // literal / length code
  huffman_lengths(sh.freq, kPngLitSyms, 15, sh.len, sh.hs);
  if (t == 0) {
    canonical_codes(sh.len, kPngLitSyms, sh.code);
    int nlit = 257;
    for (int s = 257; s < kPngLitSyms; ++s)
      if (sh.len[s]) nlit = s + 1;
    // the code-length sequence len[0..nlit) + the distance code's length 1, run-length coded
    int nrle = 0, i = 0;
    const int total = nlit + 1;
    while (i < total) {
      const int v = i < nlit ? sh.len[i] : 1;
      int n = 1;
      while (i + n < total && (i + n < nlit ? sh.len[i + n] : 1) == v) ++n;
      i += n;
      if (v == 0) {
        while (n >= 11) {
          const int k = min(n, 138);
          sh.rle[nrle++] = static_cast<uint16_t>(18 | ((k - 11) << 5));
          n -= k;
        }
        if (n >= 3) {
          sh.rle[nrle++] = static_cast<uint16_t>(17 | ((n - 3) << 5));
          n = 0;
        }
        for (; n > 0; --n) sh.rle[nrle++] = 0;
      } else {
        sh.rle[nrle++] = static_cast<uint16_t>(v);
        --n;
        while (n >= 3) {
          const int k = min(n, 6);
          sh.rle[nrle++] = static_cast<uint16_t>(16 | ((k - 3) << 5));
          n -= k;
        }
        for (; n > 0; --n) sh.rle[nrle++] = static_cast<uint16_t>(v);
      }
    }
    for (int k = 0; k < nrle; ++k) sh.clfreq[sh.rle[k] & 31] += 1;
    sh.nlit = nlit;
    sh.nrle = nrle;
  }
  __syncthreads();
  huffman_lengths(sh.clfreq, 19, 7, sh.cllen, sh.hs);
  if (t == 0) {
    canonical_codes(sh.cllen, 19, sh.clcode);
    int ncl = 4;
    for (int k = 0; k < 19; ++k)
      if (sh.cllen[kClOrder[k]]) ncl = max(ncl, k + 1);
    int bits = 3 + 5 + 5 + 4 + 3 * ncl;
    for (int k = 0; k < sh.nrle; ++k) {
      const int s = sh.rle[k] & 31;
      bits += sh.cllen[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
    sh.ncl = ncl;
    sh.header_bits = bits + sh.len[256];            // the end-of-block code included
  }
  __syncthreads();

  // exact bit count of the data, and this thread's offset in it
  int my_bits = 0;
  for_each_run(d, beg, end, next, [&](int v, int n) {
    run_tokens(v, n, [&](int sym, int eb, int, int match) { my_bits += sh.len[sym] + eb + match; });
  });
  int data_bits = 0;
  const int my_off = block_exclusive_sum(my_bits, sh.warp_i, data_bits);
  const int head = seg == 0 ? 2 : 0;
  const int dyn_bytes = (sh.header_bits + data_bits + 3 + 7) / 8 + 4;
  const bool dynamic = dyn_bytes < L + 10;
  const int data_bytes = head + (dynamic ? dyn_bytes : L + 10);   // the chunk's data length
  const int words_used = (4 + data_bytes + 3) / 4;
  for (int k = t; k < words_used; k += kPngThreads) words[k] = 0;
  __syncthreads();
  if (t == 0) words[0] = 0x54414449u;               // "IDAT"
  if (dynamic) {
    const uint32_t base = 32 + 8 * head;
    if (t == 0) {
      if (head) put_bits(words, 32, 0x0178u, 16);
      uint32_t p = base;
      put_bits(words, p, 4u, 3);                   // BFINAL 0, BTYPE 10
      put_bits(words, p + 3, sh.nlit - 257, 5);
      put_bits(words, p + 8, 0, 5);                // one distance code
      put_bits(words, p + 13, sh.ncl - 4, 4);
      p += 17;
      for (int k = 0; k < sh.ncl; ++k, p += 3) put_bits(words, p, sh.cllen[kClOrder[k]], 3);
      for (int k = 0; k < sh.nrle; ++k) {
        const int s = sh.rle[k] & 31, ev = sh.rle[k] >> 5;
        const int eb = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
        put_bits(words, p, sh.clcode[s] | (ev << sh.cllen[s]), sh.cllen[s] + eb);
        p += sh.cllen[s] + eb;
      }
      put_bits(words, p + data_bits, sh.code[256], sh.len[256]);
      const uint32_t flush = (p + data_bits + sh.len[256] + 3 + 7) / 8;
      put_bits(words, 8 * flush + 16, 0xFFFFu, 16);   // 00 00 FF FF: the zero bytes are already there
      sh.data_pos = p;
    }
    __syncthreads();
    uint32_t p = sh.data_pos + my_off;
    for_each_run(d, beg, end, next, [&](int v, int n) {
      run_tokens(v, n, [&](int sym, int eb, int ev, int match) {
        const int l = sh.len[sym];
        put_bits(words, p, sh.code[sym] | (static_cast<uint32_t>(ev) << l), l + eb);
        p += l + eb + match;                       // the distance code is one zero bit
      });
    });
  } else {
    uint8_t* o = obytes + 4 + head;
    if (t == 0) {
      if (head) { obytes[4] = 0x78; obytes[5] = 0x01; }
      o[0] = 0;
      o[1] = static_cast<uint8_t>(L);
      o[2] = static_cast<uint8_t>(L >> 8);
      o[3] = static_cast<uint8_t>(~L);
      o[4] = static_cast<uint8_t>(~L >> 8);
      o[L + 5] = 0;
      o[L + 6] = 0;
      o[L + 7] = 0;
      o[L + 8] = 0xFF;
      o[L + 9] = 0xFF;
    }
    for (int i = t; i < L; i += kPngThreads) o[5 + i] = d[i];
  }
  if (t == 0) sh.crc = 0;
  __syncthreads();

  // CRC of "IDAT" + data: thread slices aligned to the end, so thread k's slice is followed by (T - 1 - k) * slice bytes
  const int crc_len = 4 + data_bytes;
  const int slice = (crc_len + kPngThreads - 1) / kPngThreads;
  const int s_end = crc_len - (kPngThreads - 1 - t) * slice;
  const int s_beg = max(0, s_end - slice);
  uint32_t c = 0;
  for (int i = max(0, s_beg); i < s_end; ++i) c = sh.crc_table[(c ^ obytes[i]) & 0xFF] ^ (c >> 8);
  if (s_end > 0 && t != kPngThreads - 1) c = crc_multmodp(crc_shift_op(static_cast<uint32_t>(crc_len - s_end), sh.x2n), c);
  if (s_end <= 0) c = 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
  if ((t & 31) == 0) atomicXor(&sh.crc, c);
  __syncthreads();

  // the chunk into its slot: length, "IDAT" + data, CRC
  uint8_t* slot = slots + (static_cast<size_t>(f) * nseg + seg) * seg_cap;
  for (int i = t; i < crc_len; i += kPngThreads) slot[4 + i] = obytes[i];
  if (t == 0) {
    const uint32_t crc = ~(sh.crc ^ crc_multmodp(crc_shift_op(static_cast<uint32_t>(crc_len), sh.x2n), 0xFFFFFFFFu));
    for (int k = 0; k < 4; ++k) {
      slot[k] = static_cast<uint8_t>(static_cast<uint32_t>(data_bytes) >> (24 - 8 * k));
      slot[4 + crc_len + k] = static_cast<uint8_t>(crc >> (24 - 8 * k));
    }
    sizes[f * nseg + seg] = 12 + data_bytes;
    adler[2 * (f * nseg + seg)] = static_cast<uint32_t>(sh.adler1 % kAdlerMod);
    adler[2 * (f * nseg + seg) + 1] = static_cast<uint32_t>(sh.adler2 % kAdlerMod);
  }
}

// the segment's bytes, then room for "IDAT", the zlib header and a stored block with its flush
inline int png_segment_smem(int seg_bytes_cap) { return ((seg_bytes_cap + 15) & ~15) + ((4 + 2 + seg_bytes_cap + 10 + 8) & ~3); }

// ---- assemble -------------------------------------------------------------------------------------------------------

__device__ uint32_t crc32_bytes(const uint8_t* p, int n) {
  uint32_t c = 0xFFFFFFFFu;
  for (int i = 0; i < n; ++i) {
    c ^= p[i];
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
  }
  return ~c;
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
  p[0] = static_cast<uint8_t>(v >> 24);
  p[1] = static_cast<uint8_t>(v >> 16);
  p[2] = static_cast<uint8_t>(v >> 8);
  p[3] = static_cast<uint8_t>(v);
}

// The whole PLTE chunk of a palette file (length, type, 3 * entries bytes, CRC), built on the host; bytes == 0: a
// grayscale file.
struct PngPlte {
  uint8_t chunk[12 + 3 * 256];
  int bytes;
};

__global__ void __launch_bounds__(256) png_assemble_kernel(const uint8_t* __restrict__ slots, const int* __restrict__ sizes,
                                                           const uint32_t* __restrict__ adler, uint8_t* out,
                                                           long long* lengths, int h, int w, int rows, int nseg,
                                                           int seg_cap, size_t max_bytes, PngPlte plte) {
  __shared__ unsigned long long red[3][8];
  __shared__ uint8_t tail[30];
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int seg = blockIdx.x, f = blockIdx.y;
  const bool last = seg == nseg - 1;
  const int* fs = sizes + static_cast<size_t>(f) * nseg;
  const unsigned long long N = static_cast<unsigned long long>(h) * (w + 1);
  unsigned long long off = 0, s1 = 0, s2 = 0;
  for (int k = t; k < (last ? nseg : seg); k += 256) {
    if (k < seg) off += fs[k];
    if (last) {
      const uint32_t* a = adler + 2 * (static_cast<size_t>(f) * nseg + k);
      const unsigned long long o = static_cast<unsigned long long>(k) * rows * (w + 1);
      const unsigned long long L = static_cast<unsigned long long>(min(rows, h - k * rows)) * (w + 1);
      s1 += a[0];
      s2 += (a[1] + ((N - o - L) % kAdlerMod) * a[0]) % kAdlerMod;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    off += __shfl_xor_sync(0xffffffffu, off, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lane == 0) { red[0][wid] = off; red[1][wid] = s1; red[2][wid] = s2; }
  __syncthreads();
  off = 33 + plte.bytes;                           // signature + IHDR (+ PLTE)
  s1 = 1;
  s2 = N % kAdlerMod;
  for (int k = 0; k < 8; ++k) { off += red[0][k]; s1 += red[1][k]; s2 += red[2][k]; }
  uint8_t* file = out + static_cast<size_t>(f) * max_bytes;
  const uint8_t* slot = slots + (static_cast<size_t>(f) * nseg + seg) * seg_cap;
  const int size = fs[seg];
  for (int i = t; i < size; i += 256) file[off + i] = slot[i];
  if (seg == 0 && t == 0) {
    uint8_t hdr[33] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n', 0, 0, 0, 13, 'I', 'H', 'D', 'R'};
    put_be32(hdr + 16, static_cast<uint32_t>(w));
    put_be32(hdr + 20, static_cast<uint32_t>(h));
    hdr[24] = 8;                                   // bit depth; colour type 0 (grey) or 3 (palette), no interlace
    hdr[25] = plte.bytes ? 3 : 0;
    hdr[26] = hdr[27] = hdr[28] = 0;
    put_be32(hdr + 29, crc32_bytes(hdr + 12, 17));
    for (int i = 0; i < 33; ++i) file[i] = hdr[i];
  }
  if (seg == 0)
    for (int i = t; i < plte.bytes; i += 256) file[33 + i] = plte.chunk[i];
  if (last && t == 0) {
    const uint32_t a = static_cast<uint32_t>(((s2 % kAdlerMod) << 16) | (s1 % kAdlerMod));
    const uint8_t fixed[14] = {0, 0, 0, 6, 'I', 'D', 'A', 'T', 0x03, 0x00};
    for (int i = 0; i < 10; ++i) tail[i] = fixed[i];
    put_be32(tail + 10, a);
    put_be32(tail + 14, crc32_bytes(tail + 4, 10));
    const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    for (int i = 0; i < 12; ++i) tail[18 + i] = iend[i];
    const unsigned long long end = off + size;
    for (int i = 0; i < 30; ++i) file[end + i] = tail[i];
    lengths[f] = static_cast<long long>(end + 30);
  }
}

}  // namespace osvos

using namespace osvos;

extern "C" size_t osvos_png_max_bytes(int h, int w) { return png_dims_ok(h, w) ? png_max_bytes(h, w) : 0; }

extern "C" size_t osvos_png_encode_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || n >= 65536 || !png_dims_ok(h, w)) return 0;
  return png_plan(n, h, w).bytes;
}

extern "C" size_t osvos_png_max_bytes_palette(int h, int w, int entries) {
  return png_dims_ok(h, w) && entries >= 1 && entries <= 256 ? png_max_bytes(h, w) + 12 + 3 * entries : 0;
}

static uint32_t png_host_crc32(const uint8_t* p, int n) {
  uint32_t c = 0xFFFFFFFFu;
  for (int i = 0; i < n; ++i) {
    c ^= p[i];
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
  }
  return ~c;
}

static int png_encode_impl(const uint8_t* src, const PngPlte& plte, uint8_t* out, int64_t* lengths, void* workspace,
                           int n, int h, int w, size_t max_bytes, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(src != nullptr && out != nullptr && lengths != nullptr && workspace != nullptr);
  OSVOS_CHECK_ARG(n > 0 && n < 65536 && png_dims_ok(h, w));
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(lengths) & 7) == 0);
  const PngPlan p = png_plan(n, h, w);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  uint8_t* filt = ws + p.filt_off;
  uint8_t* slots = ws + p.slot_off;
  int* sizes = reinterpret_cast<int*>(ws + p.size_off);
  uint32_t* adler = reinterpret_cast<uint32_t*>(ws + p.adler_off);
  const long long total_rows = static_cast<long long>(n) * h;
  png_filter_kernel<<<static_cast<unsigned>((total_rows + 7) / 8), 256, 0, stream>>>(src, filt, n, h, w);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  const int seg_bytes_cap = p.rows * (w + 1);
  static uint64_t smem_done = 0;
  OSVOS_CHECK_CUDA(ensure_dynamic_smem(png_segment_kernel, png_segment_smem(32768), &smem_done));
  png_segment_kernel<<<dim3(p.nseg, n), kPngThreads, png_segment_smem(seg_bytes_cap), stream>>>(filt, slots, sizes, adler, h, w, p.rows, p.nseg,
                                                                    p.seg_cap, seg_bytes_cap);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  png_assemble_kernel<<<dim3(p.nseg, n), 256, 0, stream>>>(slots, sizes, adler, out, reinterpret_cast<long long*>(lengths),
                                                           h, w, p.rows, p.nseg, p.seg_cap, max_bytes, plte);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

extern "C" int osvos_png_encode(const uint8_t* src, uint8_t* out, int64_t* lengths, void* workspace, int n, int h, int w,
                                osvos_stream_t stream) {
  PngPlte plte{};
  return png_encode_impl(src, plte, out, lengths, workspace, n, h, w, png_dims_ok(h, w) ? png_max_bytes(h, w) : 0,
                         stream);
}

extern "C" int osvos_png_encode_palette(const uint8_t* src, const uint8_t* palette, int entries, uint8_t* out,
                                        int64_t* lengths, void* workspace, int n, int h, int w, osvos_stream_t stream) {
  OSVOS_CHECK_ARG(palette != nullptr && entries >= 1 && entries <= 256);
  PngPlte plte{};
  const int len = 3 * entries;
  plte.chunk[0] = plte.chunk[1] = 0;
  plte.chunk[2] = static_cast<uint8_t>(len >> 8);
  plte.chunk[3] = static_cast<uint8_t>(len);
  memcpy(plte.chunk + 4, "PLTE", 4);
  memcpy(plte.chunk + 8, palette, len);
  const uint32_t crc = png_host_crc32(plte.chunk + 4, 4 + len);
  for (int k = 0; k < 4; ++k) plte.chunk[8 + len + k] = static_cast<uint8_t>(crc >> (24 - 8 * k));
  plte.bytes = 12 + len;
  return png_encode_impl(src, plte, out, lengths, workspace, n, h, w, osvos_png_max_bytes_palette(h, w, entries), stream);
}

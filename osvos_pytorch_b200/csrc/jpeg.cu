// Baseline JPEG decode bit-identical to cv2.imread (libjpeg-turbo 3.1 as OpenCV configures it: ISLOW IDCT, fancy
// upsampling, fixed-point YCbCr -> BGR; DESIGN.md §19).  The host (osvos_pytorch_b200/jpeg.py) parses the markers and
// packs a batch into one blob: headers, quantisation tables in natural order, Huffman lookup tables and the de-stuffed
// entropy-coded segments, split at RST markers.  The stages:
//   1. sync:  one CTA per segment.  The segment is cut into chunks of S bits; a window of blockDim chunks is decoded
//             speculatively, each chunk from (its first bit, block 0 of the MCU, zig-zag 0), recording the state it
//             leaves its chunk in.  In rounds, a chunk whose predecessor's exit state differs from its entry state
//             re-decodes from the corrected state until no exit changes (chunk 0 starts from the true state, so round
//             r has at least r chunks right).  The window's block counts go through an exclusive scan; the last exit
//             state and the block total carry into the next window.
//   2. write: one thread per chunk decodes again from its synced entry and writes int16 coefficients in natural
//             order (the DC slot holds the difference) into a zeroed buffer, capped at the segment's block count.
//   3. dc:    one CTA per segment: a scan of the DC differences per component in MCU order (reset at each restart).
//   4. idct:  one thread per block: dequantise, jidctint.c's ISLOW IDCT with its 10-bit range-limit wrap, into a
//             component plane padded to whole MCUs.
//   5. color: one thread per pixel: jdsample.c's fancy upsampling with its edge rules, jdcolor.c's tables -> BGR.
// libjpeg-turbo's rules for short data are kept: bits past a segment's end read as zero, the MCU in which the data
// ran out is decoded from those zeros, and the MCUs after it in that segment stay zero (DC included).  Every loop is
// bounded by the segment's length: each Huffman symbol consumes at least one bit.
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace osvos {

constexpr uint32_t kJpegMagic = 0x3147504A;
constexpr int kSyncThreads = 256;
constexpr int kDcThreads = 256;
constexpr int kJpegThreads = 256;
constexpr int kStatusBadCode = 1, kStatusZigzag = 2, kStatusShort = 4, kStatusBadHeader = 8;

struct JpegHeader {
  int32_t magic, n, nseg, nq, nh, pad[3];
  int64_t img_off, seg_off, q_off, h_off, data_off, data_bytes;
};
struct JpegImage {
  int32_t h, w, ncomp, hs, vs, mcux, mcuy, bpm, restart, seg0, nseg, q[3], dc[3], ac[3], pad[4];
};
struct JpegSegment {
  int64_t byte_off, nbits;
  int32_t image, first_block, nblocks, pad;
};
struct HuffTable {
  uint16_t lookup[512];            // (length << 8) | symbol for codes of <= 9 bits; length 10: longer code
  int32_t maxcode[18];
  int32_t valoffset[18];
  uint8_t vals[256];
};
static_assert(sizeof(JpegHeader) == 80 && sizeof(JpegImage) == 96 && sizeof(JpegSegment) == 32 &&
              sizeof(HuffTable) == 1424, "layout of osvos_pytorch_b200/jpeg.py");

__constant__ uint8_t kNatural[80] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33,
                                     40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36,
                                     29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
                                     47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

struct JpegParams {
  const uint8_t* blob;
  size_t blob_bytes;
  uint8_t* out;
  int32_t* status;
  int16_t* coef;         // [n][max_blocks][64]
  uint8_t* planes;       // [n][plane_bytes]
  int64_t* entry;        // [max_chunks] synced entry state per chunk
  int32_t* first;        // [max_chunks] first block (segment-local) per chunk
  int32_t* decoded;      // [nseg] blocks decoded per segment
  int n, h, w, nseg, S;
  int64_t max_blocks, plane_bytes;
};

// ---- blob access ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ const JpegHeader* hdr(const JpegParams& p) {
  return reinterpret_cast<const JpegHeader*>(p.blob);
}

// The blob's header agrees with the arguments and every table lies inside the blob.
__device__ bool header_ok(const JpegParams& p) {
  const JpegHeader* hd = hdr(p);
  const int64_t b = static_cast<int64_t>(p.blob_bytes);
  auto fits = [b](int64_t off, int64_t count, int64_t size) {
    return off >= static_cast<int64_t>(sizeof(JpegHeader)) && (off & 15) == 0 && count >= 0 && off <= b &&
           count <= (b - off) / size;
  };
  return hd->magic == static_cast<int32_t>(kJpegMagic) && hd->n == p.n && hd->nseg == p.nseg &&
         fits(hd->img_off, hd->n, sizeof(JpegImage)) && fits(hd->seg_off, hd->nseg, sizeof(JpegSegment)) &&
         fits(hd->q_off, hd->nq, 128) && fits(hd->h_off, hd->nh, sizeof(HuffTable)) &&
         fits(hd->data_off, hd->data_bytes, 1);
}

__device__ __forceinline__ const JpegImage& image(const JpegParams& p, int i) {
  return reinterpret_cast<const JpegImage*>(p.blob + hdr(p)->img_off)[i];
}
__device__ __forceinline__ const JpegSegment& segment(const JpegParams& p, int s) {
  return reinterpret_cast<const JpegSegment*>(p.blob + hdr(p)->seg_off)[s];
}
__device__ __forceinline__ const HuffTable* huff(const JpegParams& p, int t) {
  return reinterpret_cast<const HuffTable*>(p.blob + hdr(p)->h_off) + t;
}
__device__ __forceinline__ const uint16_t* qtable(const JpegParams& p, int t) {
  return reinterpret_cast<const uint16_t*>(p.blob + hdr(p)->q_off) + 64 * t;
}

__device__ __forceinline__ int block_component(const JpegImage& im, int k) {
  const int nl = im.hs * im.vs;
  return im.ncomp == 1 ? 0 : (k < nl ? 0 : k - nl + 1);
}

__device__ __forceinline__ int64_t chunk_base(const JpegParams& p, int s) {      // first chunk slot of segment s
  return s + segment(p, s).byte_off * 8 / p.S;
}
__device__ __forceinline__ int chunk_count(const JpegParams& p, int s) {
  const int64_t nb = segment(p, s).nbits;
  return nb == 0 ? 1 : static_cast<int>((nb + p.S - 1) / p.S);
}

// ---- Huffman decoding ----------------------------------------------------------------------------------------------
// State at a symbol boundary, packed: bit position << 16 | block in MCU << 8 | zig-zag index.
__device__ __forceinline__ int64_t pack_state(int64_t pos, int blk, int zz) { return (pos << 16) | (blk << 8) | zz; }

struct BitReader {
  const uint8_t* d;
  int64_t nbytes;
  int64_t win_pos;     // bit position of win's most significant bit
  uint64_t win;
  __device__ void load(int64_t pos) {
    const int64_t b = pos >> 3;
    uint64_t v = 0;
    if (b + 8 <= nbytes) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v = (v << 8) | __ldg(d + b + i);
    } else {
      for (int i = 0; i < 8; ++i) v = (v << 8) | (b + i < nbytes ? __ldg(d + b + i) : 0u);   // zeros past the end
    }
    win = v;
    win_pos = b * 8;
  }
  // 32 bits from `pos` on (bits past the segment's end are zero).
  __device__ __forceinline__ uint32_t peek32(int64_t pos) {
    if (static_cast<uint64_t>(pos - win_pos) > 32) load(pos);
    return static_cast<uint32_t>((win << (pos - win_pos)) >> 32);
  }
};

struct Tables {
  const HuffTable* dc[3];
  const HuffTable* ac[3];
  int ncomp, nl, bpm;
};

// -> symbol; *len = code length; a bad code decodes as symbol 0 after 16 bits, as libjpeg-turbo's slow path.
__device__ __forceinline__ int huff_symbol(const HuffTable* t, uint32_t v, int* len, int* bad) {
  const uint32_t p16 = v >> 16;
  const int e = t->lookup[p16 >> 7];
  if ((e >> 8) >= 1 && (e >> 8) <= 9) {
    *len = e >> 8;
    return e & 0xFF;
  }
  int l = 10;
  while (l <= 16 && static_cast<int>(p16 >> (16 - l)) > t->maxcode[l]) ++l;
  if (l > 16) {
    *len = 16;
    *bad = 1;
    return 0;
  }
  *len = l;
  return t->vals[(static_cast<int>(p16 >> (16 - l)) + t->valoffset[l]) & 0xFF];
}

__device__ __forceinline__ int extend(uint32_t r, int s) {
  return static_cast<int>(r) < (1 << (s - 1)) ? static_cast<int>(r) - (1 << s) + 1 : static_cast<int>(r);
}

// Decode from `state` while pos < end (`last`: the segment's last chunk stops only at an MCU boundary past the
// segment's end).  Emit(block, zz, value) receives each coefficient (zz 0: the DC difference) and End(block, end_pos,
// flags) each completed block, `block` counting blocks completed in this span.  Returns the exit state; *nblocks the
// blocks completed.
template <bool kEmit, class Emit, class End>
__device__ int64_t decode_span(BitReader& br, const Tables& tb, int64_t state, int64_t end, bool last, int64_t nbits,
                               int* nblocks, Emit emit, End block_end) {
  int64_t pos = state >> 16;
  int blk = (state >> 8) & 0xFF, zz = state & 0xFF;
  int nb = 0, flags = 0;
  while (true) {
    if (last ? (blk == 0 && zz == 0 && pos > nbits) : pos >= end) break;
    const int c = tb.ncomp == 1 ? 0 : (blk < tb.nl ? 0 : blk - tb.nl + 1);
    const uint32_t v = br.peek32(pos);
    int len, bad = 0;
    if (zz == 0) {
      int s = huff_symbol(tb.dc[c], v, &len, &bad);
      if (s > 15) {                                  // a DC category libjpeg rejects with its table
        s = 0;
        bad = 1;
      }
      const int val = s ? extend((v << len) >> (32 - s), s) : 0;
      pos += len + s;
      if (kEmit) emit(nb, 0, val);
      zz = 1;
    } else {
      const int rs = huff_symbol(tb.ac[c], v, &len, &bad);
      const int r = rs >> 4, s = rs & 15;
      if (s) {
        zz += r;
        if (zz > 63) flags |= kStatusZigzag;
        const int val = extend((v << len) >> (32 - s), s);
        pos += len + s;
        if (kEmit) emit(nb, zz, val);
        ++zz;
      } else {
        pos += len;
        if (r == 15) {
          zz += 16;
          if (zz > 64) flags |= kStatusZigzag;
        } else {
          zz = 64;
        }
      }
    }
    if (bad) flags |= kStatusBadCode;
    if (zz >= 64) {
      if (kEmit) block_end(nb, pos, flags);
      flags = 0;
      ++nb;
      zz = 0;
      blk = blk + 1 < tb.bpm ? blk + 1 : 0;
    }
  }
  *nblocks = nb;
  return pack_state(pos, blk, zz);
}

struct NoEmit {
  __device__ void operator()(int, int, int) const {}
  __device__ void operator()(int, int64_t, int) const {}
};

// Image i is decodable: its header agrees with the call, sampling and tables are in range.  Its segments are checked by
// the kernels that read them (segment_ok).
__device__ bool image_ok(const JpegParams& p, const JpegImage& im) {
  const JpegHeader* hd = hdr(p);
  if (im.h != p.h || im.w != p.w || (im.ncomp != 1 && im.ncomp != 3)) return false;
  if (im.hs < 1 || im.hs > 2 || im.vs < 1 || im.vs > 2 || (im.ncomp == 1 && (im.hs != 1 || im.vs != 1))) return false;
  if (im.mcux != (im.w + 8 * im.hs - 1) / (8 * im.hs) || im.mcuy != (im.h + 8 * im.vs - 1) / (8 * im.vs)) return false;
  if (im.bpm != (im.ncomp == 3 ? im.hs * im.vs + 2 : 1) || im.restart < 1) return false;
  const int64_t mcus = static_cast<int64_t>(im.mcux) * im.mcuy;
  if (static_cast<int64_t>(im.nseg) != (mcus + im.restart - 1) / im.restart) return false;
  if (im.seg0 < 0 || im.nseg < 1 || im.seg0 > hd->nseg - im.nseg) return false;
  for (int c = 0; c < im.ncomp; ++c)
    if (im.q[c] < 0 || im.q[c] >= hd->nq || im.dc[c] < 0 || im.dc[c] >= hd->nh || im.ac[c] < 0 || im.ac[c] >= hd->nh)
      return false;
  return true;
}

__device__ bool segment_ok(const JpegParams& p, const JpegSegment& sg, int s) {
  const JpegHeader* hd = hdr(p);
  if (sg.image < 0 || sg.image >= p.n) return false;
  const JpegImage& im = image(p, sg.image);
  const int k = s - im.seg0;
  if (k < 0 || k >= im.nseg) return false;
  const int64_t per = static_cast<int64_t>(im.restart) * im.bpm;
  const int64_t total = static_cast<int64_t>(im.mcux) * im.mcuy * im.bpm;
  return sg.first_block == k * per && sg.nblocks == min(per, total - k * per) && sg.byte_off >= 0 &&
         (sg.nbits & 7) == 0 && sg.nbits >= 0 && sg.byte_off <= hd->data_bytes &&
         sg.nbits / 8 <= hd->data_bytes - sg.byte_off && (s == 0 || (segment(p, s - 1).byte_off >= 0 && segment(p, s - 1).nbits >= 0 &&
                     segment(p, s - 1).byte_off + segment(p, s - 1).nbits / 8 <= sg.byte_off));
}

// ---- 0. validation -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kJpegThreads) jpeg_validate_kernel(JpegParams p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  bool ok = header_ok(p) && image_ok(p, image(p, i));
  if (ok) {
    const JpegImage& im = image(p, i);
    for (int s = im.seg0; s < im.seg0 + im.nseg && ok; ++s) ok = segment_ok(p, segment(p, s), s);
  }
  p.status[i] = ok ? 0 : kStatusBadHeader;
}

__device__ __forceinline__ bool segment_live(const JpegParams& p, int s) {
  const int i = segment(p, s).image;
  if (i < 0 || i >= p.n || (p.status[i] & kStatusBadHeader)) return false;   // other bits: decode it still
  const JpegImage& im = image(p, i);
  return s >= im.seg0 && s < im.seg0 + im.nseg;      // validated with its image
}

__device__ void load_tables(const JpegParams& p, const JpegImage& im, Tables& tb) {
  tb.ncomp = im.ncomp;
  tb.nl = im.hs * im.vs;
  tb.bpm = im.bpm;
  for (int c = 0; c < 3; ++c) {
    const int cc = c < im.ncomp ? c : 0;
    tb.dc[c] = huff(p, im.dc[cc]);
    tb.ac[c] = huff(p, im.ac[cc]);
  }
}

// ---- 1. speculative decode and synchronisation ---------------------------------------------------------------------
__global__ void __launch_bounds__(kSyncThreads) jpeg_sync_kernel(JpegParams p) {
  using Scan = cub::BlockScan<int, kSyncThreads>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int64_t s_exit[kSyncThreads];
  __shared__ int64_t s_carry;
  __shared__ int s_carry_blocks;
  __shared__ HuffTable s_tab[6];                               // the segment's DC and AC tables per component
  const int s = blockIdx.x;
  if (!header_ok(p) || !segment_live(p, s)) return;
  const JpegSegment& sg = segment(p, s);
  const JpegImage& im = image(p, sg.image);
  Tables tb;
  load_tables(p, im, tb);
  constexpr int kWords = sizeof(HuffTable) / 4;
  for (int k = threadIdx.x; k < 6 * kWords; k += blockDim.x) {
    const int j = k / kWords;
    const HuffTable* src = j < 3 ? tb.dc[j] : tb.ac[j - 3];
    reinterpret_cast<uint32_t*>(s_tab + j)[k - j * kWords] = reinterpret_cast<const uint32_t*>(src)[k - j * kWords];
  }
  for (int c = 0; c < 3; ++c) {
    tb.dc[c] = s_tab + c;
    tb.ac[c] = s_tab + 3 + c;
  }
  BitReader br{p.blob + hdr(p)->data_off + sg.byte_off, sg.nbits / 8, INT64_MIN / 2, 0};
  const int nch = chunk_count(p, s);
  const int64_t base = chunk_base(p, s);
  const int t = threadIdx.x;
  if (t == 0) {
    s_carry = 0;
    s_carry_blocks = 0;
  }
  __syncthreads();
  for (int w0 = 0; w0 < nch; w0 += kSyncThreads) {
    const int c = w0 + t;
    const bool active = c < nch;
    const int64_t end = min(static_cast<int64_t>(c + 1) * p.S, sg.nbits);
    const bool last = c == nch - 1;
    int64_t entry = t == 0 ? s_carry : pack_state(static_cast<int64_t>(c) * p.S, 0, 0);
    int cnt = 0;
    int64_t exit_state = entry;
    if (active) exit_state = decode_span<false>(br, tb, entry, end, last, sg.nbits, &cnt, NoEmit{}, NoEmit{});
    s_exit[t] = exit_state;
    for (int round = 0; round <= kSyncThreads; ++round) {
      __syncthreads();
      const int64_t pred = t == 0 ? entry : s_exit[t - 1];
      const bool changed = active && pred != entry;
      __syncthreads();
      if (changed) {
        entry = pred;
        exit_state = decode_span<false>(br, tb, entry, end, last, sg.nbits, &cnt, NoEmit{}, NoEmit{});
        s_exit[t] = exit_state;
      }
      if (!__syncthreads_or(changed)) break;
    }
    int off, total;
    Scan(scan_tmp).ExclusiveSum(active ? cnt : 0, off, total);
    if (active) {
      p.entry[base + c] = entry;
      p.first[base + c] = s_carry_blocks + off;
    }
    __syncthreads();
    if (t == min(nch - w0, kSyncThreads) - 1) {
      s_carry = exit_state;
      s_carry_blocks += total;
    }
    __syncthreads();
  }
  if (t == 0) {
    p.decoded[s] = min(s_carry_blocks, sg.nblocks);
    if (s_carry_blocks < sg.nblocks) atomicOr(p.status + sg.image, kStatusShort);
  }
}

// ---- 2. coefficients -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kJpegThreads) jpeg_write_kernel(JpegParams p, int64_t chunk_slots) {
  const int64_t slot = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (slot >= chunk_slots || !header_ok(p)) return;
  int lo = 0, hi = p.nseg - 1;                                  // last segment with chunk_base <= slot
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (chunk_base(p, mid) <= slot) lo = mid; else hi = mid - 1;
  }
  const int s = lo;
  const int c = static_cast<int>(slot - chunk_base(p, s));
  if (c < 0 || c >= chunk_count(p, s) || !segment_live(p, s)) return;
  const JpegSegment& sg = segment(p, s);
  const JpegImage& im = image(p, sg.image);
  Tables tb;
  load_tables(p, im, tb);
  BitReader br{p.blob + hdr(p)->data_off + sg.byte_off, sg.nbits / 8, INT64_MIN / 2, 0};
  const int nch = chunk_count(p, s);
  const int64_t end = min(static_cast<int64_t>(c + 1) * p.S, sg.nbits);
  const int first = p.first[slot];
  const int limit = sg.nblocks;
  int16_t* coef = p.coef + (static_cast<size_t>(sg.image) * p.max_blocks + sg.first_block) * 64;
  int32_t* status = p.status + sg.image;
  const int64_t nbits = sg.nbits;
  int nb;
  decode_span<true>(
      br, tb, p.entry[slot], end, c == nch - 1, nbits, &nb,
      [&](int b, int zz, int v) {
        if (first + b < limit) coef[static_cast<size_t>(first + b) * 64 + kNatural[min(zz, 79)]] = static_cast<int16_t>(v);
      },
      [&](int b, int64_t pos, int flags) {
        if (first + b < limit && (flags != 0 || pos > nbits)) atomicOr(status, flags | (pos > nbits ? kStatusShort : 0));
      });
}

// ---- 3. DC prefix sums ---------------------------------------------------------------------------------------------
struct Int3 {
  int v[3];
};
struct Int3Sum {
  __device__ Int3 operator()(const Int3& a, const Int3& b) const {
    return Int3{{a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2]}};
  }
};

__global__ void __launch_bounds__(kDcThreads) jpeg_dc_kernel(JpegParams p) {
  using Scan = cub::BlockScan<Int3, kDcThreads>;
  __shared__ typename Scan::TempStorage scan_tmp;
  const int s = blockIdx.x;
  if (!header_ok(p) || !segment_live(p, s)) return;
  const JpegSegment& sg = segment(p, s);
  const JpegImage& im = image(p, sg.image);
  int16_t* coef = p.coef + (static_cast<size_t>(sg.image) * p.max_blocks + sg.first_block) * 64;
  const int done = p.decoded[s];
  Int3 carry{{0, 0, 0}};
  for (int b0 = 0; b0 < done; b0 += kDcThreads) {           // sg.first_block is a whole number of MCUs
    const int b = b0 + threadIdx.x;
    const int c = block_component(im, b % im.bpm);
    Int3 v{{0, 0, 0}};
    if (b < done) v.v[c] = coef[static_cast<size_t>(b) * 64];
    Int3 incl, agg;
    Scan(scan_tmp).InclusiveScan(v, incl, Int3Sum(), agg);
    if (b < done) coef[static_cast<size_t>(b) * 64] = static_cast<int16_t>(carry.v[c] + incl.v[c]);
    carry = Int3Sum()(carry, agg);
    __syncthreads();
  }
}

// ---- 4. IDCT -------------------------------------------------------------------------------------------------------
struct PlaneGeom {
  int64_t off[3];
  int pitch[3];
};

__device__ __forceinline__ PlaneGeom plane_geom(const JpegImage& im) {
  PlaneGeom g;
  g.pitch[0] = im.mcux * im.hs * 8;
  g.pitch[1] = g.pitch[2] = im.mcux * 8;
  g.off[0] = 0;
  g.off[1] = static_cast<int64_t>(g.pitch[0]) * im.mcuy * im.vs * 8;
  g.off[2] = g.off[1] + static_cast<int64_t>(g.pitch[1]) * im.mcuy * 8;
  return g;
}

constexpr int kFix0298 = 2446, kFix0390 = 3196, kFix0541 = 4433, kFix0765 = 6270, kFix0899 = 7373, kFix1175 = 9633,
              kFix1501 = 12299, kFix1847 = 15137, kFix1961 = 16069, kFix2053 = 16819, kFix2562 = 20995,
              kFix3072 = 25172;

// One 1-D pass of jidctint.c on x[0..7] (stride `st`), descaled by `shift` bits.
template <class T>
__device__ __forceinline__ void idct_1d(T* x, int st, int shift) {
  const int64_t x0 = x[0], x1 = x[st], x2 = x[2 * st], x3 = x[3 * st], x4 = x[4 * st], x5 = x[5 * st], x6 = x[6 * st],
                x7 = x[7 * st];
  int64_t z1 = (x2 + x6) * kFix0541;
  const int64_t tmp2e = z1 - x6 * kFix1847;
  const int64_t tmp3e = z1 + x2 * kFix0765;
  const int64_t tmp0e = (x0 + x4) * 8192;
  const int64_t tmp1e = (x0 - x4) * 8192;
  const int64_t t10 = tmp0e + tmp3e, t13 = tmp0e - tmp3e, t11 = tmp1e + tmp2e, t12 = tmp1e - tmp2e;
  int64_t z2, z3, z4;
  z1 = x7 + x1;
  z2 = x5 + x3;
  z3 = x7 + x3;
  z4 = x5 + x1;
  const int64_t z5 = (z3 + z4) * kFix1175;
  int64_t a0 = x7 * kFix0298, a1 = x5 * kFix2053, a2 = x3 * kFix3072, a3 = x1 * kFix1501;
  z1 *= -kFix0899;
  z2 *= -kFix2562;
  z3 = z3 * -kFix1961 + z5;
  z4 = z4 * -kFix0390 + z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  const int64_t r = int64_t(1) << (shift - 1);
  x[0] = static_cast<T>((t10 + a3 + r) >> shift);
  x[7 * st] = static_cast<T>((t10 - a3 + r) >> shift);
  x[st] = static_cast<T>((t11 + a2 + r) >> shift);
  x[6 * st] = static_cast<T>((t11 - a2 + r) >> shift);
  x[2 * st] = static_cast<T>((t12 + a1 + r) >> shift);
  x[5 * st] = static_cast<T>((t12 - a1 + r) >> shift);
  x[3 * st] = static_cast<T>((t13 + a0 + r) >> shift);
  x[4 * st] = static_cast<T>((t13 - a0 + r) >> shift);
}

__global__ void __launch_bounds__(kJpegThreads) jpeg_idct_kernel(JpegParams p) {
  const int i = blockIdx.y;
  const int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p.status[i] & kStatusBadHeader) return;
  const JpegImage& im = image(p, i);
  const int64_t total = static_cast<int64_t>(im.mcux) * im.mcuy * im.bpm;
  if (g >= total) return;
  const int m = static_cast<int>(g / im.bpm), k = static_cast<int>(g % im.bpm);
  const int c = block_component(im, k);
  const int my = m / im.mcux, mx = m - my * im.mcux;
  const int by = c == 0 ? my * im.vs + k / im.hs : my;
  const int bx = c == 0 ? mx * im.hs + k % im.hs : mx;
  const int16_t* src = p.coef + (static_cast<size_t>(i) * p.max_blocks + g) * 64;
  const uint16_t* q = qtable(p, im.q[c]);
  int ws[64];
  const int4* s4 = reinterpret_cast<const int4*>(src);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int4 v = s4[j];
    const int words[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c16 = static_cast<int16_t>(static_cast<uint32_t>(words[e >> 1]) >> (16 * (e & 1)));
      ws[8 * j + e] = c16 * static_cast<int>(__ldg(q + 8 * j + e));
    }
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) idct_1d(ws + u, 8, 11);              // columns, scaled by 2^PASS1_BITS
  const PlaneGeom pg = plane_geom(im);
  uint8_t* dst = p.planes + static_cast<size_t>(i) * p.plane_bytes + pg.off[c] + static_cast<int64_t>(by) * 8 * pg.pitch[c] +
                 bx * 8;
#pragma unroll
  for (int y = 0; y < 8; ++y) {
    idct_1d(ws + 8 * y, 1, 18);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      const int v = ((ws[8 * y + x] & 1023) ^ 512) - 512;        // the 10-bit range-limit wrap, then the clamp
      const uint32_t b = static_cast<uint32_t>(min(max(v + 128, 0), 255));
      if (x < 4) lo |= b << (8 * x); else hi |= b << (8 * (x - 4));
    }
    *reinterpret_cast<uint2*>(dst + static_cast<int64_t>(y) * pg.pitch[c]) = make_uint2(lo, hi);
  }
}

// ---- 5. upsampling and colour --------------------------------------------------------------------------------------
// Chroma at luma pixel (y, x): libjpeg-turbo's h2v1 / h1v2 / h2v2 fancy upsampling (box when the downsampled width is
// <= 2 for h2v1 / h2v2), context rows replicated at the top and bottom of the image.
__device__ __forceinline__ int chroma(const uint8_t* pl, int pitch, int hs, int vs, int dw, int dh, int y, int x) {
  if (hs == 1 && vs == 1) return pl[static_cast<int64_t>(y) * pitch + x];
  if (vs == 1) {
    const uint8_t* r = pl + static_cast<int64_t>(y) * pitch;
    const int j = x >> 1;
    if (dw <= 2) return r[j];
    if ((x & 1) == 0) return j == 0 ? r[0] : (3 * r[j] + r[j - 1] + 1) >> 2;
    return j == dw - 1 ? r[j] : (3 * r[j] + r[j + 1] + 2) >> 2;
  }
  const int rr = y >> 1;
  const int r1 = min(max((y & 1) ? rr + 1 : rr - 1, 0), dh - 1);
  const uint8_t* r0p = pl + static_cast<int64_t>(rr) * pitch;
  const uint8_t* r1p = pl + static_cast<int64_t>(r1) * pitch;
  if (hs == 1) return (3 * r0p[x] + r1p[x] + ((y & 1) ? 2 : 1)) >> 2;
  const int j = x >> 1;
  if (dw <= 2) return r0p[j];
  const int cs = 3 * r0p[j] + r1p[j];
  if ((x & 1) == 0) return j == 0 ? (cs * 4 + 8) >> 4 : (3 * cs + 3 * r0p[j - 1] + r1p[j - 1] + 8) >> 4;
  return j == dw - 1 ? (cs * 4 + 7) >> 4 : (3 * cs + 3 * r0p[j + 1] + r1p[j + 1] + 7) >> 4;
}

__global__ void __launch_bounds__(kJpegThreads) jpeg_color_kernel(JpegParams p) {
  const int i = blockIdx.z, y = blockIdx.y;
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= p.w || (p.status[i] & kStatusBadHeader)) return;
  const JpegImage& im = image(p, i);
  const PlaneGeom pg = plane_geom(im);
  const uint8_t* base = p.planes + static_cast<size_t>(i) * p.plane_bytes;
  const int yy = base[pg.off[0] + static_cast<int64_t>(y) * pg.pitch[0] + x];
  uint8_t* o = p.out + ((static_cast<size_t>(i) * p.h + y) * p.w + x) * 3;
  if (im.ncomp == 1) {
    o[0] = o[1] = o[2] = static_cast<uint8_t>(yy);
    return;
  }
  const int dw = (p.w + im.hs - 1) / im.hs, dh = (p.h + im.vs - 1) / im.vs;
  const int cb = chroma(base + pg.off[1], pg.pitch[1], im.hs, im.vs, dw, dh, y, x) - 128;
  const int cr = chroma(base + pg.off[2], pg.pitch[2], im.hs, im.vs, dw, dh, y, x) - 128;
  constexpr int kHalf = 1 << 15;
  const int r = yy + ((91881 * cr + kHalf) >> 16);                 // FIX(1.40200)
  const int b = yy + ((116130 * cb + kHalf) >> 16);                // FIX(1.77200)
  const int g = yy + ((-22554 * cb + kHalf - 46802 * cr) >> 16);   // FIX(0.34414), FIX(0.71414)
  o[0] = static_cast<uint8_t>(min(max(b, 0), 255));
  o[1] = static_cast<uint8_t>(min(max(g, 0), 255));
  o[2] = static_cast<uint8_t>(min(max(r, 0), 255));
}

// ---- workspace -----------------------------------------------------------------------------------------------------
struct JpegPlan {
  int S;
  int64_t max_blocks, plane_bytes, chunk_slots;
  size_t coef_off, planes_off, entry_off, first_off, decoded_off, bytes;
};

inline size_t align16j(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

JpegPlan jpeg_plan(int n, int h, int w, int nseg, size_t blob_bytes, int chunk_bits) {
  JpegPlan p{};
  p.S = chunk_bits == 0 ? OSVOS_JPEG_DEFAULT_CHUNK_BITS : chunk_bits;
  const int64_t mh = (h + 15) / 16, mw = (w + 15) / 16;
  p.max_blocks = 3 * (2 * mh) * (2 * mw);                         // bounds every supported sampling
  p.plane_bytes = 3 * (16 * mh) * (16 * mw);
  p.chunk_slots = nseg + (static_cast<int64_t>(blob_bytes) * 8 + p.S - 1) / p.S;
  p.coef_off = 0;
  p.planes_off = align16j(sizeof(int16_t) * 64 * static_cast<size_t>(n) * p.max_blocks);
  p.entry_off = p.planes_off + align16j(static_cast<size_t>(n) * p.plane_bytes);
  p.first_off = p.entry_off + align16j(sizeof(int64_t) * p.chunk_slots);
  p.decoded_off = p.first_off + align16j(sizeof(int32_t) * p.chunk_slots);
  p.bytes = p.decoded_off + align16j(sizeof(int32_t) * nseg);
  return p;
}

}  // namespace osvos

using namespace osvos;

static bool jpeg_dims_ok(int n, int h, int w, int nseg, size_t blob_bytes, int chunk_bits) {
  return n > 0 && n < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768 && nseg >= n && nseg < (1 << 30) &&
         blob_bytes >= sizeof(JpegHeader) && blob_bytes < (static_cast<size_t>(1) << 31) &&
         (chunk_bits == 0 || (chunk_bits >= 32 && chunk_bits <= (1 << 20)));
}

extern "C" size_t osvos_jpeg_decode_workspace_bytes(int n, int h, int w, int nseg, size_t blob_bytes, int chunk_bits) {
  if (!jpeg_dims_ok(n, h, w, nseg, blob_bytes, chunk_bits)) return 0;
  return jpeg_plan(n, h, w, nseg, blob_bytes, chunk_bits).bytes;
}

extern "C" int osvos_jpeg_decode(const osvos_jpeg_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr);
  OSVOS_CHECK_ARG(a->blob != nullptr && a->out != nullptr && a->status != nullptr && a->workspace != nullptr);
  OSVOS_CHECK_ARG(jpeg_dims_ok(a->n, a->h, a->w, a->nseg, a->blob_bytes, a->chunk_bits));
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->blob) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->status) & 3) == 0);
  const JpegPlan pl = jpeg_plan(a->n, a->h, a->w, a->nseg, a->blob_bytes, a->chunk_bits);
  uint8_t* ws = static_cast<uint8_t*>(a->workspace);
  JpegParams p{};
  p.blob = static_cast<const uint8_t*>(a->blob);
  p.blob_bytes = a->blob_bytes;
  p.out = a->out;
  p.status = a->status;
  p.coef = reinterpret_cast<int16_t*>(ws + pl.coef_off);
  p.planes = ws + pl.planes_off;
  p.entry = reinterpret_cast<int64_t*>(ws + pl.entry_off);
  p.first = reinterpret_cast<int32_t*>(ws + pl.first_off);
  p.decoded = reinterpret_cast<int32_t*>(ws + pl.decoded_off);
  p.n = a->n;
  p.h = a->h;
  p.w = a->w;
  p.nseg = a->nseg;
  p.S = pl.S;
  p.max_blocks = pl.max_blocks;
  p.plane_bytes = pl.plane_bytes;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  OSVOS_CHECK_CUDA(cudaMemsetAsync(p.coef, 0, pl.planes_off, stream));
  jpeg_validate_kernel<<<(a->n + kJpegThreads - 1) / kJpegThreads, kJpegThreads, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_sync_kernel<<<a->nseg, kSyncThreads, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_write_kernel<<<static_cast<unsigned>((pl.chunk_slots + kJpegThreads - 1) / kJpegThreads), kJpegThreads, 0,
                      stream>>>(p, pl.chunk_slots);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_dc_kernel<<<a->nseg, kDcThreads, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_idct_kernel<<<dim3(static_cast<unsigned>((pl.max_blocks + kJpegThreads - 1) / kJpegThreads), a->n), kJpegThreads,
                     0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  jpeg_color_kernel<<<dim3((a->w + kJpegThreads - 1) / kJpegThreads, a->h, a->n), kJpegThreads, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

// PNG decoder for 8-bit and 1-bit grayscale files and 1/2/4/8-bit palette files (DESIGN.md §22, §24): the inverse of
// csrc/png.cu, and of any other encoder that stays inside the subset osvos_pytorch_b200/png.py parses (colour type 0 at
// depth 8 or 1, or, when the caller asks for indices, colour type 3 at depth 1, 2, 4 or 8; no interlace).
//
// The host walks the chunks, checks the CRCs, concatenates the IDAT payloads into one zlib stream per file and PROPOSES
// cuts of that stream: positions just after an IDAT payload that ends in 00 00 FF FF, where a full flush would leave the
// stream on a byte boundary with no match reaching back.  The blob (png.pack) is
//   PngBlobHeader | PngBlobFile[n] | PngBlobSegment[nseg] | the streams,
// every table 16-byte aligned, all files of one size h x w.  Segment k of a file covers the stream bytes [beg, end):
// segment 0 begins after the 2-byte zlib header, the last one ends with the 4 Adler-32 bytes.
//
// Kernels, in stream order:
//   png_validate_kernel  one thread per file: the tables against (n, h, w) and the blob's size -> status 0 or 32;
//   png_count_kernel     one warp per segment of a file with several: inflates WITHOUT writing and records the output
//                        length and whether the segment is `clean`: no error, every distance inside the segment's own
//                        output, and the read position exactly on the segment's end at a block boundary (the last one:
//                        BFINAL seen and exactly the four Adler-32 bytes left).  Segment 0 starts at the true start of
//                        the stream, so segment 0 clean proves cut 1 is a block boundary, and so on: all segments clean
//                        and lengths adding up to h * (rowbytes + 1) PROVES the proposed cuts; nothing is assumed;
//   png_segment_kernel   one warp per segment: when the file's cuts are proven, inflates again, writing at the summed
//                        offset into the file's filtered buffer;
//   png_serial_kernel    one warp per file: files with one segment, and files whose cuts were not proven, in order;
//   png_adler_kernel     partial Adler-32 sums of 16 KiB slices of the filtered bytes;
//   png_unfilter_kernel  one CTA per file: combines the slices and compares with the trailer, then undoes the row
//                        filters in place, rows in order: runs of Sub rows one warp per row (prefix sum), runs of Up
//                        rows one thread per column, runs of Average / Paeth rows as a skewed wavefront in one warp
//                        (lane j on row r + j, one pixel behind lane j - 1, the row above handed down by shuffle);
//   png_expand_kernel    the rows without their type bytes into out; gray depth 1 expanded to 0 / 255, palette
//                        samples unpacked MSB first to their raw index.
// Inflate is one warp per stream with every lane running the same control flow on the same bits: the Huffman tables are
// built by the warp in shared memory (canonical codes, a first-level lookup plus the per-length counts for longer
// codes), lane 0 writes literals and all lanes copy matches.  Every read is bounded by the segment's end and every
// write by the counted (or expected) length; a corrupt file gets status bits, never an out-of-range access.
#include "common.cuh"

namespace osvos {

constexpr uint32_t kPngBlobMagic = 0x31474E50u;   // "PNG1"
constexpr int kPngStatusCode = 1, kPngStatusDistance = 2, kPngStatusShort = 4, kPngStatusAdler = 8,
              kPngStatusFilter = 16, kPngStatusHeader = 32;
constexpr uint32_t kAdlerModulus = 65521u;
constexpr int kAdlerSlice = 16384;
constexpr int kInflateWarps = 4;
constexpr int kLitFast = 10, kDistFast = 8;
constexpr int kUnfilterThreads = 256;

struct PngBlobHeader {
  int32_t magic, n, nseg, h, w, pad[3];
  int64_t files_off, segs_off, data_off, data_bytes;
};
struct PngBlobFile {
  int32_t h, w, depth, seg0, nseg, colour, pad[2];   // colour: PNG colour type, 0 (grayscale) or 3 (palette)
  int64_t stream_off, stream_len;    // the zlib stream (header, deflate data, Adler-32) inside the data area
};
struct PngBlobSegment {
  int64_t beg, end;                  // inside the data area
  int32_t file, index;
};
static_assert(sizeof(PngBlobHeader) == 64 && sizeof(PngBlobFile) == 48 && sizeof(PngBlobSegment) == 24, "blob layout");

struct PngDecodeParams {
  const uint8_t* blob;
  size_t blob_bytes;
  uint8_t* out;
  int32_t* status;
  int32_t* path;        // or nullptr
  uint8_t* filt;        // [n][fstride]
  int32_t* seg_len;     // [nseg]
  int32_t* seg_clean;   // [nseg]
  int64_t* trailer;     // [n] position of the Adler-32 bytes in the data area
  uint32_t* adler;      // [n][nslice][2]
  size_t fstride;
  int n, h, w, nseg, nslice;
};

struct PngLayout {
  const PngBlobFile* files;
  const PngBlobSegment* segs;
  const uint8_t* data;
  int64_t data_bytes;
  bool ok;
};

__device__ PngLayout png_layout(const PngDecodeParams& p) {
  const PngBlobHeader* hd = reinterpret_cast<const PngBlobHeader*>(p.blob);
  const int64_t total = static_cast<int64_t>(p.blob_bytes);
  PngLayout l{};
  l.ok = static_cast<uint32_t>(hd->magic) == kPngBlobMagic && hd->n == p.n && hd->nseg == p.nseg && hd->h == p.h &&
         hd->w == p.w && hd->files_off >= static_cast<int64_t>(sizeof(PngBlobHeader)) && hd->files_off <= total &&
         (hd->files_off & 15) == 0 && hd->files_off + static_cast<int64_t>(p.n) * sizeof(PngBlobFile) <= total &&
         hd->segs_off >= 0 && hd->segs_off <= total && (hd->segs_off & 15) == 0 &&
         hd->segs_off + static_cast<int64_t>(p.nseg) * sizeof(PngBlobSegment) <= total && hd->data_off >= 0 &&
         hd->data_off <= total && hd->data_bytes >= 0 && hd->data_bytes <= total - hd->data_off;
  if (!l.ok) return l;
  l.files = reinterpret_cast<const PngBlobFile*>(p.blob + hd->files_off);
  l.segs = reinterpret_cast<const PngBlobSegment*>(p.blob + hd->segs_off);
  l.data = p.blob + hd->data_off;
  l.data_bytes = hd->data_bytes;
  return l;
}

__device__ __forceinline__ int png_row_bytes(int depth, int w) { return (w * depth + 7) >> 3; }

// grayscale at depth 8 or 1, palette at depth 1, 2, 4 or 8
__device__ __forceinline__ bool png_format_ok(int colour, int depth) {
  return colour == 0 ? (depth == 8 || depth == 1) : colour == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8);
}

// ---- validate -------------------------------------------------------------------------------------------------------

__global__ void png_validate_kernel(PngDecodeParams p) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= p.n) return;
  if (p.path) p.path[f] = 0;
  const PngLayout l = png_layout(p);
  bool ok = l.ok;
  if (ok) {
    const PngBlobFile F = l.files[f];
    const int64_t prev_end = f == 0 ? 0 : static_cast<int64_t>(l.files[f - 1].seg0) + l.files[f - 1].nseg;
    ok = F.h == p.h && F.w == p.w && png_format_ok(F.colour, F.depth) && F.nseg >= 1 && F.seg0 >= 0 &&
         F.seg0 == prev_end && static_cast<int64_t>(F.seg0) + F.nseg <= p.nseg &&
         (f + 1 < p.n || static_cast<int64_t>(F.seg0) + F.nseg == p.nseg) && F.stream_off >= 0 && F.stream_len >= 6 &&
         F.stream_off <= l.data_bytes && F.stream_len <= l.data_bytes - F.stream_off;
    if (ok) {
      int64_t at = F.stream_off + 2;
      for (int k = 0; k < F.nseg && ok; ++k) {
        const PngBlobSegment s = l.segs[F.seg0 + k];
        ok = s.file == f && s.index == k && s.beg == at && s.end >= s.beg && s.end <= F.stream_off + F.stream_len;
        at = s.end;
      }
      ok = ok && at == F.stream_off + F.stream_len;
    }
  }
  p.status[f] = ok ? 0 : kPngStatusHeader;
}

// Segment g of a validated blob: its file, index and byte range; false when its file is not to be decoded.
__device__ bool png_segment(const PngDecodeParams& p, const PngLayout& l, int g, int& f, PngBlobFile& F,
                            PngBlobSegment& s) {
  if (!l.ok || g >= p.nseg) return false;
  s = l.segs[g];
  f = s.file;
  if (f < 0 || f >= p.n || p.status[f] != 0) return false;
  F = l.files[f];
  return g >= F.seg0 && g - F.seg0 < F.nseg && s.index == g - F.seg0;
}

// ---- inflate --------------------------------------------------------------------------------------------------------

__constant__ uint16_t kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83,
                                      99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5,
                                      5, 0};
__constant__ uint16_t kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                       1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
                                       12, 12, 13, 13};
__constant__ uint8_t kCodeLengthOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// A canonical Huffman code: codes of <= FAST bits by lookup ((length << 9) | symbol, 0: longer or undefined), the rest
// by the per-length counts over the symbols sorted by (length, symbol).
template <int FAST, int NSYM>
struct HuffTable {
  uint16_t fast[1 << FAST];
  uint16_t sym[NSYM];
  int count[16];
  int offs[16], first[16], run[16];
  int bad;
};

struct WarpScratch {
  HuffTable<kLitFast, 288> lit;
  HuffTable<kDistFast, 32> dist;    // also the code-length code while a dynamic header is read
  uint8_t lens[320];
};

// LSB-first bit reader over data[pos, end); bits past the end read as zero and set `over`.
struct BitReader {
  const uint8_t* data;
  long long pos, end;
  uint64_t buf;
  int cnt;
  bool over;
  __device__ __forceinline__ void refill() {
    while (cnt <= 56 && pos < end) {
      buf |= static_cast<uint64_t>(__ldg(data + pos)) << cnt;
      ++pos;
      cnt += 8;
    }
  }
  __device__ __forceinline__ void drop(int n) {
    if (n > cnt) {
      over = true;
      buf = 0;
      cnt = 0;
    } else {
      buf >>= n;
      cnt -= n;
    }
  }
  __device__ __forceinline__ uint32_t take(int n) {
    const uint32_t v = static_cast<uint32_t>(buf) & ((1u << n) - 1u);
    drop(n);
    return v;
  }
  __device__ __forceinline__ long long consumed_bits() const { return pos * 8 - cnt; }
};

// Builds the table of lens[0..n) with the whole warp; false for an over-subscribed code, or an incomplete one that is
// not a single one-bit code (zlib's rule).  Ends with the warp synchronised.
template <int FAST, int NSYM>
__device__ bool build_table(HuffTable<FAST, NSYM>& t, const uint8_t* lens, int n) {
  const int lane = threadIdx.x & 31;
  __syncwarp();
  if (lane < 16) t.count[lane] = 0;
  __syncwarp();
  for (int s = lane; s < n; s += 32) atomicAdd(&t.count[lens[s]], 1);
  __syncwarp();
  if (lane == 0) {
    int left = 1, code = 0, at = 0, maxlen = 0;
    bool bad = false;
    t.count[0] = 0;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - t.count[l];
      bad = bad || left < 0;
      code = (code + t.count[l - 1]) << 1;
      t.first[l] = code;
      t.offs[l] = t.run[l] = at;
      at += t.count[l];
      if (t.count[l]) maxlen = l;
    }
    t.offs[0] = at;                               // the number of used symbols
    t.bad = bad || (left > 0 && maxlen > 1);
  }
  for (int k = lane; k < (1 << FAST); k += 32) t.fast[k] = 0;
  __syncwarp();
  const bool bad = t.bad;
  if (bad) return false;
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const int l = s < n ? lens[s] : 0;
    const unsigned same = __match_any_sync(0xffffffffu, l);
    if (l) t.sym[t.run[l] + __popc(same & ((1u << lane) - 1u))] = static_cast<uint16_t>(s);
    __syncwarp();
    if (l && (same & ((1u << lane) - 1u)) == 0) t.run[l] += __popc(same);
    __syncwarp();
  }
  const int used = t.offs[0];
  for (int i = lane; i < used; i += 32) {
    const int s = t.sym[i], l = lens[s];
    if (l <= FAST) {
      const uint32_t code = static_cast<uint32_t>(t.first[l] + (i - t.offs[l]));
      const uint32_t rev = __brev(code) >> (32 - l);
      for (uint32_t k = rev; k < (1u << FAST); k += 1u << l) t.fast[k] = static_cast<uint16_t>((l << 9) | s);
    }
  }
  __syncwarp();
  return true;
}

// The next symbol, or -1 for a bit pattern no code has.
template <int FAST, int NSYM>
__device__ __forceinline__ int decode_symbol(const HuffTable<FAST, NSYM>& t, BitReader& b) {
  const uint32_t e = t.fast[static_cast<uint32_t>(b.buf) & ((1u << FAST) - 1u)];
  if (e) {
    b.drop(e >> 9);
    return e & 511;
  }
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= static_cast<int>((b.buf >> (l - 1)) & 1u);
    const int c = t.count[l];
    if (code - c < first) {
      b.drop(l);
      return t.sym[index + (code - first)];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

struct InflateResult {
  int err;                  // kPngStatusCode | kPngStatusDistance | kPngStatusShort, or 0
  int len;                  // bytes produced
  bool final;               // stopped after a BFINAL block
  bool at_end;              // stopped at a block boundary with the read position exactly on `end`
  long long aligned_end;    // the next whole byte after the last block
};

// Raw deflate from data[beg, end) by one warp.  WRITE: the output goes to out[0, limit); otherwise it is only counted
// (and may not pass limit either).  stop_at_end: also stop at a block boundary that lies exactly on `end`.
template <bool WRITE>
__device__ InflateResult inflate_warp(const uint8_t* data, long long beg, long long end, uint8_t* out, int limit,
                                      bool stop_at_end, WarpScratch& S) {
  const int lane = threadIdx.x & 31;
  BitReader b{data, beg, end, 0, 0, false};
  InflateResult r{0, 0, false, false, beg};
  int outpos = 0, err = 0;
  for (;;) {
    b.refill();
    const uint32_t hdr = b.take(3);
    if (b.over) { err = kPngStatusShort; break; }
    r.final = hdr & 1;
    const int type = hdr >> 1;
    if (type == 0) {
      b.drop(b.cnt & 7);
      b.refill();
      const uint32_t len = b.take(16), nlen = b.take(16);
      if (b.over) { err = kPngStatusShort; break; }
      if ((len ^ 0xFFFFu) != nlen) { err = kPngStatusCode; break; }
      b.pos -= b.cnt >> 3;                        // hand the buffered whole bytes back
      b.buf = 0;
      b.cnt = 0;
      if (b.pos + len > end || outpos + static_cast<int>(len) > limit) { err = kPngStatusShort; break; }
      if (WRITE)
        for (uint32_t i = lane; i < len; i += 32) out[outpos + i] = __ldg(data + b.pos + i);
      b.pos += len;
      outpos += len;
    } else if (type == 1 || type == 2) {
      if (type == 1) {
        __syncwarp();
        for (int s = lane; s < 320; s += 32) S.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
        __syncwarp();
        build_table(S.lit, S.lens, 288);
        build_table(S.dist, S.lens + 288, 32);       // 30 and 31 complete the code and are refused when met
      } else {
        b.refill();
        const int hlit = b.take(5) + 257, hdist = b.take(5) + 1, hclen = b.take(4) + 4;
        if (b.over) { err = kPngStatusShort; break; }
        if (hlit > 286 || hdist > 30) { err = kPngStatusCode; break; }
        __syncwarp();
        if (lane < 19) S.lens[lane] = 0;
        __syncwarp();
        for (int k = 0; k < hclen; ++k) {
          b.refill();
          const uint32_t v = b.take(3);
          if (lane == 0) S.lens[kCodeLengthOrder[k]] = static_cast<uint8_t>(v);
        }
        if (b.over) { err = kPngStatusShort; break; }
        if (!build_table(S.dist, S.lens, 19)) { err = kPngStatusCode; break; }
        const int total = hlit + hdist;
        int idx = 0, prev = 0;
        while (idx < total && !err) {
          b.refill();
          const int sym = decode_symbol(S.dist, b);
          int rep = 1, val = sym;
          if (sym < 0 || sym > 18) {
            err = kPngStatusCode;
          } else if (sym == 16) {
            if (idx == 0) err = kPngStatusCode;
            rep = 3 + b.take(2);
            val = prev;
          } else if (sym == 17) {
            rep = 3 + b.take(3);
            val = 0;
          } else if (sym == 18) {
            rep = 11 + b.take(7);
            val = 0;
          }
          if (b.over) err = kPngStatusShort;
          if (!err && idx + rep > total) err = kPngStatusCode;
          if (err) break;
          __syncwarp();
          if (lane < rep) S.lens[idx + lane] = static_cast<uint8_t>(val);
          if (lane + 32 < rep) S.lens[idx + lane + 32] = static_cast<uint8_t>(val);
          if (lane + 64 < rep) S.lens[idx + lane + 64] = static_cast<uint8_t>(val);
          if (lane + 96 < rep) S.lens[idx + lane + 96] = static_cast<uint8_t>(val);
          if (lane + 128 < rep) S.lens[idx + lane + 128] = static_cast<uint8_t>(val);
          idx += rep;
          prev = val;
        }
        if (err) break;
        __syncwarp();
        if (S.lens[256] == 0) { err = kPngStatusCode; break; }
        // the distance lengths sit behind the literal lengths: build that table first, it does not overwrite them
        if (!build_table(S.lit, S.lens, hlit) || !build_table(S.dist, S.lens + hlit, hdist)) {
          err = kPngStatusCode;
          break;
        }
      }
      for (;;) {
        b.refill();
        int sym = decode_symbol(S.lit, b);
        if (b.over) { err = kPngStatusShort; break; }
        if (sym < 0) { err = kPngStatusCode; break; }
        if (sym < 256) {
          if (outpos >= limit) { err = kPngStatusShort; break; }
          if (WRITE && lane == 0) out[outpos] = static_cast<uint8_t>(sym);
          ++outpos;
          continue;
        }
        if (sym == 256) break;
        sym -= 257;
        if (sym >= 29) { err = kPngStatusCode; break; }
        const int len = kLenBase[sym] + b.take(kLenExtra[sym]);
        const int ds = decode_symbol(S.dist, b);
        if (b.over) { err = kPngStatusShort; break; }
        if (ds < 0 || ds >= 30) { err = kPngStatusCode; break; }
        const int dist = kDistBase[ds] + b.take(kDistExtra[ds]);
        if (b.over) { err = kPngStatusShort; break; }
        if (dist > outpos) { err = kPngStatusDistance; break; }
        if (len > limit - outpos) { err = kPngStatusShort; break; }
        if (WRITE) {
          // every source byte lies before outpos: written earlier by lanes of this warp
          __syncwarp();
          const uint8_t* src = out + outpos - dist;
          if (dist >= len) {
            for (int i = lane; i < len; i += 32) out[outpos + i] = src[i];
          } else {
            for (int i = lane; i < len; i += 32) out[outpos + i] = src[i % dist];
          }
          __syncwarp();
        }
        outpos += len;
      }
      if (err) break;
    } else {
      err = kPngStatusCode;
      break;
    }
    if (r.final) break;
    if (stop_at_end && b.consumed_bits() == end * 8) {
      r.at_end = true;
      break;
    }
  }
  r.err = err;
  r.len = outpos;
  r.aligned_end = (b.consumed_bits() + 7) >> 3;
  if (WRITE) __syncwarp();
  return r;
}

// Whether the proposed cuts of file F are proven, and the output offset and length of its segment k.
__device__ bool png_cuts_proven(const PngDecodeParams& p, const PngBlobFile& F, int k, int& before, int& mine) {
  const int lane = threadIdx.x & 31;
  long long sum = 0, pre = 0;
  int clean = 1;
  for (int j = lane; j < F.nseg; j += 32) {
    const int len = p.seg_len[F.seg0 + j];
    clean &= p.seg_clean[F.seg0 + j];
    sum += len;
    if (j < k) pre += len;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    pre += __shfl_xor_sync(0xffffffffu, pre, o);
    clean &= __shfl_xor_sync(0xffffffffu, clean, o);
  }
  const long long expect = static_cast<long long>(F.h) * (png_row_bytes(F.depth, F.w) + 1);
  before = static_cast<int>(pre);
  mine = p.seg_len[F.seg0 + k];
  return clean && sum == expect;
}

__global__ void __launch_bounds__(32 * kInflateWarps) png_count_kernel(PngDecodeParams p) {
  __shared__ WarpScratch scratch[kInflateWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * kInflateWarps + warp;
  const PngLayout l = png_layout(p);
  int f;
  PngBlobFile F;
  PngBlobSegment s;
  if (!png_segment(p, l, g, f, F, s) || F.nseg == 1) return;
  const long long expect = static_cast<long long>(F.h) * (png_row_bytes(F.depth, F.w) + 1);
  const bool last = s.index == F.nseg - 1;
  const InflateResult r = inflate_warp<false>(l.data, s.beg, s.end, nullptr, static_cast<int>(expect), !last,
                                              scratch[warp]);
  const bool clean = r.err == 0 && (last ? (r.final && r.aligned_end + 4 == s.end) : (!r.final && r.at_end));
  if (lane == 0) {
    p.seg_len[g] = r.len;
    p.seg_clean[g] = clean;
  }
}

__global__ void __launch_bounds__(32 * kInflateWarps) png_segment_kernel(PngDecodeParams p) {
  __shared__ WarpScratch scratch[kInflateWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * kInflateWarps + warp;
  const PngLayout l = png_layout(p);
  int f;
  PngBlobFile F;
  PngBlobSegment s;
  if (!png_segment(p, l, g, f, F, s) || F.nseg == 1) return;
  int before, mine;
  if (!png_cuts_proven(p, F, s.index, before, mine)) return;
  const bool last = s.index == F.nseg - 1;
  const InflateResult r = inflate_warp<true>(l.data, s.beg, s.end, p.filt + static_cast<size_t>(f) * p.fstride + before,
                                             mine, !last, scratch[warp]);
  if (lane == 0) {
    if (r.err) atomicOr(p.status + f, r.err);
    if (s.index == 0 && p.path) p.path[f] = 1;
    if (last) p.trailer[f] = r.aligned_end;
  }
}

__global__ void __launch_bounds__(32 * kInflateWarps) png_serial_kernel(PngDecodeParams p) {
  __shared__ WarpScratch scratch[kInflateWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kInflateWarps + warp;
  const PngLayout l = png_layout(p);
  if (!l.ok || f >= p.n || p.status[f] != 0) return;
  const PngBlobFile F = l.files[f];
  int before, mine;
  if (F.nseg > 1 && png_cuts_proven(p, F, 0, before, mine)) return;
  const long long expect = static_cast<long long>(F.h) * (png_row_bytes(F.depth, F.w) + 1);
  const long long end = F.stream_off + F.stream_len;
  const InflateResult r = inflate_warp<true>(l.data, F.stream_off + 2, end, p.filt + static_cast<size_t>(f) * p.fstride,
                                             static_cast<int>(expect), false, scratch[warp]);
  if (lane == 0) {
    int st = r.err;
    if (!st && (r.len != expect || r.aligned_end + 4 > end)) st = kPngStatusShort;
    if (st) atomicOr(p.status + f, st);
    if (p.path) p.path[f] = 2;
    p.trailer[f] = r.aligned_end;
  }
}

// ---- Adler-32 -------------------------------------------------------------------------------------------------------

// Slice s of file f: (sum d_i, sum (L - i) d_i) modulo 65521 over its L bytes.
__global__ void __launch_bounds__(256) png_adler_kernel(PngDecodeParams p) {
  __shared__ unsigned long long red[2][8];
  const int slice = blockIdx.x, f = blockIdx.y, t = threadIdx.x;
  const PngLayout l = png_layout(p);
  if (!l.ok || p.status[f] != 0) return;
  const PngBlobFile F = l.files[f];
  const long long expect = static_cast<long long>(F.h) * (png_row_bytes(F.depth, F.w) + 1);
  const long long o = static_cast<long long>(slice) * kAdlerSlice;
  const int L = static_cast<int>(max(0ll, min(static_cast<long long>(kAdlerSlice), expect - o)));
  const uint8_t* d = p.filt + static_cast<size_t>(f) * p.fstride + o;
  unsigned long long a1 = 0, a2 = 0;
  for (int i = t; i < L; i += 256) {
    const unsigned v = d[i];
    a1 += v;
    a2 += static_cast<unsigned long long>(L - i) * v;
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    a1 += __shfl_xor_sync(0xffffffffu, a1, k);
    a2 += __shfl_xor_sync(0xffffffffu, a2, k);
  }
  if ((t & 31) == 0) { red[0][t >> 5] = a1; red[1][t >> 5] = a2; }
  __syncthreads();
  if (t == 0) {
    a1 = a2 = 0;
    for (int k = 0; k < 8; ++k) { a1 += red[0][k]; a2 += red[1][k]; }
    uint32_t* dst = p.adler + 2 * (static_cast<size_t>(f) * p.nslice + slice);
    dst[0] = static_cast<uint32_t>(a1 % kAdlerModulus);
    dst[1] = static_cast<uint32_t>(a2 % kAdlerModulus);
  }
}

// ---- unfilter -------------------------------------------------------------------------------------------------------

__device__ __forceinline__ int paeth_predictor(int a, int b, int c) {
  const int pp = a + b - c;
  const int pa = abs(pp - a), pb = abs(pp - b), pc = abs(pp - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__global__ void __launch_bounds__(kUnfilterThreads) png_unfilter_kernel(PngDecodeParams p) {
  __shared__ int verdict;
  const int f = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const PngLayout l = png_layout(p);
  if (!l.ok || p.status[f] != 0) return;
  const PngBlobFile F = l.files[f];
  const int rb = png_row_bytes(F.depth, F.w), stride = rb + 1, h = F.h;
  const long long expect = static_cast<long long>(h) * stride;
  uint8_t* fb = p.filt + static_cast<size_t>(f) * p.fstride;

  if (warp == 0) {
    unsigned long long s1 = 0, s2 = 0;
    const int used = static_cast<int>((expect + kAdlerSlice - 1) / kAdlerSlice);
    for (int k = lane; k < used; k += 32) {
      const uint32_t* a = p.adler + 2 * (static_cast<size_t>(f) * p.nslice + k);
      const long long o = static_cast<long long>(k) * kAdlerSlice;
      const long long L = min(static_cast<long long>(kAdlerSlice), expect - o);
      s1 += a[0];
      s2 += (a[1] + static_cast<unsigned long long>((expect - o - L) % kAdlerModulus) * a[0]) % kAdlerModulus;
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, k);
      s2 += __shfl_xor_sync(0xffffffffu, s2, k);
    }
    if (lane == 0) {
      s1 = (s1 + 1) % kAdlerModulus;
      s2 = (s2 + expect % kAdlerModulus) % kAdlerModulus;
      const uint8_t* tr = l.data + p.trailer[f];      // the inflate pass checked that four bytes follow
      const uint32_t want = (static_cast<uint32_t>(tr[0]) << 24) | (tr[1] << 16) | (tr[2] << 8) | tr[3];
      verdict = want == ((static_cast<uint32_t>(s2) << 16) | static_cast<uint32_t>(s1)) ? 0 : kPngStatusAdler;
      if (verdict) atomicOr(p.status + f, verdict);
    }
  }
  __syncthreads();
  if (verdict) return;

  int r = 0;
  while (r < h) {
    const int type = fb[static_cast<size_t>(r) * stride];
    if (type > 4) {
      if (t == 0) atomicOr(p.status + f, kPngStatusFilter);
      return;
    }
    // the run of rows handled the same way: [r, e)
    int e = r + 1;
    const bool serial = type >= 3;
    while (e < h) {
      const int te = fb[static_cast<size_t>(e) * stride];
      if (serial ? (te != 3 && te != 4) : te != type) break;
      ++e;
    }
    if (type == 0) {
      r = e;
      continue;
    }
    __syncthreads();                               // the row above is complete
    if (type == 1) {
      // inclusive prefix sum modulo 256 along each row, one warp per row, a contiguous piece per lane
      const int piece = (rb + 31) / 32;
      for (int y = r + warp; y < e; y += kUnfilterThreads / 32) {
        uint8_t* row = fb + static_cast<size_t>(y) * stride + 1;
        const int i0 = min(rb, lane * piece), i1 = min(rb, i0 + piece);
        unsigned sum = 0;
        for (int i = i0; i < i1; ++i) sum += row[i];
        unsigned incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned u = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += u;
        }
        unsigned acc = incl - sum;
        for (int i = i0; i < i1; ++i) {
          acc += row[i];
          row[i] = static_cast<uint8_t>(acc);
        }
      }
    } else if (type == 2) {
      for (int x = t; x < rb; x += kUnfilterThreads) {
        unsigned acc = r > 0 ? fb[static_cast<size_t>(r - 1) * stride + 1 + x] : 0;
        for (int y = r; y < e; ++y) {
          uint8_t* q = fb + static_cast<size_t>(y) * stride + 1 + x;
          acc += *q;
          *q = static_cast<uint8_t>(acc);
        }
      }
    } else if (warp == 0) {
      for (int g0 = r; g0 < e; g0 += 32) {
        const int m = min(32, e - g0), y = g0 + lane;
        const bool mine = lane < m;
        const int ty = mine ? fb[static_cast<size_t>(y) * stride] : 0;
        uint8_t* row = fb + static_cast<size_t>(mine ? y : g0) * stride + 1;
        const uint8_t* above = g0 > 0 ? fb + static_cast<size_t>(g0 - 1) * stride + 1 : nullptr;
        int a = 0, c = 0, x = 0;
        const int steps = rb + m - 1;
        for (int s = 0; s < steps; ++s) {
          const int i = s - lane;
          int b = __shfl_up_sync(0xffffffffu, x, 1);
          const bool on = mine && i >= 0 && i < rb;
          if (lane == 0) b = (above && on) ? above[i] : 0;
          if (on) {
            const int pred = ty == 3 ? ((a + b) >> 1) : paeth_predictor(a, b, c);
            x = (row[i] + pred) & 255;
            row[i] = static_cast<uint8_t>(x);
            a = x;
            c = b;
          }
        }
        __syncwarp();                              // the group's last row is the next group's row above
      }
    }
    r = e;
  }
}

__global__ void __launch_bounds__(256) png_expand_kernel(PngDecodeParams p) {
  const int f = blockIdx.y;
  const PngLayout l = png_layout(p);
  if (!l.ok || p.status[f] != 0) return;
  const int depth = l.files[f].depth;
  const bool gray = l.files[f].colour == 0;
  const int rb = png_row_bytes(depth, p.w), stride = rb + 1;
  const int per_byte_log2 = depth == 1 ? 3 : depth == 2 ? 2 : depth == 4 ? 1 : 0;
  const int mask = (1 << depth) - 1;
  const uint8_t* fb = p.filt + static_cast<size_t>(f) * p.fstride;
  uint8_t* out = p.out + static_cast<size_t>(f) * p.h * p.w;
  const long long total = static_cast<long long>(p.h) * p.w;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * 256) {
    const int y = static_cast<int>(i / p.w), x = static_cast<int>(i - static_cast<long long>(y) * p.w);
    const uint8_t* row = fb + static_cast<size_t>(y) * stride + 1;
    // samples MSB first; a palette sample is its index, a 1-bit gray sample 0 / 255
    const int shift = 8 - depth * ((x & ((1 << per_byte_log2) - 1)) + 1);
    const int v = (row[x >> per_byte_log2] >> shift) & mask;
    out[i] = static_cast<uint8_t>(gray && depth == 1 ? v * 255 : v);
  }
}

// ---- workspace ------------------------------------------------------------------------------------------------------

struct PngDecodePlan {
  size_t fstride, len_off, clean_off, trailer_off, adler_off, bytes;
  int nslice;
};

inline size_t png_decode_align16(size_t v) { return (v + 15) & ~static_cast<size_t>(15); }

PngDecodePlan png_decode_plan(int n, int h, int w, int nseg) {
  PngDecodePlan q{};
  const size_t filtered = static_cast<size_t>(h) * (w + 1);
  q.fstride = png_decode_align16(filtered);
  q.nslice = static_cast<int>((filtered + kAdlerSlice - 1) / kAdlerSlice);
  q.len_off = q.fstride * n;
  q.clean_off = q.len_off + png_decode_align16(sizeof(int32_t) * static_cast<size_t>(nseg));
  q.trailer_off = q.clean_off + png_decode_align16(sizeof(int32_t) * static_cast<size_t>(nseg));
  q.adler_off = q.trailer_off + png_decode_align16(sizeof(int64_t) * static_cast<size_t>(n));
  q.bytes = q.adler_off + png_decode_align16(2 * sizeof(uint32_t) * static_cast<size_t>(n) * q.nslice);
  return q;
}

}  // namespace osvos

using namespace osvos;

static bool png_decode_dims_ok(int n, int h, int w, int nseg, size_t blob_bytes) {
  return n > 0 && n < 65536 && h > 0 && w > 0 && h < 32768 && w < 32768 && nseg >= n && nseg < (1 << 30) &&
         blob_bytes >= sizeof(PngBlobHeader) && blob_bytes < (static_cast<size_t>(1) << 31);
}

extern "C" size_t osvos_png_decode_workspace_bytes(int n, int h, int w, int nseg, size_t blob_bytes) {
  if (!png_decode_dims_ok(n, h, w, nseg, blob_bytes)) return 0;
  return png_decode_plan(n, h, w, nseg).bytes;
}

extern "C" int osvos_png_decode(const osvos_png_decode_args* a, osvos_stream_t stream_) {
  OSVOS_CHECK_ARG(a != nullptr);
  OSVOS_CHECK_ARG(a->blob != nullptr && a->out != nullptr && a->status != nullptr && a->workspace != nullptr);
  OSVOS_CHECK_ARG(png_decode_dims_ok(a->n, a->h, a->w, a->nseg, a->blob_bytes));
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->blob) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0);
  OSVOS_CHECK_ARG((reinterpret_cast<uintptr_t>(a->status) & 3) == 0 && (reinterpret_cast<uintptr_t>(a->path) & 3) == 0);
  const PngDecodePlan q = png_decode_plan(a->n, a->h, a->w, a->nseg);
  uint8_t* ws = static_cast<uint8_t*>(a->workspace);
  PngDecodeParams p{};
  p.blob = static_cast<const uint8_t*>(a->blob);
  p.blob_bytes = a->blob_bytes;
  p.out = a->out;
  p.status = a->status;
  p.path = a->path;
  p.filt = ws;
  p.seg_len = reinterpret_cast<int32_t*>(ws + q.len_off);
  p.seg_clean = reinterpret_cast<int32_t*>(ws + q.clean_off);
  p.trailer = reinterpret_cast<int64_t*>(ws + q.trailer_off);
  p.adler = reinterpret_cast<uint32_t*>(ws + q.adler_off);
  p.fstride = q.fstride;
  p.n = a->n;
  p.h = a->h;
  p.w = a->w;
  p.nseg = a->nseg;
  p.nslice = q.nslice;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // segments of single-segment files are never counted: their slots read as "not clean"
  OSVOS_CHECK_CUDA(cudaMemsetAsync(ws + q.len_off, 0, q.trailer_off - q.len_off, stream));
  png_validate_kernel<<<(a->n + 127) / 128, 128, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  const unsigned seg_blocks = (a->nseg + kInflateWarps - 1) / kInflateWarps;
  if (a->nseg > a->n) {
    png_count_kernel<<<seg_blocks, 32 * kInflateWarps, 0, stream>>>(p);
    OSVOS_CHECK_CUDA(cudaGetLastError());
    png_segment_kernel<<<seg_blocks, 32 * kInflateWarps, 0, stream>>>(p);
    OSVOS_CHECK_CUDA(cudaGetLastError());
  }
  png_serial_kernel<<<(a->n + kInflateWarps - 1) / kInflateWarps, 32 * kInflateWarps, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  png_adler_kernel<<<dim3(q.nslice, a->n), 256, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  png_unfilter_kernel<<<a->n, kUnfilterThreads, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  const long long pixels = static_cast<long long>(a->h) * a->w;
  png_expand_kernel<<<dim3(static_cast<unsigned>(min(1024ll, (pixels + 2047) / 2048)), a->n), 256, 0, stream>>>(p);
  OSVOS_CHECK_CUDA(cudaGetLastError());
  return OSVOS_OK;
}

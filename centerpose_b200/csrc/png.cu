// cpb200_png_decode_batch: cv2.imread(path, IMREAD_COLOR) of PNG files on the device, byte for byte, for many files
// per launch.  Three kernels:
//   png_inflate_kernel   one warp per image: zlib header, then the deflate blocks (RFC 1951) into the filtered
//                        scanlines in the workspace.  Every lane holds the same bit reader and decodes the same
//                        symbols from Huffman tables in shared memory; lane 0 stores literals, the warp copies matches,
//   png_unfilter_kernel  one warp per image: lane l undoes the filter of row 32k + l one pixel behind lane l - 1, which
//                        hands it the row above through a shuffle; the lanes also sum the Adler-32 of what they read,
//   png_output_kernel    one thread per output pixel: Adam7 position, depth / palette expansion, BGR, and OpenCV's EXIF
//                        orientation as an index mapping.
// Inflate and unfilter are serial within an image, so the batch gives the parallelism.  The host side
// (centerpose_b200/png.py) parses the chunks and builds the table; the kernels trust it.
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_png_image) == 72, "cpb200_png_image layout is part of the C ABI");

constexpr int kLutBits = 10;
constexpr uint32_t kAdlerMod = 65521;

// Adam7: x start, y start, x step, y step of passes 1..7
__constant__ unsigned char kAdam7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8}, {2, 0, 4, 4},
                                           {0, 2, 2, 4}, {1, 0, 2, 2}, {0, 1, 1, 2}};
// pass (0-based) of the pixel at (y & 7, x & 7)
__constant__ unsigned char kAdam7Pass[8][8] = {
    {0, 5, 3, 5, 1, 5, 3, 5}, {6, 6, 6, 6, 6, 6, 6, 6}, {4, 5, 4, 5, 4, 5, 4, 5}, {6, 6, 6, 6, 6, 6, 6, 6},
    {2, 5, 3, 5, 2, 5, 3, 5}, {6, 6, 6, 6, 6, 6, 6, 6}, {4, 5, 4, 5, 4, 5, 4, 5}, {6, 6, 6, 6, 6, 6, 6, 6}};
// RFC 1951 3.2.5: base and extra bits of length symbols 257..285 and distance symbols 0..29
__constant__ unsigned short kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                            31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2,
                                            2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned short kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,    49,    65,    97,    129,
                                             193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ unsigned char kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6,
                                             6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ unsigned char kClenOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ int channels(int ct) { return ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1; }

// (width, height) of reduced image k (the whole image when not interlaced); either may be 0
__device__ __forceinline__ void pass_size(const cpb200_png_image &e, int k, int &pw, int &ph) {
  if (!e.interlace) {
    pw = e.w; ph = e.h;
    return;
  }
  const int x0 = kAdam7[k][0], y0 = kAdam7[k][1], dx = kAdam7[k][2], dy = kAdam7[k][3];
  pw = e.w > x0 ? (e.w - x0 + dx - 1) / dx : 0;
  ph = e.h > y0 ? (e.h - y0 + dy - 1) / dy : 0;
}

__device__ __forceinline__ int64_t row_bytes(const cpb200_png_image &e, int pw) {
  return ((int64_t)pw * channels(e.color_type) * e.depth + 7) >> 3;
}

// size of the inflated stream: per non-empty pass, rows of a filter byte and the packed samples
__device__ __forceinline__ int64_t filtered_bytes(const cpb200_png_image &e) {
  int64_t f = 0;
  for (int k = 0; k < (e.interlace ? 7 : 1); ++k) {
    int pw, ph;
    pass_size(e, k, pw, ph);
    if (pw && ph) f += (int64_t)ph * (1 + row_bytes(e, pw));
  }
  return f;
}

// the scanlines, rounded up to 16 bytes, and the stream's Adler-32 behind them lie inside the workspace
__device__ __forceinline__ bool fits(const cpb200_png_image &e, int64_t f, size_t ws_bytes) {
  return e.ws_offset >= 0 && e.ws_bytes >= ((f + 15) & ~15ll) + 16 && (uint64_t)e.ws_offset + e.ws_bytes <= ws_bytes;
}

// canonical Huffman code in shared memory: lut[b] for the next kLutBits bits b (LSB first) is (length << 9 | symbol),
// 0 when the code is longer or unused; longer codes are decoded bit by bit from count / sym (as zlib's puff.c)
struct Huff {
  unsigned short lut[1 << kLutBits];
  unsigned short count[16];
  unsigned short sym[288];
  unsigned short code[288];
  unsigned short offs[16], next[16];                     // build's scratch: per length, next slot in sym / next code
};

// LSB-first bit reader over one zlib stream, refilled with 8-byte loads (the stream is followed by 32 readable bytes).
// Every lane holds the same state.  `p` counts the bytes moved into `acc`, past `end` when the stream ran out
struct Bits {
  const unsigned char *s;
  int64_t p, end;
  uint64_t acc;
  int n;

  __device__ __forceinline__ void fill() {
    const uintptr_t a = reinterpret_cast<uintptr_t>(s + p);
    const uint64_t *w = reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7);
    const int sh = (int)(a & 7) * 8;
    uint64_t v = __ldg(w) >> sh;
    if (sh) v |= __ldg(w + 1) << (64 - sh);
    acc |= v << n;
    p += (63 - n) >> 3;
    n |= 56;
  }
  __device__ __forceinline__ void drop(int k) { acc >>= k; n -= k; }
  __device__ __forceinline__ uint32_t get(int k) {   // k <= 32
    if (n < k) fill();
    const uint32_t v = (uint32_t)(acc & ((1ull << k) - 1));
    drop(k);
    return v;
  }
  __device__ __forceinline__ bool overrun() const { return p > end + 8; }
  __device__ __forceinline__ int64_t consumed() const { return 8 * p - n; }
};

// the warp builds `h` from code lengths len[0..nsym); false where zlib's inflate_table refuses the lengths (and
// libpng with it): an over-subscribed code, or an incomplete one unless it is a single code of length 1 of a literal /
// length or distance code (`codes`: the code-length code, which may never be incomplete).  All lengths zero is
// accepted, as zlib does; decoding any symbol of that code then fails
__device__ bool build(Huff &h, const unsigned char *len, int nsym, int lane, bool codes = false) {
  if (lane < 16) {
    int c = 0;
    for (int s = 0; s < nsym; ++s) c += len[s] == lane;
    h.count[lane] = lane ? c : 0;
  }
  for (int i = lane; i < (1 << kLutBits); i += 32) h.lut[i] = 0;
  __syncwarp();
  int ok = 1;
  if (lane == 0) {
    int left = 1, longest = 0;
    unsigned short *offs = h.offs, *next = h.next;
    offs[1] = 0; next[1] = 0;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - h.count[l];
      if (left < 0) ok = 0;
      if (h.count[l]) longest = l;
      if (l < 15) {
        offs[l + 1] = offs[l] + h.count[l];
        next[l + 1] = (next[l] + h.count[l]) << 1;
      }
    }
    if (longest && left > 0 && (codes || longest != 1)) ok = 0;
    if (ok)
      for (int s = 0; s < nsym; ++s)
        if (len[s]) {
          h.sym[offs[len[s]]++] = (unsigned short)s;
          h.code[s] = next[len[s]]++;
        }
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  __syncwarp();
  if (!ok) return false;
  for (int s = lane; s < nsym; s += 32) {
    const int l = len[s];
    if (l && l <= kLutBits) {
      const unsigned rev = __brev(h.code[s]) >> (32 - l);
      for (unsigned k = rev; k < (1u << kLutBits); k += 1u << l) h.lut[k] = (unsigned short)(l << 9 | s);
    }
  }
  __syncwarp();
  return true;
}

// next symbol of `h` (the reader holds >= 15 bits), -1 for an unused code
__device__ __forceinline__ int decode(Bits &r, const Huff &h) {
  const unsigned e = h.lut[r.acc & ((1u << kLutBits) - 1)];
  if (e) {
    r.drop(e >> 9);
    return e & 511;
  }
  int code = 0, first = 0, index = 0;
  uint64_t a = r.acc;
  for (int l = 1; l < 16; ++l) {
    code |= (int)(a & 1);
    a >>= 1;
    const int count = h.count[l];
    if (code - count < first) {
      r.drop(l);
      return h.sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// grid B CTAs x 32 threads: CTA b inflates image b's stream into its workspace and stores the stream's Adler-32 after
// the scanlines; status 1 for a bad stream, 2 when the workspace does not fit
__global__ void __launch_bounds__(32) png_inflate_kernel(const unsigned char *__restrict__ src,
                                                         const cpb200_png_image *__restrict__ table,
                                                         unsigned char *__restrict__ ws, size_t ws_bytes,
                                                         int *__restrict__ status) {
  __shared__ Huff lit, dist;
  __shared__ unsigned char lens[320];
  const cpb200_png_image &e = table[blockIdx.x];
  const int lane = threadIdx.x;
  const int64_t total = filtered_bytes(e);
  if (!fits(e, total, ws_bytes)) {
    if (lane == 0) status[blockIdx.x] = 2;
    return;
  }
  unsigned char *out = ws + e.ws_offset;
  Bits r{src + e.src_offset, 0, e.src_bytes, 0ull, 0};
  int64_t pos = 0;
  int fixed = 0;                                           // the tables hold the fixed code
  int window;                                              // CINFO's window: libpng's zlib refuses farther distances
  r.fill();
  {
    const uint32_t cmf = r.get(8), flg = r.get(8);
    // deflate, window <= 32K, no preset dictionary, header check
    if ((cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 32) || (cmf * 256 + flg) % 31) goto bad;
    window = 1 << ((cmf >> 4) + 8);
  }
  for (int final = 0; !final;) {
    r.fill();
    if (r.overrun()) goto bad;
    final = (int)r.get(1);
    const int type = (int)r.get(2);
    if (type == 0) {                                       // stored
      r.drop(r.n & 7);
      const uint32_t len = r.get(16), nlen = r.get(16);
      if ((len ^ 0xFFFF) != nlen) goto bad;
      const int64_t q = r.p - r.n / 8;                     // the block's first byte
      if (q + len > r.end || pos + len > total) goto bad;
      for (uint32_t i = lane; i < len; i += 32) out[pos + i] = r.s[q + i];
      pos += len;
      r.p = q + len; r.acc = 0; r.n = 0;
      __syncwarp();
      continue;
    }
    if (type == 3) goto bad;
    if (type == 1) {
      if (!fixed) {
        for (int s = lane; s < 320; s += 32) lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
        __syncwarp();
        build(lit, lens, 288, lane);
        build(dist, lens + 288, 32, lane);   // 30 and 31 are coded but invalid, as in zlib
        fixed = 1;
      }
    } else {
      fixed = 0;
      const int hlit = (int)r.get(5) + 257, hdist = (int)r.get(5) + 1, hclen = (int)r.get(4) + 4;
      if (hlit > 286 || hdist > 30) goto bad;
      for (int i = lane; i < 19; i += 32) lens[kClenOrder[i]] = 0;
      __syncwarp();
      for (int i = 0; i < hclen; ++i) {
        const unsigned v = r.get(3);
        if (lane == 0) lens[kClenOrder[i]] = (unsigned char)v;
      }
      __syncwarp();
      if (!build(lit, lens, 19, lane, true)) goto bad;
      // code lengths: literal / length ones at lens[0..hlit), distance ones at lens[288..288 + hdist)
      for (int i = 0; i < hlit + hdist;) {
        r.fill();
        if (r.overrun()) goto bad;
        const int sym = decode(r, lit);
        if (sym < 0) goto bad;
        int rep, v;
        if (sym < 16) {
          rep = 1; v = sym;
        } else if (sym == 16) {
          if (i == 0) goto bad;
          __syncwarp();
          v = lens[i - 1 < hlit ? i - 1 : i - 1 - hlit + 288]; rep = 3 + (int)r.get(2);
        } else {
          v = 0; rep = sym == 17 ? 3 + (int)r.get(3) : 11 + (int)r.get(7);
        }
        if (i + rep > hlit + hdist) goto bad;
        if (lane == 0)
          for (int k = i; k < i + rep; ++k) lens[k < hlit ? k : k - hlit + 288] = (unsigned char)v;
        i += rep;
      }
      __syncwarp();
      if (lens[256] == 0) goto bad;                        // no end-of-block code
      if (!build(lit, lens, hlit, lane) || !build(dist, lens + 288, hdist, lane)) goto bad;
    }
    for (;;) {                                             // the block's symbols
      if (r.n < 48) {
        r.fill();
        if (r.overrun()) goto bad;
      }
      const int sym = decode(r, lit);
      if (sym < 256) {
        if (sym < 0 || pos >= total) goto bad;
        if (lane == 0) out[pos] = (unsigned char)sym;
        ++pos;
        continue;
      }
      if (sym == 256) break;
      if (sym > 285) goto bad;
      const int li = sym - 257;
      const int len = kLenBase[li] + (int)(r.acc & ((1u << kLenExtra[li]) - 1));
      r.drop(kLenExtra[li]);
      const int ds = decode(r, dist);
      if (ds < 0 || ds > 29) goto bad;
      const int d = kDistBase[ds] + (int)(r.acc & ((1u << kDistExtra[ds]) - 1));
      r.drop(kDistExtra[ds]);
      if (d > pos || d > window || pos + len > total) goto bad;
      __syncwarp();                                        // lane 0's literals are visible to the copy
      unsigned char *o = out + pos;
      if (d >= len) {
        if (lane < len) o[lane] = o[lane - d];
        for (int j = lane + 32; j < len; j += 32) o[j] = o[j - d];
      } else {
        // an overlapping copy repeats the last d bytes: o[j] = o[j mod d - d]
        for (int j = lane; j < len; j += 32) o[j] = o[j % d - d];
      }
      __syncwarp();
      pos += len;
    }
  }
  {
    r.drop(r.n & 7);
    uint32_t adler = 0;
    for (int k = 0; k < 4; ++k) adler = adler << 8 | r.get(8);
    if (pos != total || r.consumed() > 8 * r.end) goto bad;
    if (lane == 0) {
      *reinterpret_cast<uint32_t *>(out + ((total + 15) & ~15ll)) = adler;
      status[blockIdx.x] = 0;
    }
    return;
  }
bad:
  if (lane == 0) status[blockIdx.x] = 1;
}

__device__ __forceinline__ unsigned byte_of(uint32_t lo, uint32_t hi, int k) {
  return ((k < 4 ? lo : hi) >> (8 * (k & 3))) & 255;
}

// PNG spec 9.4 predictor
__device__ __forceinline__ unsigned paeth(unsigned a, unsigned b, unsigned c) {
  const int p = (int)a + (int)b - (int)c;
  const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
  return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

// grid B CTAs x 32 threads: CTA b undoes image b's filters in place, pass by pass, 32 rows at a time.  Lane l takes row
// 32k + l and at step t its filter unit (pixel, or byte below 8 bits per pixel) t - l: the unit above is the one lane
// l - 1 finished at step t - 1, handed over by a shuffle (lane 0 reads it from memory).  Each lane also sums, over the
// bytes it reads, the two Adler-32 sums, which the warp reduces and compares with the stream's; status 1 on a
// mismatch or a filter type above 4.  Images whose inflate failed are skipped.
__global__ void __launch_bounds__(32) png_unfilter_kernel(const cpb200_png_image *__restrict__ table,
                                                          unsigned char *__restrict__ ws, int *__restrict__ status) {
  const cpb200_png_image &e = table[blockIdx.x];
  if (status[blockIdx.x]) return;
  const int lane = threadIdx.x;
  unsigned char *img = ws + e.ws_offset;
  const int bits = channels(e.color_type) * e.depth;
  const int bpp = bits >= 8 ? bits >> 3 : 1;
  uint64_t s1 = 0, s2 = 0;                                 // sum of bytes; sum of (index mod 65521) * byte, mod 65521
  int bad = 0;
  int64_t base = 0;
  for (int k = 0; k < (e.interlace ? 7 : 1); ++k) {
    int pw, ph;
    pass_size(e, k, pw, ph);
    if (!pw || !ph) continue;
    const int64_t rb = row_bytes(e, pw), units = rb / bpp;
    for (int g = 0; g < ph; g += 32) {
      const int y = g + lane;
      const bool active = y < ph;
      unsigned char *row = img + base + (int64_t)y * (rb + 1);
      const unsigned char *above = y ? row - (rb + 1) + 1 : nullptr;   // lane 0 reads the row above from memory
      const int ft = active ? row[0] : 0;
      if (ft > 4) bad = 1;
      uint64_t rs1 = ft, rs2 = 0;                          // this row's sums; rs2 weights by the index in the row
      uint32_t alo = 0, ahi = 0, clo = 0, chi = 0, ulo = 0, uhi = 0;   // left, up-left, own last unit
      const int64_t steps = units + min(32, ph - g) - 1;
      for (int64_t t = 0; t < steps; ++t) {
        const uint32_t blo = __shfl_up_sync(0xffffffffu, ulo, 1), bhi = __shfl_up_sync(0xffffffffu, uhi, 1);
        const int64_t x = t - lane;
        if (active && x >= 0 && x < units) {
          unsigned char *px = row + 1 + x * bpp;
          uint32_t nlo = 0, nhi = 0, ulo2 = blo, uhi2 = bhi;
          if (lane == 0) {
            ulo2 = uhi2 = 0;
            if (above)
#pragma unroll
              for (int c = 0; c < 8; ++c)
                if (c < bpp) (c < 4 ? ulo2 : uhi2) |= (uint32_t)above[x * bpp + c] << (8 * (c & 3));
          }
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            if (c < bpp) {
              const unsigned f = px[c];
              rs1 += f;
              rs2 += (uint64_t)(1 + x * bpp + c) * f;
              const unsigned a = byte_of(alo, ahi, c), b = byte_of(ulo2, uhi2, c), cc = byte_of(clo, chi, c);
              unsigned v = f;
              if (ft == 1) v = f + a;
              else if (ft == 2) v = f + b;
              else if (ft == 3) v = f + ((a + b) >> 1);
              else if (ft == 4) v = f + paeth(a, b, cc);
              v &= 255;
              px[c] = (unsigned char)v;
              (c < 4 ? nlo : nhi) |= v << (8 * (c & 3));
            }
          }
          alo = nlo; ahi = nhi; clo = ulo2; chi = uhi2; ulo = nlo; uhi = nhi;
        }
        __syncwarp();
      }
      if (active) {
        const uint64_t start = (uint64_t)(base + (int64_t)y * (rb + 1)) % kAdlerMod;
        s1 += rs1;
        s2 = (s2 + start * (rs1 % kAdlerMod) + rs2 % kAdlerMod) % kAdlerMod;
      }
      __syncwarp();
    }
    base += (int64_t)ph * (rb + 1);
  }
  for (int o = 16; o; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 = (s2 + __shfl_xor_sync(0xffffffffu, s2, o)) % kAdlerMod;
  }
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) {
    // a = 1 + sum d_i, b = N + sum (N - i) d_i over the N bytes (RFC 1950 8.2)
    const uint64_t n = (uint64_t)base % kAdlerMod, a = (1 + s1) % kAdlerMod;
    const uint64_t b = (n + n * (s1 % kAdlerMod) + kAdlerMod - s2) % kAdlerMod;
    const uint32_t want = *reinterpret_cast<const uint32_t *>(img + ((base + 15) & ~15ll));
    if (bad || want != (uint32_t)(b << 16 | a)) status[blockIdx.x] = 1;
  }
}

// grid (pixel blocks, image) x 256 threads: one thread per output pixel in row-major order of the oriented image
__global__ void __launch_bounds__(256) png_output_kernel(const unsigned char *__restrict__ src,
                                                         const cpb200_png_image *__restrict__ table,
                                                         const unsigned char *__restrict__ ws,
                                                         const int *__restrict__ status, unsigned char *__restrict__ dst) {
  __shared__ int64_t pbase[7], prb[7];
  const cpb200_png_image &e = table[blockIdx.y];
  if (status[blockIdx.y]) return;
  if (threadIdx.x == 0) {
    int64_t base = 0;
    for (int k = 0; k < 7; ++k) {
      int pw = 0, ph = 0;
      if (k == 0 || e.interlace) pass_size(e, k, pw, ph);
      pbase[k] = base;
      prb[k] = row_bytes(e, pw);
      if (pw && ph) base += (int64_t)ph * (prb[k] + 1);
    }
  }
  __syncthreads();
  const int h = e.h, w = e.w, o = e.orientation, ct = e.color_type, depth = e.depth;
  const int ow = o >= 5 ? h : w;
  const int64_t total = (int64_t)h * w;
  const unsigned char *img = ws + e.ws_offset;
  const unsigned char *pal = src + e.palette_offset;
  const int ch = channels(ct), sb = depth == 16 ? 2 : 1;
  unsigned char *out = dst + e.dst_offset;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i - (int64_t)oy * ow);
    // cv2's ApplyExifOrientation: transpose for 5..8, then flips
    int sy, sx;
    switch (o) {
      case 2: sy = oy; sx = w - 1 - ox; break;
      case 3: sy = h - 1 - oy; sx = w - 1 - ox; break;
      case 4: sy = h - 1 - oy; sx = ox; break;
      case 5: sy = ox; sx = oy; break;
      case 6: sy = h - 1 - ox; sx = oy; break;
      case 7: sy = h - 1 - ox; sx = w - 1 - oy; break;
      case 8: sy = ox; sx = w - 1 - oy; break;
      default: sy = oy; sx = ox; break;
    }
    int k = 0, py = sy, px = sx;
    if (e.interlace) {
      k = kAdam7Pass[sy & 7][sx & 7];
      py = (sy - kAdam7[k][1]) / kAdam7[k][3];
      px = (sx - kAdam7[k][0]) / kAdam7[k][2];
    }
    const unsigned char *row = img + pbase[k] + (int64_t)py * (prb[k] + 1) + 1;
    unsigned b, g, r;
    if (depth < 8) {
      const int bit = px * depth;
      const unsigned v = (row[bit >> 3] >> (8 - depth - (bit & 7))) & ((1u << depth) - 1);
      if (ct == 3) {
        r = pal[3 * v]; g = pal[3 * v + 1]; b = pal[3 * v + 2];
      } else {
        b = g = r = v * (255u / ((1u << depth) - 1));      // libpng's expansion of 1/2/4-bit gray: bit replication
      }
    } else {
      const unsigned char *p = row + (int64_t)px * ch * sb;  // 16-bit samples: the high byte, as png_set_strip_16
      if (ct == 3) {
        const unsigned v = p[0];
        r = pal[3 * v]; g = pal[3 * v + 1]; b = pal[3 * v + 2];
      } else if (ct == 0 || ct == 4) {
        b = g = r = p[0];
      } else {
        r = p[0]; g = p[sb]; b = p[2 * sb];
      }
    }
    unsigned char *q = out + i * 3;
    q[0] = (unsigned char)b;
    q[1] = (unsigned char)g;
    q[2] = (unsigned char)r;
  }
}

}  // namespace

extern "C" int cpb200_png_decode_batch(const unsigned char *src, const cpb200_png_image *table, int B, void *workspace,
                                       size_t workspace_bytes, unsigned char *dst, int *status, void *stream) {
  if (!src || !table || !workspace || !dst || !status || B < 1)
    return cpb::fail(CPB200_ERR_ARG, "png_decode_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "png_decode_batch: B = %d images exceed one launch (max 65535)", B);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  png_inflate_kernel<<<B, 32, 0, st>>>(src, table, ws, workspace_bytes, status);
  int rc = cpb::check_launch("png_inflate_kernel");
  if (rc) return rc;
  png_unfilter_kernel<<<B, 32, 0, st>>>(table, ws, status);
  rc = cpb::check_launch("png_unfilter_kernel");
  if (rc) return rc;
  // the sizes live on the device: enough blocks per image to fill the GPU for one large image, fewer as B grows
  const dim3 grid((unsigned)std::max(1, 132 * 8 / B), (unsigned)B);
  png_output_kernel<<<grid, 256, 0, st>>>(src, table, ws, status, dst);
  return cpb::check_launch("png_output_kernel");
}

// cpb200_webp_lossless_decode_batch: cv2.imread(path, IMREAD_COLOR) of lossless WebP files (VP8L, RFC 9649) on the
// device, byte for byte as libwebp through OpenCV 4.13, for many files per launch.  Three kernels:
//   webp_lossless_entropy_kernel    one thread per image (a CTA of one thread, with the colour cache and the code
//                                   lengths in shared memory): the transform list and the predictor, cross-colour and
//                                   palette sub-images, the colour cache size, the entropy image and every prefix-code
//                                   group, then the LZ77 / colour-cache coded ARGB image at its coded width.  Serial
//                                   within an image, as libwebp is, so the batch gives the parallelism;
//   webp_lossless_transform_kernel  one CTA per image: the inverse transforms in reverse order.  Colour indexing,
//                                   subtract-green and cross-colour are per pixel; the predictor runs over the
//                                   wavefronts x + 2y = t, since a pixel reads its left, top-left, top and top-right
//                                   neighbours, all on earlier wavefronts;
//   webp_lossless_output_kernel     one thread per output pixel: ARGB -> BGR (alpha dropped, as cv2.imread's
//                                   WebPDecodeBGR does) with OpenCV's EXIF orientation as an index mapping.
// The host side (centerpose_b200/webp_lossless.py) parses the RIFF container and the 5-byte VP8L header and builds
// the table; the kernels trust it.  A stream libwebp refuses gets status 1: a code-length set that is empty,
// incomplete or over-subscribed (one used symbol is a code of no bits), a repeat or max_symbol past the alphabet, a
// transform type seen twice, colour cache bits outside 1..11, a backward reference before the image start or past its
// end, or more bits read than the data holds.  Status 2: the entropy image names more than kMaxGroups groups, or the
// workspace does not fit.
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_webp_lossless_image) == 56, "cpb200_webp_lossless_image layout is part of the C ABI");

enum { PREDICTOR = 0, CROSS_COLOR = 1, SUBTRACT_GREEN = 2, COLOR_INDEXING = 3 };

// Prefix-code groups a main image may use (the largest entropy-image index plus one).  cv2.imencode's default
// (lossless) files use at most 37 over the 256 files of tools/bench_webp.py --lossless; a file that needs more gets
// status 2 and is read by cv2.imread.  Each group costs kGroupBytes of workspace (webp_lossless.py MAX_GROUPS).
constexpr int kMaxGroups = CPB200_WEBP_LOSSLESS_MAX_GROUPS;
constexpr int kRootBits = 8;                           // a code's lookup table takes its next 8 bits
constexpr int kMaxCacheBits = 11;
// symbols of the five codes of a group: green + 24 length prefixes + up to 2^11 cache entries, red, blue, alpha,
// 40 distance prefixes
__constant__ int kSymOffset[6] = {0, 280 + 2048, 280 + 2048 + 256, 280 + 2048 + 512, 280 + 2048 + 768,
                                  280 + 2048 + 808};
constexpr int kSymTotal = 280 + 2048 + 808;
// one group in the workspace: per code a 256-entry table (length << 12 | symbol, 0 for a longer code), 16 code-length
// counts (count[0]: 1 + the symbol of a single-symbol code, else 0), then the symbols sorted by code
constexpr int64_t kGroupBytes = 5 * 256 * 2 + 5 * 16 * 2 + kSymTotal * 2;
static_assert(kGroupBytes == 8992 && kGroupBytes % 16 == 0, "webp_lossless.py GROUP_BYTES");
constexpr int kHeaderBytes = 128;

// RFC 9649 3.7.2.1.1: the order of the code-length code's lengths
__constant__ unsigned char kCodeLengthOrder[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
// RFC 9649 4.2.2: (xi, yi) of distance codes 1..120
__constant__ signed char kDistanceMap[240] = {
    0, 1, 1, 0, 1, 1, -1, 1, 0, 2, 2, 0, 1, 2, -1, 2, 2, 1, -2, 1, 2, 2, -2, 2, 0, 3, 3, 0,
    1, 3, -1, 3, 3, 1, -3, 1, 2, 3, -2, 3, 3, 2, -3, 2, 0, 4, 4, 0, 1, 4, -1, 4, 4, 1,
    -4, 1, 3, 3, -3, 3, 2, 4, -2, 4, 4, 2, -4, 2, 0, 5, 3, 4, -3, 4, 4, 3, -4, 3, 5, 0,
    1, 5, -1, 5, 5, 1, -5, 1, 2, 5, -2, 5, 5, 2, -5, 2, 4, 4, -4, 4, 3, 5, -3, 5, 5, 3,
    -5, 3, 0, 6, 6, 0, 1, 6, -1, 6, 6, 1, -6, 1, 2, 6, -2, 6, 6, 2, -6, 2, 4, 5, -4, 5,
    5, 4, -5, 4, 3, 6, -3, 6, 6, 3, -6, 3, 0, 7, 7, 0, 1, 7, -1, 7, 5, 5, -5, 5, 7, 1,
    -7, 1, 4, 6, -4, 6, 6, 4, -6, 4, 2, 7, -2, 7, 7, 2, -7, 2, 3, 7, -3, 7, 7, 3, -7, 3,
    5, 6, -5, 6, 6, 5, -6, 5, 8, 0, 4, 7, -4, 7, 7, 4, -7, 4, 8, 1, 8, 2, 6, 6, -6, 6,
    8, 3, 5, 7, -5, 7, 7, 5, -7, 5, 8, 4, 6, 7, -6, 7, 7, 6, -7, 6, 8, 5, 7, 7, -7, 7,
    8, 6, 8, 7,
};

// what the entropy kernel leaves for the transform and output kernels at the start of an image's workspace
struct Header {
  int ntrans, final_plane, pad0, pad1;
  int type[4], bits[4], xsize[4];
  int64_t data[4];                                     // uint32 index of the transform's data in the sub-image area
};
static_assert(sizeof(Header) <= kHeaderBytes, "header");

// an image's workspace: header, two ARGB planes of w x h (the coded image, and the output of colour indexing), the
// sub-images (predictor, cross-colour and entropy images of at most ceil(w/4) x ceil(h/4) each, the 256-entry
// palette), the prefix-code groups (webp_lossless.py workspace_bytes)
struct Layout {
  int64_t plane0, plane1, sub, groups, total;
};

__device__ __forceinline__ int64_t up16(int64_t x) { return (x + 15) & ~(int64_t)15; }

__device__ __forceinline__ Layout layout(int w, int h) {
  Layout L;
  const int64_t px = (int64_t)w * h, tiles = (int64_t)((w + 3) >> 2) * ((h + 3) >> 2);
  L.plane0 = kHeaderBytes;
  L.plane1 = L.plane0 + up16(4 * px);
  L.sub = L.plane1 + up16(4 * px);
  L.groups = L.sub + up16(4 * (3 * tiles + 256));
  L.total = L.groups + kMaxGroups * kGroupBytes;
  return L;
}

__device__ __forceinline__ bool fits(const cpb200_webp_lossless_image &e, const Layout &L, size_t ws_bytes) {
  return e.ws_offset >= 0 && e.ws_bytes >= L.total && (uint64_t)e.ws_offset + e.ws_bytes <= ws_bytes;
}

__device__ __forceinline__ int subsample(int size, int bits) { return (size + (1 << bits) - 1) >> bits; }

// LSB-first bit reader.  libwebp's reader flags the end of the stream once more bits were read than the data holds,
// counting at least 8 bytes (it loads 8 bytes up front), and every header and image it reads fails then.  Past the
// data it reads zero bits: `s` is followed by >= 32 zero bytes, and no byte past those is loaded
struct Bits {
  const unsigned char *s;
  int64_t p, len, limit;
  uint64_t acc;
  int n;

  __device__ void init(const unsigned char *src, int64_t bytes) {
    s = src; p = 0; len = bytes; acc = 0; n = 0;
    limit = 8 * (bytes > 8 ? bytes : 8);
  }
  __device__ __forceinline__ void fill() {
    if (p <= len + 8) {
      const uintptr_t a = reinterpret_cast<uintptr_t>(s + p);
      const uint64_t *w = reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7);
      const int sh = (int)(a & 7) * 8;
      uint64_t v = __ldg(w) >> sh;
      if (sh) v |= __ldg(w + 1) << (64 - sh);
      acc |= v << n;
    }
    p += (63 - n) >> 3;
    n |= 56;
  }
  __device__ __forceinline__ uint32_t get(int k) {     // k <= 24
    if (n < k) fill();
    const uint32_t v = (uint32_t)(acc & ((1ull << k) - 1));
    acc >>= k;
    n -= k;
    return v;
  }
  __device__ __forceinline__ bool eos() const { return 8 * p - n > limit; }
};

// one prefix code of a group, read from the workspace
struct Code {
  const unsigned short *lut, *count, *sym;
};

__device__ __forceinline__ Code code_of(unsigned char *group, int j) {
  unsigned short *g = reinterpret_cast<unsigned short *>(group);
  return Code{g + 256 * j, g + 5 * 256 + 16 * j, g + 5 * 256 + 5 * 16 + kSymOffset[j]};
}

// builds the code of lengths len[0..n) into `lut` (2^root entries) / `count` / `sym`; false where libwebp refuses
// the lengths: none used, or (more than one used) a code that is over-subscribed or incomplete
__device__ bool build(const unsigned char *len, int n, int root, unsigned short *lut, unsigned short *count,
                      unsigned short *sym) {
  int cnt[16], used = 0, last = 0;
  for (int l = 0; l < 16; ++l) cnt[l] = 0;
  for (int s = 0; s < n; ++s) {
    ++cnt[len[s]];
    if (len[s]) { ++used; last = s; }
  }
  if (!used) return false;
  if (used == 1) {                                     // no bits: libwebp's table of bits-0 entries
    count[0] = (unsigned short)(last + 1);
    return true;
  }
  int left = 1;
  for (int l = 1; l < 16; ++l) {
    left = 2 * left - cnt[l];
    if (left < 0) return false;
  }
  if (left) return false;
  int offs[16], next[16];
  count[0] = 0;
  offs[1] = 0; next[1] = 0;
  for (int l = 1; l < 16; ++l) {
    count[l] = (unsigned short)cnt[l];
    if (l < 15) {
      offs[l + 1] = offs[l] + cnt[l];
      next[l + 1] = (next[l] + cnt[l]) << 1;
    }
  }
  for (int i = 0; i < (1 << root); ++i) lut[i] = 0;
  for (int s = 0; s < n; ++s) {
    const int l = len[s];
    if (!l) continue;
    sym[offs[l]++] = (unsigned short)s;
    const int c = next[l]++;
    if (l <= root) {
      const unsigned rev = __brev((unsigned)c) >> (32 - l);
      for (unsigned k = rev; k < (1u << root); k += 1u << l) lut[k] = (unsigned short)(l << 12 | s);
    }
  }
  return true;
}

// the next symbol of a built (so complete) code
__device__ __forceinline__ int read_symbol(Bits &br, const Code &c, int root) {
  if (c.count[0]) return c.count[0] - 1;
  if (br.n < 15) br.fill();
  const unsigned e = c.lut[br.acc & ((1u << root) - 1)];
  if (e) {
    br.acc >>= e >> 12;
    br.n -= e >> 12;
    return e & 4095;
  }
  int code = 0, first = 0, index = 0;
  uint64_t a = br.acc;
  for (int l = 1; l < 16; ++l) {
    code |= (int)(a & 1);
    a >>= 1;
    const int count = c.count[l];
    if (code - count < first) {
      br.acc >>= l;
      br.n -= l;
      return c.sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return 0;                                            // not reached: every built code is complete
}

struct Ctx {
  Bits br;
  unsigned char *groups;
  uint32_t *cache;                                     // shared, 2^11 entries
  unsigned char *lengths;                              // shared, kSymOffset[1] entries
};

// one prefix code (RFC 9649 3.7.2.1) of `alphabet` symbols into group slot `j` of `group`
__device__ bool read_code(Ctx &c, int alphabet, unsigned char *group, int j) {
  Bits &br = c.br;
  unsigned char *len = c.lengths;
  for (int s = 0; s < alphabet; ++s) len[s] = 0;
  if (br.get(1)) {                                     // simple: one or two symbols of at most 8 bits
    const int two = br.get(1);
    int s = br.get(br.get(1) ? 8 : 1);
    if (s < alphabet) len[s] = 1;
    if (two) {
      s = br.get(8);
      if (s < alphabet) len[s] = 1;
    }
  } else {
    unsigned char cl[19];
    for (int k = 0; k < 19; ++k) cl[k] = 0;
    const int ncl = br.get(4) + 4;
    for (int k = 0; k < ncl; ++k) cl[kCodeLengthOrder[k]] = (unsigned char)br.get(3);
    unsigned short lut[128], count[16], sym[19];
    if (!build(cl, 19, 7, lut, count, sym)) return false;
    const Code clc{lut, count, sym};
    int max_symbol = alphabet;
    if (br.get(1)) {
      max_symbol = 2 + br.get(2 + 2 * br.get(3));
      if (max_symbol > alphabet) return false;
    }
    int prev = 8;
    for (int s = 0; s < alphabet;) {
      if (max_symbol-- == 0) break;
      const int v = read_symbol(br, clc, 7);
      if (v < 16) {
        len[s++] = (unsigned char)v;
        if (v) prev = v;
      } else {
        const int rep = br.get(v == 16 ? 2 : v == 17 ? 3 : 7) + (v == 18 ? 11 : 3);
        if (s + rep > alphabet) return false;
        const unsigned char l = v == 16 ? (unsigned char)prev : 0;
        for (int k = 0; k < rep; ++k) len[s++] = l;
      }
    }
  }
  if (br.eos()) return false;
  unsigned short *g = reinterpret_cast<unsigned short *>(group);
  return build(len, alphabet, kRootBits, g + 256 * j, g + 5 * 256 + 16 * j, g + 5 * 256 + 5 * 16 + kSymOffset[j]);
}

__device__ bool read_group(Ctx &c, unsigned char *group, int cache_bits) {
  for (int j = 0; j < 5; ++j) {
    const int alphabet = j == 0 ? 280 + (cache_bits ? 1 << cache_bits : 0) : j == 4 ? 40 : 256;
    if (!read_code(c, alphabet, group, j)) return false;
  }
  return true;
}

__device__ __forceinline__ int prefix_value(Bits &br, int sym) {
  if (sym < 4) return sym + 1;
  const int extra = (sym - 2) >> 1;
  return ((2 + (sym & 1)) << extra) + (int)br.get(extra) + 1;
}

__device__ __forceinline__ void cache_put(uint32_t *cache, int bits, uint32_t v) {
  if (bits) cache[(0x1e35a7bdu * v) >> (32 - bits)] = v;
}

// the LZ77 / colour-cache coded pixels of a w x h image (RFC 9649 5.2), group g of the pixel at (x, y) being
// meta[(y >> mb) * mw + (x >> mb)] (group 0 without an entropy image); 0, or the status
__device__ int read_pixels(Ctx &c, int w, int h, uint32_t *out, int cache_bits, const uint32_t *meta, int mb, int mw) {
  Bits &br = c.br;
  uint32_t *cache = c.cache;
  if (cache_bits)
    for (int i = 0; i < (1 << cache_bits); ++i) cache[i] = 0;
  const int64_t n = (int64_t)w * h;
  int64_t pos = 0;
  int x = 0, y = 0, cur = -1;
  Code g[5];
  while (pos < n) {
    const int gi = meta ? (int)((meta[(int64_t)(y >> mb) * mw + (x >> mb)] >> 8) & 0xffff) : 0;
    if (gi != cur) {
      cur = gi;
      for (int j = 0; j < 5; ++j) g[j] = code_of(c.groups + (int64_t)gi * kGroupBytes, j);
    }
    const int s = read_symbol(br, g[0], kRootBits);
    if (s < 256) {
      const int r = read_symbol(br, g[1], kRootBits);
      const int b = read_symbol(br, g[2], kRootBits);
      const int a = read_symbol(br, g[3], kRootBits);
      if (br.eos()) return 1;
      const uint32_t v = (uint32_t)a << 24 | (uint32_t)r << 16 | (uint32_t)s << 8 | (uint32_t)b;
      out[pos++] = v;
      cache_put(cache, cache_bits, v);
      if (++x == w) { x = 0; ++y; }
    } else if (s < 280) {
      const int length = prefix_value(br, s - 256);
      const int code = prefix_value(br, read_symbol(br, g[4], kRootBits));
      int64_t dist;
      if (code > 120) {
        dist = code - 120;
      } else {
        dist = kDistanceMap[2 * (code - 1)] + (int64_t)kDistanceMap[2 * (code - 1) + 1] * w;
        if (dist < 1) dist = 1;
      }
      if (br.eos()) return 1;
      if (dist > pos || length > n - pos) return 1;
      for (int k = 0; k < length; ++k, ++pos) {
        const uint32_t v = out[pos - dist];
        out[pos] = v;
        cache_put(cache, cache_bits, v);
      }
      x += length;
      while (x >= w) { x -= w; ++y; }
    } else {
      if (br.eos()) return 1;
      const uint32_t v = cache[s - 280];
      out[pos++] = v;
      cache_put(cache, cache_bits, v);
      if (++x == w) { x = 0; ++y; }
    }
  }
  return br.eos() ? 1 : 0;
}

__device__ int read_cache_bits(Bits &br) {
  if (!br.get(1)) return 0;
  const int bits = br.get(4);
  return bits >= 1 && bits <= kMaxCacheBits ? bits : -1;
}

// a sub-image (transform data or entropy image): its own colour cache and one group, no entropy image
__device__ int read_sub_image(Ctx &c, int w, int h, uint32_t *out) {
  const int cache_bits = read_cache_bits(c.br);
  if (cache_bits < 0) return 1;
  if (!read_group(c, c.groups, cache_bits)) return 1;
  return read_pixels(c, w, h, out, cache_bits, nullptr, 0, 0);
}

__device__ int decode_stream(Ctx &c, int w, int h, Header &hd, uint32_t *plane, uint32_t *sub) {
  Bits &br = c.br;
  br.get(8); br.get(14); br.get(14); br.get(1); br.get(3);   // the header, checked on the host
  int64_t used = 0;                                    // uint32 entries of the sub-image area taken
  int xs = w, seen = 0;
  hd.ntrans = 0;
  while (br.get(1)) {
    const int type = br.get(2);
    if (seen & (1 << type)) return 1;
    seen |= 1 << type;
    const int k = hd.ntrans++;
    hd.type[k] = type;
    hd.xsize[k] = xs;
    hd.bits[k] = 0;
    hd.data[k] = used;
    if (type == PREDICTOR || type == CROSS_COLOR) {
      const int bits = br.get(3) + 2;
      hd.bits[k] = bits;
      const int tw = subsample(xs, bits), th = subsample(h, bits);
      if (read_sub_image(c, tw, th, sub + used)) return 1;
      used += (int64_t)tw * th;
    } else if (type == COLOR_INDEXING) {
      const int ncolors = br.get(8) + 1;
      const int bits = ncolors > 16 ? 0 : ncolors > 4 ? 1 : ncolors > 2 ? 2 : 3;
      hd.bits[k] = bits;
      uint32_t *pal = sub + used;
      if (read_sub_image(c, ncolors, 1, pal)) return 1;
      for (int i = 1; i < ncolors; ++i) {                // delta-coded per byte; entries past the palette are 0
        const uint32_t a = pal[i], b = pal[i - 1];
        pal[i] = (((a & 0xff00ff00u) + (b & 0xff00ff00u)) & 0xff00ff00u) |
                 (((a & 0x00ff00ffu) + (b & 0x00ff00ffu)) & 0x00ff00ffu);
      }
      for (int i = ncolors; i < 256; ++i) pal[i] = 0;
      used += 256;
      xs = subsample(xs, bits);
    }
  }
  const int cache_bits = read_cache_bits(br);
  if (cache_bits < 0) return 1;
  const uint32_t *meta = nullptr;
  int mb = 0, mw = 0, ngroups = 1;
  if (br.get(1)) {
    mb = br.get(3) + 2;
    mw = subsample(xs, mb);
    const int mh = subsample(h, mb);
    uint32_t *m = sub + used;
    if (read_sub_image(c, mw, mh, m)) return 1;
    for (int64_t i = 0; i < (int64_t)mw * mh; ++i) {
      const int gi = (int)((m[i] >> 8) & 0xffff);
      if (gi >= ngroups) ngroups = gi + 1;
    }
    meta = m;
  }
  if (br.eos()) return 1;
  if (ngroups > kMaxGroups) return 2;
  // every group up to the largest index is read and checked, used or not
  for (int gi = 0; gi < ngroups; ++gi)
    if (!read_group(c, c.groups + (int64_t)gi * kGroupBytes, cache_bits)) return 1;
  hd.final_plane = 0;
  return read_pixels(c, xs, h, plane, cache_bits, meta, mb, mw);
}

// grid B CTAs x 1 thread: CTA b entropy-decodes image b into its workspace
__global__ void __launch_bounds__(1) webp_lossless_entropy_kernel(const unsigned char *__restrict__ src,
                                                                  const cpb200_webp_lossless_image *__restrict__ table,
                                                                  unsigned char *__restrict__ ws, size_t ws_bytes,
                                                                  int *__restrict__ status) {
  __shared__ uint32_t cache[1 << kMaxCacheBits];
  __shared__ unsigned char lengths[280 + (1 << kMaxCacheBits)];
  const cpb200_webp_lossless_image &e = table[blockIdx.x];
  const Layout L = layout(e.w, e.h);
  if (!fits(e, L, ws_bytes)) {
    status[blockIdx.x] = 2;
    return;
  }
  unsigned char *img = ws + e.ws_offset;
  Ctx c;
  c.br.init(src + e.src_offset, e.src_bytes);
  c.groups = img + L.groups;
  c.cache = cache;
  c.lengths = lengths;
  Header hd;
  const int st = decode_stream(c, e.w, e.h, hd, reinterpret_cast<uint32_t *>(img + L.plane0),
                               reinterpret_cast<uint32_t *>(img + L.sub));
  if (!st) {
    for (int k = 0; k < hd.ntrans; ++k)
      if (hd.type[k] == COLOR_INDEXING) hd.final_plane = 1;
    *reinterpret_cast<Header *>(img) = hd;
  }
  status[blockIdx.x] = st;
}

__device__ __forceinline__ uint32_t add_pixels(uint32_t a, uint32_t b) {
  return (((a & 0xff00ff00u) + (b & 0xff00ff00u)) & 0xff00ff00u) | (((a & 0x00ff00ffu) + (b & 0x00ff00ffu)) & 0x00ff00ffu);
}
__device__ __forceinline__ uint32_t average2(uint32_t a, uint32_t b) { return (((a ^ b) & 0xfefefefeu) >> 1) + (a & b); }
__device__ __forceinline__ int clip255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

// libwebp's predictors; 14 and 15 predict ARGB black, as mode 0 does
__device__ uint32_t predict(int mode, uint32_t L, uint32_t T, uint32_t TL, uint32_t TR) {
  switch (mode) {
    case 1: return L;
    case 2: return T;
    case 3: return TR;
    case 4: return TL;
    case 5: return average2(average2(L, TR), T);
    case 6: return average2(L, TL);
    case 7: return average2(L, T);
    case 8: return average2(TL, T);
    case 9: return average2(T, TR);
    case 10: return average2(average2(L, TL), average2(T, TR));
    case 11: {                                         // Select: T on a tie
      int d = 0;
      for (int s = 0; s < 32; s += 8) {
        const int l = (L >> s) & 255, t = (T >> s) & 255, tl = (TL >> s) & 255;
        d += abs(l - tl) - abs(t - tl);
      }
      return d <= 0 ? T : L;
    }
    case 12: {
      uint32_t v = 0;
      for (int s = 0; s < 32; s += 8)
        v |= (uint32_t)clip255((int)((L >> s) & 255) + (int)((T >> s) & 255) - (int)((TL >> s) & 255)) << s;
      return v;
    }
    case 13: {
      const uint32_t a = average2(L, T);
      uint32_t v = 0;
      for (int s = 0; s < 32; s += 8) {
        const int x = (a >> s) & 255, tl = (TL >> s) & 255;
        v |= (uint32_t)clip255(x + (x - tl) / 2) << s;
      }
      return v;
    }
    default: return 0xff000000u;
  }
}

// grid B CTAs x 512 threads: CTA b undoes image b's transforms, last read first
__global__ void __launch_bounds__(512) webp_lossless_transform_kernel(const cpb200_webp_lossless_image *__restrict__ table,
                                                                      unsigned char *__restrict__ ws,
                                                                      const int *__restrict__ status) {
  if (status[blockIdx.x]) return;
  const cpb200_webp_lossless_image &e = table[blockIdx.x];
  const Layout L = layout(e.w, e.h);
  unsigned char *img = ws + e.ws_offset;
  const Header hd = *reinterpret_cast<const Header *>(img);
  uint32_t *cur = reinterpret_cast<uint32_t *>(img + L.plane0);
  const uint32_t *sub = reinterpret_cast<const uint32_t *>(img + L.sub);
  const int h = e.h, tid = threadIdx.x, nt = blockDim.x;
  for (int k = hd.ntrans - 1; k >= 0; --k) {
    const int W = hd.xsize[k], bits = hd.bits[k];
    const int64_t n = (int64_t)W * h;
    const uint32_t *data = sub + hd.data[k];
    if (hd.type[k] == SUBTRACT_GREEN) {
      for (int64_t i = tid; i < n; i += nt) {
        const uint32_t v = cur[i], g = (v >> 8) & 255;
        cur[i] = (v & 0xff00ff00u) | ((((v >> 16) + g) & 255) << 16) | ((v + g) & 255);
      }
    } else if (hd.type[k] == CROSS_COLOR) {
      const int tw = subsample(W, bits);
      for (int64_t i = tid; i < n; i += nt) {
        const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
        const uint32_t m = data[(int64_t)(y >> bits) * tw + (x >> bits)], v = cur[i];
        const int g = (signed char)(v >> 8);
        const int r = ((int)(v >> 16) + (((signed char)m * g) >> 5)) & 255;
        const int b = ((int)v + (((signed char)(m >> 8) * g) >> 5) + (((signed char)(m >> 16) * (signed char)r) >> 5)) & 255;
        cur[i] = (v & 0xff00ff00u) | (uint32_t)r << 16 | (uint32_t)b;
      }
    } else if (hd.type[k] == COLOR_INDEXING) {
      uint32_t *out = reinterpret_cast<uint32_t *>(img + L.plane1);
      const int pw = subsample(W, bits), per = 8 >> bits;
      for (int64_t i = tid; i < n; i += nt) {
        const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
        const uint32_t packed = (cur[(int64_t)y * pw + (x >> bits)] >> 8) & 255;
        out[i] = data[(packed >> ((x & ((1 << bits) - 1)) * per)) & ((1u << per) - 1)];
      }
      cur = out;
    } else {                                           // PREDICTOR, in place over the wavefronts x + 2y = t
      const int tw = subsample(W, bits);
      for (int t = 0; t <= W - 1 + 2 * (h - 1); ++t) {
        const int ylo = t > W - 1 ? (t - W + 2) >> 1 : 0, yhi = min(h - 1, t >> 1);
        for (int y = ylo + tid; y <= yhi; y += nt) {
          const int x = t - 2 * y;
          const int64_t i = (int64_t)y * W + x;
          uint32_t p;
          if (y == 0) {
            p = x == 0 ? 0xff000000u : cur[i - 1];
          } else if (x == 0) {
            p = cur[i - W];
          } else {
            const int mode = (data[(int64_t)(y >> bits) * tw + (x >> bits)] >> 8) & 15;
            // the top-right of the last column is the first pixel of this row, as in libwebp's row-major buffer
            p = predict(mode, cur[i - 1], cur[i - W], cur[i - W - 1], cur[i - W + 1]);
          }
          cur[i] = add_pixels(cur[i], p);
        }
        __syncthreads();
      }
    }
    __syncthreads();
  }
}

// grid (pixel blocks, image) x 256 threads: one thread per output pixel in row-major order of the oriented image
__global__ void __launch_bounds__(256) webp_lossless_output_kernel(const cpb200_webp_lossless_image *__restrict__ table,
                                                                   const unsigned char *__restrict__ ws,
                                                                   const int *__restrict__ status,
                                                                   unsigned char *__restrict__ dst) {
  if (status[blockIdx.y]) return;
  const cpb200_webp_lossless_image &e = table[blockIdx.y];
  const Layout L = layout(e.w, e.h);
  const unsigned char *img = ws + e.ws_offset;
  const Header *hd = reinterpret_cast<const Header *>(img);
  const uint32_t *argb = reinterpret_cast<const uint32_t *>(img + (hd->final_plane ? L.plane1 : L.plane0));
  const int h = e.h, w = e.w, o = e.orientation;
  const int ow = o >= 5 ? h : w;
  const int64_t total = (int64_t)h * w;
  unsigned char *out = dst + e.dst_offset;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i - (int64_t)oy * ow);
    int sy, sx;
    cpb::exif_source(o, oy, ox, h, w, sy, sx);
    const uint32_t v = argb[(int64_t)sy * w + sx];
    unsigned char *q = out + i * 3;
    q[0] = (unsigned char)v;
    q[1] = (unsigned char)(v >> 8);
    q[2] = (unsigned char)(v >> 16);
  }
}

}  // namespace

extern "C" int cpb200_webp_lossless_decode_batch(const unsigned char *src, const cpb200_webp_lossless_image *table,
                                                 int B, void *workspace, size_t workspace_bytes, unsigned char *dst,
                                                 int *status, void *stream) {
  if (!src || !table || !workspace || !dst || !status || B < 1)
    return cpb::fail(CPB200_ERR_ARG, "webp_lossless_decode_batch: bad arguments");
  if (B > 65535)
    return cpb::fail(CPB200_ERR_ARG, "webp_lossless_decode_batch: B = %d images exceed one launch (max 65535)", B);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  webp_lossless_entropy_kernel<<<B, 1, 0, st>>>(src, table, ws, workspace_bytes, status);
  int rc = cpb::check_launch("webp_lossless_entropy_kernel");
  if (rc) return rc;
  webp_lossless_transform_kernel<<<B, 512, 0, st>>>(table, ws, status);
  rc = cpb::check_launch("webp_lossless_transform_kernel");
  if (rc) return rc;
  const dim3 grid((unsigned)std::max(1, 132 * 8 / B), (unsigned)B);
  webp_lossless_output_kernel<<<grid, 256, 0, st>>>(table, ws, status, dst);
  return cpb::check_launch("webp_lossless_output_kernel");
}

// cv2.imencode('.png', img) of BGR uint8 images, byte for byte: cpb200_png_encode_batch.
//
// OpenCV 4.13 writes through libpng with the Sub filter, zlib level 1, strategy Z_RLE and memLevel 8.  Every choice
// that makes the file is then fixed, and the one that looks serial, deflate_rle's parse, is closed form per run of
// equal bytes: a literal, then matches of 258 at distance 1, then the remainder as one match if >= 3, else literals.
// So each byte knows from the start and end of its run whether it emits a symbol, and a prefix sum places the symbol.
//
//   filter_kernel     per 4096-byte tile: Sub (None at width 1) over RGB -> scanlines; run-start / run-end flags,
//                     Adler-32 partial sums; zeroes its share of the zlib stream
//   scan_tiles_kernel per image (one warp): where the run through each tile's first and last byte starts and ends;
//                     the Adler-32
//   symbols_kernel    per tile: each byte's run -> its symbol (count pass, then write pass at the prefix sums)
//   scan_syms_kernel  per image (one warp): the tiles' symbol offsets, the symbol count, the block count
//   blocks_kernel     per deflate block of 16383 symbols (lit_bufsize - 1) and the final one: histograms, zlib's
//                     build_tree / build_bl_tree, and _tr_flush_block's choice of stored / static / dynamic
//   layout_kernel     one CTA: per image the blocks' bit offsets (a stored block's padding depends on its bit
//                     position), the zlib header (libpng's window reduction and optimize_cmf) and Adler-32 trailer,
//                     the file size; the files' offsets packed back to back in input order
//   emit_kernel       per deflate block: the block header and trees, every symbol's code OR-ed into the stream at its
//                     bit offset (a prefix sum of the code lengths), or the stored bytes
//   assemble_kernel   per IDAT chunk (one warp): the signature and IHDR, 8192 bytes of the stream, its CRC-32 (per
//                     lane, combined), IEND, written at the file's packed offset
#include "common.cuh"

#include <climits>

namespace {

static_assert(sizeof(cpb200_png_encode_image) == 96, "cpb200_png_encode_image layout is part of the C ABI");

constexpr int kThreads = 256;
constexpr int kTile = CPB200_PNG_ENCODE_TILE;
constexpr int kPerThread = kTile / kThreads;
constexpr int kBlockSymbols = 16383;
constexpr int kMaxMatch = 258;
constexpr int kIdat = 8192;
constexpr int L_CODES = 286, D_CODES = 30, BL_CODES = 19, HEAP_SIZE = 2 * L_CODES + 1;
constexpr int MAX_BITS = 15, MAX_BL_BITS = 7, END_BLOCK = 256;
constexpr int kStored = 0, kStatic = 1, kDynamic = 2;
static_assert(kPerThread == 16, "one tile is 16 bytes per thread");

__constant__ unsigned char c_extra_lbits[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4,
                                                5, 5, 5, 5, 0};
__constant__ unsigned char c_base_length[29] = {0,  1,  2,  3,  4,  5,  6,  7,  8,   10,  12,  14,  16,  20, 24,
                                                28, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192, 224, 0};
__constant__ unsigned char c_extra_dbits[D_CODES] = {0, 0, 0, 0, 1, 1, 2, 2,  3,  3,  4,  4,  5,  5,  6,
                                                     6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ unsigned char c_extra_blbits[BL_CODES] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};
__constant__ unsigned char c_bl_order[BL_CODES] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
// x^(2^k) modulo the CRC-32 polynomial, reflected (zlib's x2n_table)
__constant__ uint32_t c_x2n[32] = {
    0x40000000u, 0x20000000u, 0x08000000u, 0x00800000u, 0x00008000u, 0xedb88320u, 0xb1e6b092u, 0xa06a2517u,
    0xed627daeu, 0x88d14467u, 0xd7bbfe6au, 0xec447f11u, 0x8e7ea170u, 0x6427800eu, 0x4d47bae0u, 0x09fe548fu,
    0x83852d0fu, 0x30362f1au, 0x7b5a9cc3u, 0x31fec169u, 0x9fec022au, 0x6c8dedc4u, 0x15d6874du, 0x5fde7a4eu,
    0xbad90e37u, 0x2e4e5eefu, 0x4eaba214u, 0xa8a472c0u, 0x429a969eu, 0x148d302au, 0xc40ba6d0u, 0xc4e22c3cu};

struct Tile {
  int last_start;    // last run start in the tile, -1 if none
  int first_end;     // first run end in the tile, INT_MAX if none
  int s_in;          // last run start before the tile
  int e_out;         // first run end after the tile
  int nsym, sym_off;
  unsigned a1, a2;   // sum b and sum (N - p) b of the tile's bytes, mod 65521
};
static_assert(sizeof(Tile) == CPB200_PNG_ENCODE_TILE_REC, "tile record size");

struct State {
  long long nsym, file_offset, file_bytes, zbytes;
  int nblocks, nchunks;
  unsigned adler;
  int pad[5];
};
static_assert(sizeof(State) == CPB200_PNG_ENCODE_STATE_REC, "state record size");

struct Block {
  long long stored_len;   // bytes the block covers
  long long byte_start;   // its first byte in the scanlines
  long long bit_off;      // its first bit in the zlib stream
  long long nbits;        // its size in bits, header and EOB included
  int kind, nsym;
  short lcodes, dcodes, blcodes, pad;
  unsigned short lcode[L_CODES];
  unsigned char llen[L_CODES];
  unsigned short dcode[D_CODES];
  unsigned char dlen[D_CODES];
  unsigned short blcode[BL_CODES];
  unsigned char bllen[BL_CODES];
};
static_assert(sizeof(Block) <= CPB200_PNG_ENCODE_BLOCK_REC, "block record size");

__device__ __forceinline__ long long filtered_bytes(const cpb200_png_encode_image &e) {
  return (long long)e.h * (1 + 3 * (long long)e.w);
}

// the image whose slots [first, next image's first) hold `slot` (firsts ascending)
template <int cpb200_png_encode_image::*Field>
__device__ int find_image(const cpb200_png_encode_image *table, int B, int slot) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].*Field <= slot) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// filtered byte p: the row's filter type (1 Sub, 0 None for one-pixel rows), else R, G, B minus the pixel to the left
__device__ __forceinline__ unsigned char filt(const cpb200_png_encode_image &e, int p) {
  const int rowlen = 1 + 3 * e.w;
  const int y = p / rowlen, c = p - y * rowlen;
  if (c == 0) return e.w == 1 ? 0 : 1;
  const int i = c - 1, x = i / 3, ch = 2 - (i - 3 * x);
  const unsigned char *r = e.src + (long long)y * e.pitch;
  const unsigned char v = r[3 * x + ch];
  return (e.w > 1 && x > 0) ? (unsigned char)(v - r[3 * x - 3 + ch]) : v;
}

// ---- CTA scans over kThreads threads ----
template <typename T, typename Op>
__device__ T block_exclusive_scan(T v, T init, Op op, T *sm, T *total = nullptr) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x = op(x, y);
  }
  if (lane == 31) sm[warp] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    T acc = init;
    for (int w = 0; w < kThreads / 32; ++w) { const T t = sm[w]; sm[w] = acc; acc = op(acc, t); }
    sm[kThreads / 32] = acc;
  }
  __syncthreads();
  T prev = __shfl_up_sync(0xffffffffu, x, 1);
  const T r = lane == 0 ? sm[warp] : op(sm[warp], prev);
  if (total) *total = sm[kThreads / 32];
  __syncthreads();
  return r;
}

// suffix form: op over the threads after this one, and init
template <typename T, typename Op>
__device__ T block_exclusive_suffix(T v, T init, Op op, T *sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_down_sync(0xffffffffu, x, o);
    if (lane + o < 32) x = op(x, y);
  }
  if (lane == 0) sm[warp] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    T acc = init;
    for (int w = kThreads / 32 - 1; w >= 0; --w) { const T t = sm[w]; sm[w] = acc; acc = op(acc, t); }
  }
  __syncthreads();
  const T next = __shfl_down_sync(0xffffffffu, x, 1);
  const T r = lane == 31 ? sm[warp] : op(sm[warp], next);
  __syncthreads();
  return r;
}

struct MaxOp { __device__ int operator()(int a, int b) const { return a > b ? a : b; } };
struct MinOp { __device__ int operator()(int a, int b) const { return a < b ? a : b; } };
struct SumOp {
  __device__ int operator()(int a, int b) const { return a + b; }
  __device__ long long operator()(long long a, long long b) const { return a + b; }
};

__global__ void __launch_bounds__(kThreads) filter_kernel(const cpb200_png_encode_image *table, int B,
                                                          unsigned char *ws) {
  __shared__ unsigned char f[kTile + 2];
  __shared__ int s_ls, s_fe;
  __shared__ unsigned long long s_a1, s_a2;
  const int n = find_image<&cpb200_png_encode_image::tile0>(table, B, blockIdx.x);
  const cpb200_png_encode_image e = table[n];
  const int N = (int)filtered_bytes(e);
  const int ntiles = cpb::ceil_div(N, kTile);
  const int t = blockIdx.x - e.tile0;
  const int p0 = t * kTile, p1 = min(N, p0 + kTile);
  // this tile's share of the zlib stream, zeroed for emit_kernel's OR-ed writes
  {
    const long long words = e.z_bytes / 16, per = (words + ntiles - 1) / ntiles;
    uint4 *z = reinterpret_cast<uint4 *>(ws + e.z_offset);
    for (long long i = t * per + threadIdx.x; i < min(words, (t + 1) * per); i += kThreads) z[i] = make_uint4(0, 0, 0, 0);
  }
  if (threadIdx.x == 0) { s_ls = -1; s_fe = INT_MAX; s_a1 = 0; s_a2 = 0; }
  unsigned char *out = ws + e.filt_offset;
  unsigned long long a1 = 0, a2 = 0;
  for (int i = threadIdx.x; i < p1 - p0; i += kThreads) {
    const unsigned char v = filt(e, p0 + i);
    f[i + 1] = v;
    out[p0 + i] = v;
    a1 += v;
    a2 += (unsigned long long)(N - p0 - i) * v;
  }
  if (threadIdx.x == 0) f[0] = p0 > 0 ? filt(e, p0 - 1) : 0;
  if (threadIdx.x == 1) f[p1 - p0 + 1] = p1 < N ? filt(e, p1) : 0;
  __syncthreads();
  int ls = -1, fe = INT_MAX;
  for (int i = threadIdx.x; i < p1 - p0; i += kThreads) {
    const int p = p0 + i;
    if (p == 0 || f[i + 1] != f[i]) ls = max(ls, p);
    if (p == N - 1 || f[i + 1] != f[i + 2]) fe = min(fe, p);
  }
  if (ls >= 0) atomicMax(&s_ls, ls);
  if (fe != INT_MAX) atomicMin(&s_fe, fe);
  atomicAdd(&s_a1, a1 % 65521);
  atomicAdd(&s_a2, a2 % 65521);
  __syncthreads();
  if (threadIdx.x == 0) {
    Tile *tile = reinterpret_cast<Tile *>(ws + e.tile_offset) + t;
    tile->last_start = s_ls;
    tile->first_end = s_fe;
    tile->a1 = (unsigned)(s_a1 % 65521);
    tile->a2 = (unsigned)(s_a2 % 65521);
  }
}

// one warp per image
__global__ void __launch_bounds__(kThreads) scan_tiles_kernel(const cpb200_png_encode_image *table, int B,
                                                              unsigned char *ws) {
  const int n = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= B) return;
  const cpb200_png_encode_image e = table[n];
  const int N = (int)filtered_bytes(e);
  const int ntiles = cpb::ceil_div(N, kTile);
  Tile *tiles = reinterpret_cast<Tile *>(ws + e.tile_offset);
  int carry = -1;
  unsigned long long a1 = 0, a2 = 0;
  for (int base = 0; base < ntiles; base += 32) {
    const int t = base + lane;
    int x = t < ntiles ? tiles[t].last_start : -1;
    if (t < ntiles) { a1 += tiles[t].a1; a2 += tiles[t].a2; }
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x = max(x, y);
    }
    const int prev = __shfl_up_sync(0xffffffffu, x, 1);
    if (t < ntiles) tiles[t].s_in = max(carry, lane ? prev : -1);
    carry = max(carry, __shfl_sync(0xffffffffu, x, 31));
  }
  carry = INT_MAX;
  for (int base = (ntiles - 1) / 32 * 32; base >= 0; base -= 32) {
    const int t = base + lane;
    int x = t < ntiles ? tiles[t].first_end : INT_MAX;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_down_sync(0xffffffffu, x, o);
      if (lane + o < 32) x = min(x, y);
    }
    const int next = __shfl_down_sync(0xffffffffu, x, 1);
    if (t < ntiles) tiles[t].e_out = min(carry, lane < 31 ? next : INT_MAX);
    carry = min(carry, __shfl_sync(0xffffffffu, x, 0));
  }
  for (int o = 16; o; o >>= 1) {
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    a2 += __shfl_xor_sync(0xffffffffu, a2, o);
  }
  if (lane == 0) {
    State *st = reinterpret_cast<State *>(ws + e.state_offset);
    st->adler = (unsigned)(((N + a2) % 65521) << 16 | ((1 + a1) % 65521));
  }
}

// deflate_rle's symbol at byte p of a run [s, e]: -1 for none, v < 256 a literal, 256 + length - 3 a match
__device__ __forceinline__ int rle_symbol(int p, int s, int e, unsigned char b) {
  const int k = p - s;
  if (k == 0) return b;
  const int j = k - 1, T = e - s, q = T / kMaxMatch, r = T - q * kMaxMatch;
  if (j < kMaxMatch * q) return j % kMaxMatch == 0 ? 256 + kMaxMatch - 3 : -1;
  if (r >= 3) return j == kMaxMatch * q ? 256 + r - 3 : -1;
  return b;
}

template <bool WRITE>
__global__ void __launch_bounds__(kThreads) symbols_kernel(const cpb200_png_encode_image *table, int B,
                                                           unsigned char *ws) {
  __shared__ unsigned char f[kTile + 2];
  __shared__ int sm[kThreads / 32 + 1];
  const int n = find_image<&cpb200_png_encode_image::tile0>(table, B, blockIdx.x);
  const cpb200_png_encode_image e = table[n];
  const int N = (int)filtered_bytes(e);
  const int t = blockIdx.x - e.tile0;
  const int p0 = t * kTile, p1 = min(N, p0 + kTile);
  const unsigned char *src = ws + e.filt_offset;
  Tile *tile = reinterpret_cast<Tile *>(ws + e.tile_offset) + t;
  for (int i = threadIdx.x; i < p1 - p0; i += kThreads) f[i + 1] = src[p0 + i];
  if (threadIdx.x == 0) f[0] = p0 > 0 ? src[p0 - 1] : 0;
  if (threadIdx.x == 1) f[p1 - p0 + 1] = p1 < N ? src[p1] : 0;
  __syncthreads();
  const int q0 = p0 + threadIdx.x * kPerThread, q1 = min(p1, q0 + kPerThread);
  int ls = -1, fe = INT_MAX;
  for (int p = q0; p < q1; ++p) {
    const int i = p - p0 + 1;
    if (p == 0 || f[i] != f[i - 1]) ls = p;
    if (fe == INT_MAX && (p == N - 1 || f[i] != f[i + 1])) fe = p;
  }
  int s = block_exclusive_scan(ls, tile->s_in, MaxOp(), sm);
  int en = block_exclusive_suffix(fe, tile->e_out, MinOp(), sm);
  int ends[kPerThread];
#pragma unroll
  for (int k = kPerThread - 1; k >= 0; --k) {
    const int p = q0 + k;
    if (p < q1) {
      const int i = p - p0 + 1;
      if (p == N - 1 || f[i] != f[i + 1]) en = p;
    }
    ends[k] = en;
  }
  int v[kPerThread];
  int count = 0;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const int p = q0 + k;
    v[k] = -1;
    if (p < q1) {
      const int i = p - p0 + 1;
      if (p == 0 || f[i] != f[i - 1]) s = p;
      v[k] = rle_symbol(p, s, ends[k], f[i]);
      count += v[k] >= 0;
    }
  }
  int total;
  int at = block_exclusive_scan(count, 0, SumOp(), sm, &total);
  if (!WRITE) {
    if (threadIdx.x == 0) tile->nsym = total;
    return;
  }
  unsigned short *sym = reinterpret_cast<unsigned short *>(ws + e.sym_offset) + tile->sym_off;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k)
    if (v[k] >= 0) sym[at++] = (unsigned short)v[k];
}

// one warp per image
__global__ void __launch_bounds__(kThreads) scan_syms_kernel(const cpb200_png_encode_image *table, int B,
                                                             unsigned char *ws) {
  const int n = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= B) return;
  const cpb200_png_encode_image e = table[n];
  const int ntiles = cpb::ceil_div((int)filtered_bytes(e), kTile);
  Tile *tiles = reinterpret_cast<Tile *>(ws + e.tile_offset);
  int carry = 0;
  for (int base = 0; base < ntiles; base += 32) {
    const int t = base + lane;
    int x = t < ntiles ? tiles[t].nsym : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    const int prev = __shfl_up_sync(0xffffffffu, x, 1);
    if (t < ntiles) tiles[t].sym_off = carry + (lane ? prev : 0);
    carry += __shfl_sync(0xffffffffu, x, 31);
  }
  if (lane == 0) {
    State *st = reinterpret_cast<State *>(ws + e.state_offset);
    st->nsym = carry;
    st->nblocks = carry / kBlockSymbols + 1;
  }
}

// ---- zlib's trees.c on one thread, over shared memory ----
struct TreeArrays {
  int freq[HEAP_SIZE];
  unsigned short len[HEAP_SIZE];
  unsigned short dad[HEAP_SIZE];
  unsigned short code[HEAP_SIZE];
};

struct TreeDesc {
  TreeArrays *t;
  int elems, stat;   // stat: 0 none (bl tree), 1 static literal/length lengths, 2 static distance lengths
  const unsigned char *extra;
  int base, max_length, max_code;
};

struct TreeWork {
  TreeArrays l, d, bl;
  int heap[HEAP_SIZE];
  unsigned char depth[HEAP_SIZE];
  int bl_count[MAX_BITS + 1];
  int heap_len, heap_max;
  long long opt_len, static_len;
};

__device__ __forceinline__ int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
__device__ __forceinline__ int static_len_of(int stat, int n) { return stat == 1 ? static_llen(n) : 5; }

__device__ __forceinline__ unsigned bi_reverse(unsigned code, int len) { return __brev(code) >> (32 - len); }

__device__ __forceinline__ bool smaller(const TreeArrays *t, const unsigned char *depth, int n, int m) {
  return t->freq[n] < t->freq[m] || (t->freq[n] == t->freq[m] && depth[n] <= depth[m]);
}

__device__ void pqdownheap(TreeWork &w, const TreeArrays *t, int k) {
  const int v = w.heap[k];
  int j = k << 1;
  while (j <= w.heap_len) {
    if (j < w.heap_len && smaller(t, w.depth, w.heap[j + 1], w.heap[j])) j++;
    if (smaller(t, w.depth, v, w.heap[j])) break;
    w.heap[k] = w.heap[j];
    k = j;
    j <<= 1;
  }
  w.heap[k] = v;
}

__device__ void gen_bitlen(TreeWork &w, const TreeDesc &desc) {
  TreeArrays *t = desc.t;
  for (int b = 0; b <= MAX_BITS; ++b) w.bl_count[b] = 0;
  t->len[w.heap[w.heap_max]] = 0;
  int overflow = 0, h;
  for (h = w.heap_max + 1; h < HEAP_SIZE; h++) {
    const int n = w.heap[h];
    int bits = t->len[t->dad[n]] + 1;
    if (bits > desc.max_length) bits = desc.max_length, overflow++;
    t->len[n] = (unsigned short)bits;
    if (n > desc.max_code) continue;
    w.bl_count[bits]++;
    const int xbits = n >= desc.base ? desc.extra[n - desc.base] : 0;
    const long long f = t->freq[n];
    w.opt_len += f * (bits + xbits);
    if (desc.stat) w.static_len += f * (static_len_of(desc.stat, n) + xbits);
  }
  if (overflow == 0) return;
  do {
    int bits = desc.max_length - 1;
    while (w.bl_count[bits] == 0) bits--;
    w.bl_count[bits]--;
    w.bl_count[bits + 1] += 2;
    w.bl_count[desc.max_length]--;
    overflow -= 2;
  } while (overflow > 0);
  for (int bits = desc.max_length; bits != 0; bits--) {
    int n = w.bl_count[bits];
    while (n != 0) {
      const int m = w.heap[--h];
      if (m > desc.max_code) continue;
      if (t->len[m] != bits) {
        w.opt_len += ((long long)bits - t->len[m]) * t->freq[m];
        t->len[m] = (unsigned short)bits;
      }
      n--;
    }
  }
}

__device__ void gen_codes(TreeArrays *t, int max_code, const int *bl_count) {
  unsigned short next_code[MAX_BITS + 1];
  unsigned code = 0;
  for (int bits = 1; bits <= MAX_BITS; bits++) {
    code = (code + bl_count[bits - 1]) << 1;
    next_code[bits] = (unsigned short)code;
  }
  for (int n = 0; n <= max_code; n++) {
    const int len = t->len[n];
    if (len == 0) continue;
    t->code[n] = (unsigned short)bi_reverse(next_code[len]++, len);
  }
}

__device__ void build_tree(TreeWork &w, TreeDesc &desc) {
  TreeArrays *t = desc.t;
  int max_code = -1;
  w.heap_len = 0;
  w.heap_max = HEAP_SIZE;
  for (int n = 0; n < desc.elems; n++) {
    if (t->freq[n] != 0) {
      w.heap[++w.heap_len] = max_code = n;
      w.depth[n] = 0;
    } else {
      t->len[n] = 0;
    }
  }
  // at least two codes of non-zero frequency
  while (w.heap_len < 2) {
    const int node = w.heap[++w.heap_len] = (max_code < 2 ? ++max_code : 0);
    t->freq[node] = 1;
    w.depth[node] = 0;
    w.opt_len--;
    if (desc.stat) w.static_len -= static_len_of(desc.stat, node);
  }
  desc.max_code = max_code;
  for (int n = w.heap_len / 2; n >= 1; n--) pqdownheap(w, t, n);
  int node = desc.elems;
  do {
    const int n = w.heap[1];
    w.heap[1] = w.heap[w.heap_len--];
    pqdownheap(w, t, 1);
    const int m = w.heap[1];
    w.heap[--w.heap_max] = n;
    w.heap[--w.heap_max] = m;
    t->freq[node] = t->freq[n] + t->freq[m];
    w.depth[node] = (unsigned char)((w.depth[n] >= w.depth[m] ? w.depth[n] : w.depth[m]) + 1);
    t->dad[n] = t->dad[m] = (unsigned short)node;
    w.heap[1] = node++;
    pqdownheap(w, t, 1);
  } while (w.heap_len >= 2);
  w.heap[--w.heap_max] = w.heap[1];
  gen_bitlen(w, desc);
  gen_codes(t, max_code, w.bl_count);
}

// scan_tree (SEND false: count the code-length symbols) and send_tree (SEND true: write them); 0xffff past max_code
// is zlib's guard
template <bool SEND, typename Put>
__device__ void walk_tree(const unsigned char *lens, int max_code, int *bl_freq, const unsigned short *blcode,
                          const unsigned char *bllen, Put &put) {
  int prevlen = -1, nextlen = lens[0], count = 0;
  int max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  auto code = [&](int c) { if (SEND) put(blcode[c], bllen[c]); else bl_freq[c]++; };
  for (int n = 0; n <= max_code; n++) {
    const int curlen = nextlen;
    nextlen = n + 1 <= max_code ? lens[n + 1] : 0xffff;
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      if (SEND) { do code(curlen); while (--count != 0); } else bl_freq[curlen] += count;
    } else if (curlen != 0) {
      if (curlen != prevlen) { code(curlen); count--; }
      code(16);
      if (SEND) put(count - 3, 2);
    } else if (count <= 10) {
      code(17);
      if (SEND) put(count - 3, 3);
    } else {
      code(18);
      if (SEND) put(count - 11, 7);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

struct NoPut { __device__ void operator()(unsigned, int) const {} };

__global__ void __launch_bounds__(kThreads) blocks_kernel(const cpb200_png_encode_image *table, int B,
                                                          unsigned char *ws) {
  __shared__ TreeWork w;
  __shared__ unsigned char lcode_of[256];
  __shared__ long long sm[kThreads / 32 + 1];
  __shared__ unsigned char lens8[L_CODES];
  const int n = find_image<&cpb200_png_encode_image::block0>(table, B, blockIdx.x);
  const cpb200_png_encode_image e = table[n];
  const State *st = reinterpret_cast<const State *>(ws + e.state_offset);
  const int b = blockIdx.x - e.block0;
  if (b >= st->nblocks) return;
  const int nsym_all = (int)st->nsym;
  const int s0 = b * kBlockSymbols, s1 = min(nsym_all, s0 + kBlockSymbols);
  for (int i = threadIdx.x; i < HEAP_SIZE; i += kThreads) { w.l.freq[i] = 0; w.d.freq[i] = 0; w.bl.freq[i] = 0; }
  for (int lc = threadIdx.x; lc < 256; lc += kThreads) {
    int c = 28;
    if (lc < 255) for (c = 27; c_base_length[c] > lc; --c) {}
    lcode_of[lc] = (unsigned char)c;
  }
  __syncthreads();
  const unsigned short *sym = reinterpret_cast<const unsigned short *>(ws + e.sym_offset);
  long long bytes = 0;
  int matches = 0;
  for (int i = s0 + threadIdx.x; i < s1; i += kThreads) {
    const int v = sym[i];
    if (v < 256) { atomicAdd(&w.l.freq[v], 1); bytes += 1; }
    else { atomicAdd(&w.l.freq[257 + lcode_of[v - 256]], 1); matches++; bytes += v - 253; }
  }
  long long mtotal;
  block_exclusive_scan((long long)matches, 0LL, SumOp(), sm, &mtotal);
  long long stored_len;
  block_exclusive_scan(bytes, 0LL, SumOp(), sm, &stored_len);
  Block *blk = reinterpret_cast<Block *>(ws + e.block_offset) + b;
  if (threadIdx.x != 0) return;
  w.l.freq[END_BLOCK] = 1;
  w.d.freq[0] = (int)mtotal;
  w.opt_len = w.static_len = 0;
  TreeDesc ld{&w.l, L_CODES, 1, c_extra_lbits, 257, MAX_BITS, -1};
  TreeDesc dd{&w.d, D_CODES, 2, c_extra_dbits, 0, MAX_BITS, -1};
  TreeDesc bd{&w.bl, BL_CODES, 0, c_extra_blbits, 0, MAX_BL_BITS, -1};
  build_tree(w, ld);
  build_tree(w, dd);
  NoPut np;
  for (int i = 0; i <= ld.max_code; ++i) lens8[i] = (unsigned char)w.l.len[i];
  walk_tree<false>(lens8, ld.max_code, w.bl.freq, nullptr, nullptr, np);
  for (int i = 0; i <= dd.max_code; ++i) lens8[i] = (unsigned char)w.d.len[i];
  walk_tree<false>(lens8, dd.max_code, w.bl.freq, nullptr, nullptr, np);
  build_tree(w, bd);
  int max_blindex;
  for (max_blindex = BL_CODES - 1; max_blindex >= 3; max_blindex--)
    if (w.bl.len[c_bl_order[max_blindex]] != 0) break;
  w.opt_len += 3 * ((long long)max_blindex + 1) + 5 + 5 + 4;
  // _tr_flush_block: the block's start is always in the window here (see centerpose_b200/png.py)
  long long opt_lenb = (w.opt_len + 3 + 7) >> 3;
  const long long static_lenb = (w.static_len + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
  int kind;
  if (stored_len + 4 <= opt_lenb) kind = kStored;
  else if (static_lenb == opt_lenb) kind = kStatic;
  else kind = kDynamic;
  blk->stored_len = stored_len;
  blk->kind = kind;
  blk->nsym = s1 - s0;
  blk->nbits = 3 + (kind == kStatic ? w.static_len : kind == kDynamic ? w.opt_len : 0);
  blk->lcodes = (short)(ld.max_code + 1);
  blk->dcodes = (short)(dd.max_code + 1);
  blk->blcodes = (short)(max_blindex + 1);
  if (kind == kStatic) {
    for (int i = 0; i < L_CODES; ++i) {
      const int len = static_llen(i);
      const unsigned c = i < 144 ? 0x30 + i : i < 256 ? 0x190 + (i - 144) : i < 280 ? i - 256 : 0xC0 + (i - 280);
      blk->lcode[i] = (unsigned short)bi_reverse(c, len);
      blk->llen[i] = (unsigned char)len;
    }
    for (int i = 0; i < D_CODES; ++i) { blk->dcode[i] = (unsigned short)bi_reverse(i, 5); blk->dlen[i] = 5; }
  } else {
    for (int i = 0; i < L_CODES; ++i) {
      const bool used = i <= ld.max_code && w.l.len[i];
      blk->lcode[i] = used ? w.l.code[i] : 0;
      blk->llen[i] = used ? (unsigned char)w.l.len[i] : 0;
    }
    for (int i = 0; i < D_CODES; ++i) {
      const bool used = i <= dd.max_code && w.d.len[i];
      blk->dcode[i] = used ? w.d.code[i] : 0;
      blk->dlen[i] = used ? (unsigned char)w.d.len[i] : 0;
    }
    for (int i = 0; i < BL_CODES; ++i) {
      blk->blcode[i] = w.bl.len[i] ? w.bl.code[i] : 0;
      blk->bllen[i] = (unsigned char)w.bl.len[i];
    }
  }
}

// libpng's zlib header: png_deflate_claim lowers windowBits while n + 262 fits in half the window (n <= 16 KiB),
// zlib writes CMF / FLG at level 1, then optimize_cmf lowers CINFO while n fits in half the window it claims
__device__ void zlib_header(long long n, unsigned char *z) {
  int wb = 15;
  if (n <= 16384) {
    unsigned half = 1u << (wb - 1);
    while (n + 262 <= half) { half >>= 1; --wb; }
  }
  unsigned cmf = ((unsigned)(wb - 8) << 4) | 8;
  if (n <= 16384) {
    unsigned cinfo = cmf >> 4, half = 1u << (cinfo + 7);
    if (n <= half) {
      do { half >>= 1; --cinfo; } while (cinfo > 0 && n <= half);
      cmf = (cinfo << 4) | 8;
    }
  }
  z[0] = (unsigned char)cmf;
  z[1] = (unsigned char)(31 - (cmf << 8) % 31);
}

// one CTA: one warp per image for its blocks, then the files' packed offsets
__global__ void __launch_bounds__(1024) layout_kernel(const cpb200_png_encode_image *table, int B, unsigned char *ws,
                                                      long long *sizes) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int n = warp; n < B; n += nwarps) {
    const cpb200_png_encode_image e = table[n];
    State *st = reinterpret_cast<State *>(ws + e.state_offset);
    Block *blk = reinterpret_cast<Block *>(ws + e.block_offset);
    const int nb = st->nblocks;
    long long pos = 16, byte = 0;   // the deflate data follows the two header bytes
    for (int base = 0; base < nb; base += 32) {
      const int i = base + lane;
      const int kind = i < nb ? blk[i].kind : 0;
      const long long nbits = i < nb ? blk[i].nbits : 0, slen = i < nb ? blk[i].stored_len : 0;
      for (int k = 0; k < 32 && base + k < nb; ++k) {
        const int kk = __shfl_sync(0xffffffffu, kind, k);
        long long bits = __shfl_sync(0xffffffffu, nbits, k);
        const long long sl = __shfl_sync(0xffffffffu, slen, k);
        if (kk == kStored) bits = ((pos + 3 + 7) & ~7LL) - pos + 32 + 8 * sl;
        if (lane == k) { blk[i].bit_off = pos; blk[i].byte_start = byte; blk[i].nbits = bits; }
        pos += bits;
        byte += sl;
      }
    }
    if (lane == 0) {
      unsigned char *z = ws + e.z_offset;
      const long long end = (pos + 7) >> 3;
      zlib_header(filtered_bytes(e), z);
      for (int k = 0; k < 4; ++k) z[end + k] = (unsigned char)(st->adler >> (24 - 8 * k));
      const long long zb = end + 4;
      const int chunks = (int)((zb + kIdat - 1) / kIdat);
      st->zbytes = zb;
      st->nchunks = chunks;
      st->file_bytes = 8 + 25 + 12LL * chunks + zb + 12;
    }
  }
  __syncthreads();
  if (warp == 0) {
    long long carry = 0;
    for (int base = 0; base < B; base += 32) {
      const int n = base + lane;
      State *st = n < B ? reinterpret_cast<State *>(ws + table[n].state_offset) : nullptr;
      const long long v = st ? st->file_bytes : 0;
      long long x = v;
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (st) { st->file_offset = carry + x - v; sizes[n] = v; }
      carry += __shfl_sync(0xffffffffu, x, 31);
    }
  }
}

__device__ __forceinline__ void put_bits(unsigned long long *z, long long pos, unsigned long long v, int nb) {
  if (nb == 0) return;
  const int sh = (int)(pos & 63);
  atomicOr(z + (pos >> 6), v << sh);
  if (sh + nb > 64) atomicOr(z + (pos >> 6) + 1, v >> (64 - sh));
}

__device__ __forceinline__ void put_byte(unsigned char *z, long long at, unsigned v) {
  atomicOr(reinterpret_cast<unsigned *>(z + (at & ~3LL)), v << (8 * (at & 3)));
}

struct StreamPut {
  unsigned long long *z;
  long long pos;
  __device__ void operator()(unsigned v, int nb) { put_bits(z, pos, v, nb); pos += nb; }
};

__global__ void __launch_bounds__(kThreads) emit_kernel(const cpb200_png_encode_image *table, int B,
                                                        unsigned char *ws) {
  __shared__ unsigned short lcode[L_CODES];
  __shared__ unsigned char llen[L_CODES];
  __shared__ unsigned char lcode_of[256];
  __shared__ int sm[kThreads / 32 + 1];
  const int n = find_image<&cpb200_png_encode_image::block0>(table, B, blockIdx.x);
  const cpb200_png_encode_image e = table[n];
  const State *st = reinterpret_cast<const State *>(ws + e.state_offset);
  const int b = blockIdx.x - e.block0;
  const int nb = st->nblocks;
  if (b >= nb) return;
  const Block *blk = reinterpret_cast<const Block *>(ws + e.block_offset) + b;
  unsigned char *z = ws + e.z_offset;
  unsigned long long *z64 = reinterpret_cast<unsigned long long *>(z);
  const int last = b == nb - 1;
  const long long bit_off = blk->bit_off;
  const int kind = blk->kind;
  if (kind == kStored) {
    const long long at = (bit_off + 3 + 7) >> 3;
    const long long len = blk->stored_len;
    if (threadIdx.x == 0) {
      put_bits(z64, bit_off, last, 3);
      put_byte(z, at, len & 0xff);
      put_byte(z, at + 1, (len >> 8) & 0xff);
      put_byte(z, at + 2, ~len & 0xff);
      put_byte(z, at + 3, (~len >> 8) & 0xff);
    }
    const unsigned char *f = ws + e.filt_offset + blk->byte_start;
    for (long long i = threadIdx.x; i < len; i += kThreads) put_byte(z, at + 4 + i, f[i]);
    return;
  }
  for (int i = threadIdx.x; i < L_CODES; i += kThreads) { lcode[i] = blk->lcode[i]; llen[i] = blk->llen[i]; }
  for (int lc = threadIdx.x; lc < 256; lc += kThreads) {
    int c = 28;
    if (lc < 255) for (c = 27; c_base_length[c] > lc; --c) {}
    lcode_of[lc] = (unsigned char)c;
  }
  __syncthreads();
  const unsigned dcode = blk->dcode[0];
  const int dlen = blk->dlen[0];
  const int nsym = blk->nsym, per = cpb::ceil_div(max(nsym, 1), kThreads);
  const unsigned short *sym = reinterpret_cast<const unsigned short *>(ws + e.sym_offset) + (long long)b * kBlockSymbols;
  const int a0 = min(nsym, (int)threadIdx.x * per), a1 = min(nsym, a0 + per);
  auto code_of = [&](int v, unsigned long long &val) -> int {
    if (v < 256) { val = lcode[v]; return llen[v]; }
    const int lc = v - 256, c = lcode_of[lc], xb = c_extra_lbits[c], cl = llen[257 + c];
    const unsigned long long xv = xb ? (unsigned long long)(lc - c_base_length[c]) : 0;
    val = lcode[257 + c] | xv << cl | (unsigned long long)dcode << (cl + xb);
    return cl + xb + dlen;
  };
  int cost = 0;
  for (int i = a0; i < a1; ++i) {
    unsigned long long val;
    cost += code_of(sym[i], val);
  }
  int total;
  const int off = block_exclusive_scan(cost, 0, SumOp(), sm, &total);
  const long long end = bit_off + blk->nbits;
  long long pos = end - llen[END_BLOCK] - total + off;
  for (int i = a0; i < a1; ++i) {
    unsigned long long val;
    const int nbits = code_of(sym[i], val);
    put_bits(z64, pos, val, nbits);
    pos += nbits;
  }
  if (threadIdx.x == 0) {
    put_bits(z64, end - llen[END_BLOCK], lcode[END_BLOCK], llen[END_BLOCK]);
    StreamPut put{z64, bit_off};
    put((kind == kStatic ? 2 : 4) + last, 3);
    if (kind == kDynamic) {
      const int lcodes = blk->lcodes, dcodes = blk->dcodes, blcodes = blk->blcodes;
      put(lcodes - 257, 5);
      put(dcodes - 1, 5);
      put(blcodes - 4, 4);
      for (int r = 0; r < blcodes; ++r) put(blk->bllen[c_bl_order[r]], 3);
      walk_tree<true>(llen, lcodes - 1, nullptr, blk->blcode, blk->bllen, put);
      walk_tree<true>(blk->dlen, dcodes - 1, nullptr, blk->blcode, blk->bllen, put);
    }
  }
}

// zlib's multmodp: a * b modulo the CRC-32 polynomial (reflected)
__device__ uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
  }
  return p;
}

// crc32(A + B) from crc32(A), crc32(B) and len(B) (zlib's crc32_combine)
__device__ uint32_t crc32_combine(uint32_t c1, uint32_t c2, int len2) {
  uint32_t p = 1u << 31;
  for (int k = 3; len2; len2 >>= 1, ++k)
    if (len2 & 1) p = multmodp(c_x2n[k & 31], p);
  return multmodp(p, c1) ^ c2;
}

__device__ __forceinline__ void put_be32(unsigned char *o, uint32_t v) {
  o[0] = (unsigned char)(v >> 24); o[1] = (unsigned char)(v >> 16); o[2] = (unsigned char)(v >> 8); o[3] = (unsigned char)v;
}

constexpr int kAsmWarps = 4;

__global__ void __launch_bounds__(32 * kAsmWarps) assemble_kernel(const cpb200_png_encode_image *table, int B,
                                                                  int chunks, unsigned char *ws, unsigned char *out) {
  __shared__ uint32_t crc_table[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ 0xedb88320u : c >> 1;
    crc_table[i] = c;
  }
  __syncthreads();
  const int g = blockIdx.x * kAsmWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (g >= chunks) return;
  const int n = find_image<&cpb200_png_encode_image::chunk0>(table, B, g);
  const cpb200_png_encode_image e = table[n];
  const State *st = reinterpret_cast<const State *>(ws + e.state_offset);
  const int c = g - e.chunk0;
  if (c >= st->nchunks) return;
  unsigned char *o = out + st->file_offset;
  const unsigned char *z = ws + e.z_offset + (long long)c * kIdat;
  const int len = (int)min((long long)kIdat, st->zbytes - (long long)c * kIdat);
  auto crc_bytes = [&](uint32_t crc, unsigned char v) { return crc_table[(crc ^ v) & 0xff] ^ (crc >> 8); };
  if (c == 0 && lane == 0) {
    const unsigned char head[16] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n', 0, 0, 0, 13, 'I', 'H', 'D', 'R'};
    for (int k = 0; k < 16; ++k) o[k] = head[k];
    put_be32(o + 16, (uint32_t)e.w);
    put_be32(o + 20, (uint32_t)e.h);
    o[24] = 8; o[25] = 2; o[26] = 0; o[27] = 0; o[28] = 0;
    uint32_t crc = 0xffffffffu;
    for (int k = 12; k < 29; ++k) crc = crc_bytes(crc, o[k]);
    put_be32(o + 29, ~crc);
  }
  unsigned char *ch = o + 33 + (long long)c * (kIdat + 12);
  // lane segments of "IDAT" + data, each CRC'd on its own, then combined in lane order
  const int L = 4 + len, seg = cpb::ceil_div(L, 32), i0 = min(L, lane * seg), i1 = min(L, i0 + seg);
  const unsigned char idat[4] = {'I', 'D', 'A', 'T'};
  uint32_t crc = 0xffffffffu;
  for (int i = i0; i < i1; ++i) {
    const unsigned char v = i < 4 ? idat[i] : z[i - 4];
    ch[4 + i] = v;
    crc = crc_bytes(crc, v);
  }
  crc = i1 > i0 ? ~crc : 0u;
  int seglen = i1 - i0;
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t oc = __shfl_down_sync(0xffffffffu, crc, d);
    const int ol = __shfl_down_sync(0xffffffffu, seglen, d);
    if ((lane & (2 * d - 1)) == 0 && lane + d < 32) {
      crc = crc32_combine(crc, oc, ol);
      seglen += ol;
    }
  }
  if (lane == 0) {
    put_be32(ch, (uint32_t)len);
    put_be32(ch + 8 + len, crc);
    if (c == st->nchunks - 1) {
      const unsigned char iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
      for (int k = 0; k < 12; ++k) ch[12 + len + k] = iend[k];
    }
  }
}

}  // namespace

extern "C" int cpb200_png_encode_batch(const cpb200_png_encode_image *table, int B, int tiles, int blocks, int chunks,
                                       void *workspace, unsigned char *out, int64_t *sizes, void *stream) {
  if (!table || !workspace || !out || !sizes || B < 1 || tiles < B || blocks < B || chunks < B)
    return cpb::fail(CPB200_ERR_ARG, "png_encode_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "png_encode_batch: B = %d images exceed one launch (max 65535)", B);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  const unsigned per_warp = (unsigned)cpb::ceil_div(B, kThreads / 32);
  filter_kernel<<<tiles, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode filter_kernel")) return st;
  scan_tiles_kernel<<<per_warp, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode scan_tiles_kernel")) return st;
  symbols_kernel<false><<<tiles, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode symbols_kernel (count)")) return st;
  scan_syms_kernel<<<per_warp, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode scan_syms_kernel")) return st;
  symbols_kernel<true><<<tiles, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode symbols_kernel (write)")) return st;
  blocks_kernel<<<blocks, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode blocks_kernel")) return st;
  layout_kernel<<<1, 1024, 0, s>>>(table, B, ws, reinterpret_cast<long long *>(sizes));
  if (int st = cpb::check_launch("png_encode layout_kernel")) return st;
  emit_kernel<<<blocks, kThreads, 0, s>>>(table, B, ws);
  if (int st = cpb::check_launch("png_encode emit_kernel")) return st;
  assemble_kernel<<<(unsigned)cpb::ceil_div(chunks, kAsmWarps), 32 * kAsmWarps, 0, s>>>(table, B, chunks, ws, out);
  return cpb::check_launch("png_encode assemble_kernel");
}

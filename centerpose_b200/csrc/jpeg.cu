// cpb200_jpeg_decode_batch: cv2.imread(path, IMREAD_COLOR) of sequential- and progressive-Huffman JPEG files on the
// device, byte for byte, for many files per launch.  Four kernels:
//   jpeg_entropy_kernel  sequential images: one CTA per image, one thread per entropy-coded segment (restart interval;
//                        the whole scan without DRI): Huffman decode into de-zigzagged int16 coefficient blocks,
//   jpeg_progressive_kernel  progressive images: one CTA per image runs the scans in file order into the same blocks,
//                        one thread per segment of a scan,
//   jpeg_idct_kernel     dequantise + libjpeg's ISLOW integer IDCT (jidctint.c), 8 threads per block, into 8-bit
//                        component planes padded to whole MCUs; status 1 for a block outside the 16-bit range,
//   jpeg_color_kernel    one thread per output pixel: libjpeg-turbo's fancy upsampling (jdsample.c), integer
//                        YCbCr->BGR (jdcolor.c), and OpenCV's EXIF orientation as an index mapping.
// The host side (centerpose_b200/jpeg.py) parses and checks the headers and builds the table; the kernels trust it.
// An entry with missing_eoi gets status 1 and is not decoded: cv2.imread reads or refuses such files.
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_jpeg_image) == 480, "cpb200_jpeg_image layout is part of the C ABI");
static_assert(sizeof(cpb200_jpeg_scan) == 40, "cpb200_jpeg_scan layout is part of the C ABI");
static_assert(sizeof(cpb200_jpeg_huff) == 1424, "cpb200_jpeg_huff layout is part of the C ABI");

__constant__ unsigned char kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                          12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                          35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                          58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// per-image geometry derived from the table entry
struct Geo {
  int mcux, mcuy;      // MCUs per row / column
  int bw[3], bh[3];    // blocks per row / block rows of each component (whole MCUs)
  int64_t base[3];     // first block of each component
  int64_t nblk;        // blocks of all components
};

__device__ __forceinline__ Geo geometry(const cpb200_jpeg_image &e) {
  Geo g;
  g.mcux = (e.w + 8 * e.hs - 1) / (8 * e.hs);
  g.mcuy = (e.h + 8 * e.vs - 1) / (8 * e.vs);
  g.bw[0] = g.mcux * e.hs; g.bh[0] = g.mcuy * e.vs;
  g.bw[1] = g.bw[2] = g.mcux; g.bh[1] = g.bh[2] = g.mcuy;
  g.nblk = 0;
  for (int c = 0; c < 3; ++c) {
    g.base[c] = g.nblk;
    if (c < e.ncomp) g.nblk += (int64_t)g.bw[c] * g.bh[c];
  }
  return g;
}

// a[c] by selects, so the per-component arrays stay in registers
template <typename T>
__device__ __forceinline__ T pick(const T (&a)[3], int c) { return c == 0 ? a[0] : c == 1 ? a[1] : a[2]; }

// the image's coefficients (128 bytes per block) and planes (64 bytes per block) lie inside the workspace
__device__ __forceinline__ bool fits(const cpb200_jpeg_image &e, const Geo &g, size_t ws_bytes) {
  return e.coef_offset >= 0 && e.plane_offset >= 0 && (uint64_t)e.coef_offset + (uint64_t)g.nblk * 128 <= ws_bytes &&
         (uint64_t)e.plane_offset + (uint64_t)g.nblk * 64 <= ws_bytes;
}

// MSB-first bit reader over one segment: skips stuffed zero bytes, stops at a marker or the segment's end and feeds
// zeros from there; `real` counts the bits that came from the file, `used` the bits consumed
struct Bits {
  const unsigned char *src;
  int64_t p, end;
  uint64_t acc;
  int n;
  int64_t real, used;

  __device__ __forceinline__ void fill() {
    while (n <= 56) {
      unsigned b = 0;
      if (p < end) {
        b = src[p];
        if (b != 0xFF) {
          ++p; real += 8;
        } else if (p + 1 < end && src[p + 1] == 0) {
          p += 2; real += 8;
        } else {
          p = end; b = 0;
        }
      }
      acc |= (uint64_t)b << (56 - n);
      n += 8;
    }
  }
  __device__ __forceinline__ void skip(int k) { acc <<= k; n -= k; used += k; }
  // Huffman symbol, or -1 for a code longer than 16 bits
  __device__ __forceinline__ int symbol(const cpb200_jpeg_huff *__restrict__ t) {
    fill();
    const unsigned e = __ldg(&t->lut[acc >> 55]);
    if (e) { skip(e >> 8); return e & 255; }
    int l = 10;
    while (l <= 16 && (int)(acc >> (64 - l)) > __ldg(&t->maxcode[l])) ++l;
    if (l > 16) return -1;
    const int i = (int)(acc >> (64 - l)) + __ldg(&t->valoff[l]);
    if (i < 0 || i > 255) return -1;
    skip(l);
    return __ldg(&t->val[i]);
  }
  // the next s (<= 15) bits as a signed coefficient (T.81 F.2.2.1 EXTEND)
  __device__ __forceinline__ int receive(int s) {
    if (!s) return 0;
    const int v = (int)(acc >> (64 - s));
    skip(s);
    return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v;
  }
  // the next k (1..16) bits, unsigned
  __device__ __forceinline__ int get(int k) {
    fill();
    const int v = (int)(acc >> (64 - k));
    skip(k);
    return v;
  }
};

// grid B CTAs x 32 threads: CTA b decodes image b, its threads stride over the image's segments
__global__ void __launch_bounds__(32) jpeg_entropy_kernel(const unsigned char *__restrict__ src,
                                                          const cpb200_jpeg_image *__restrict__ table,
                                                          unsigned char *__restrict__ ws, size_t ws_bytes,
                                                          int *__restrict__ status) {
  const cpb200_jpeg_image &e = table[blockIdx.x];
  if (e.nscan) return;                                      // progressive: jpeg_progressive_kernel
  const Geo g = geometry(e);
  if (!fits(e, g, ws_bytes)) {
    if (threadIdx.x == 0) status[blockIdx.x] = 2;
    return;
  }
  if (e.missing_eoi) {                                      // cv2.imread decides these files
    if (threadIdx.x == 0) status[blockIdx.x] = 1;
    return;
  }
  if (threadIdx.x == 0) status[blockIdx.x] = 0;
  __syncthreads();
  const int64_t total = (int64_t)g.mcux * g.mcuy;
  const int64_t ri = e.restart_interval ? e.restart_interval : total;
  const int64_t *seg = reinterpret_cast<const int64_t *>(src + e.seg_offset);
  const cpb200_jpeg_huff *huff = reinterpret_cast<const cpb200_jpeg_huff *>(src + e.huff_offset);
  short *coef = reinterpret_cast<short *>(ws + e.coef_offset);
  const int units = e.ncomp == 3 ? e.hs * e.vs + 2 : 1;
  for (int s = threadIdx.x; s < e.nseg; s += blockDim.x) {
    Bits r{src, seg[2 * s], seg[2 * s + 1], 0ull, 0, 0, 0};
    int pred0 = 0, pred1 = 0, pred2 = 0;
    const int64_t m1 = min((int64_t)(s + 1) * ri, total);
    for (int64_t m = (int64_t)s * ri; m < m1; ++m) {
      const int my = (int)(m / g.mcux), mx = (int)(m - (int64_t)my * g.mcux);
      for (int u = 0; u < units; ++u) {
        const int c = u < units - 2 || e.ncomp == 1 ? 0 : u - (units - 2) + 1;
        const int dy = c ? 0 : u / e.hs, dx = c ? 0 : u % e.hs;
        const int hs = c ? 1 : e.hs, vs = c ? 1 : e.vs;
        short *blk = coef + (pick(g.base, c) + (int64_t)(my * vs + dy) * pick(g.bw, c) + mx * hs + dx) * 64;
        int4 *b4 = reinterpret_cast<int4 *>(blk);
#pragma unroll
        for (int k = 0; k < 8; ++k) b4[k] = make_int4(0, 0, 0, 0);
        int sym = r.symbol(huff + e.dc_tbl[c]);
        if (sym < 0) goto bad;
        const int dc = r.receive(sym) + (c == 0 ? pred0 : c == 1 ? pred1 : pred2);
        if (c == 0) pred0 = dc; else if (c == 1) pred1 = dc; else pred2 = dc;
        blk[0] = (short)dc;
        const cpb200_jpeg_huff *ac = huff + e.ac_tbl[c];
        for (int k = 1; k < 64;) {
          sym = r.symbol(ac);
          if (sym < 0) goto bad;
          const int run = sym >> 4, sz = sym & 15;
          if (sz) {
            k += run;
            if (k > 63) goto bad;
            blk[kZigzag[k]] = (short)r.receive(sz);
            ++k;
          } else if (run == 15) {
            k += 16;
          } else {
            break;
          }
        }
      }
      if (r.used > r.real) goto bad;                        // the segment's data ended before this MCU did
    }
    continue;
  bad:
    status[blockIdx.x] = 1;
    return;
  }
}

// AC refinement of one coefficient with nonzero history: a correction bit adds p1 (or m1 below zero) unless that bit is
// already set; the sum is stored to 16 bits as libjpeg's JCOEF
__device__ __forceinline__ void refine(short *cf, Bits &r, int p1, int m1) {
  if (r.get(1) && !(*cf & p1)) *cf = (short)(*cf >= 0 ? *cf + p1 : *cf + m1);
}

// One restart segment of a progressive scan, units [u0, u1), as libjpeg-turbo's jdphuff.c decodes T.81 G.1.2: DC first
// (difference << Al), DC refinement (one bit), AC first (EOBRUN runs of empty blocks), AC refinement (correction bits
// on coefficients with nonzero history; zero runs and EOBRUN count only zero-history coefficients).  A unit is an MCU
// when the scan has several components, else one block of the component's own grid, `cbw` blocks per row.  Returns
// false on a code longer than 16 bits, a run past Se, a refinement size other than 0 or 1, or data ending before the
// segment's last unit.
__device__ __forceinline__ bool progressive_segment(const cpb200_jpeg_scan &s, const cpb200_jpeg_image &e, const Geo &g,
                                                    short *coef,
                                                    const cpb200_jpeg_huff *__restrict__ huff, Bits &r, int64_t u0,
                                                    int64_t u1, int cbw) {
  const int ss = s.ss, se = s.se, al = s.al, nc = s.ncomp;
  const int p1 = 1 << al, m1 = -p1;
  const int kind = ss == 0 ? (s.ah == 0 ? 0 : 1) : (s.ah == 0 ? 2 : 3);
  const cpb200_jpeg_huff *ac = huff + s.ac_tbl[0];
  int pred0 = 0, pred1 = 0, pred2 = 0, eobrun = 0;
  for (int64_t u = u0; u < u1; ++u) {
    const int uw = nc > 1 ? g.mcux : cbw;
    const int uy = (int)(u / uw), ux = (int)(u - (int64_t)uy * uw);
    for (int i = 0; i < nc; ++i) {
      const int c = s.comp[i];
      const int hs = nc > 1 && c == 0 ? e.hs : 1, vs = nc > 1 && c == 0 ? e.vs : 1;
      for (int b = 0; b < hs * vs; ++b) {
        short *blk = coef + (pick(g.base, c) + (int64_t)(uy * vs + b / hs) * pick(g.bw, c) + ux * hs + b % hs) * 64;
        if (kind == 0) {                                      // DC first
          const int sym = r.symbol(huff + s.dc_tbl[i]);
          if (sym < 0) return false;
          const int dc = r.receive(sym) + (i == 0 ? pred0 : i == 1 ? pred1 : pred2);
          if (i == 0) pred0 = dc; else if (i == 1) pred1 = dc; else pred2 = dc;
          blk[0] = (short)((unsigned)dc << al);
        } else if (kind == 1) {                               // DC refinement
          if (r.get(1)) blk[0] = (short)(blk[0] | p1);
        } else if (kind == 2) {                               // AC first
          if (eobrun) { --eobrun; continue; }
          for (int k = ss; k <= se; ++k) {
            const int sym = r.symbol(ac);
            if (sym < 0) return false;
            const int run = sym >> 4, sz = sym & 15;
            if (sz) {
              k += run;
              if (k > se) return false;
              blk[kZigzag[k]] = (short)((unsigned)r.receive(sz) << al);
            } else if (run == 15) {
              k += 15;
            } else {
              eobrun = (1 << run) - 1;
              if (run) eobrun += r.get(run);
              break;
            }
          }
        } else {                                              // AC refinement
          int k = ss;
          if (!eobrun) {
            for (; k <= se; ++k) {
              const int sym = r.symbol(ac);
              if (sym < 0) return false;
              int run = sym >> 4, v = 0;
              const int sz = sym & 15;
              if (sz) {
                if (sz != 1) return false;
                v = r.get(1) ? p1 : m1;
              } else if (run != 15) {
                eobrun = 1 << run;
                if (run) eobrun += r.get(run);
                break;
              }
              for (; k <= se; ++k) {
                short *cf = blk + kZigzag[k];
                if (*cf) refine(cf, r, p1, m1);
                else if (--run < 0) break;
              }
              if (v) {
                if (k > se) return false;
                blk[kZigzag[k]] = (short)v;
              }
            }
          }
          if (eobrun) {
            for (; k <= se; ++k) {
              short *cf = blk + kZigzag[k];
              if (*cf) refine(cf, r, p1, m1);
            }
            --eobrun;
          }
        }
      }
    }
    if (r.used > r.real) return false;                      // the segment's data ended before this unit did
  }
  return true;
}

// grid B CTAs x 32 threads: CTA b zeroes image b's coefficients, then runs its scans in file order, its threads
// striding over each scan's segments; sequential images return at once.  The minimum of one block per SM lets ptxas
// use the 90 registers the four decoders need (it caps the plain bound at 64 and spills)
__global__ void __launch_bounds__(32, 1) jpeg_progressive_kernel(const unsigned char *__restrict__ src,
                                                                 const cpb200_jpeg_image *__restrict__ table,
                                                                 unsigned char *__restrict__ ws, size_t ws_bytes,
                                                                 int *__restrict__ status) {
  __shared__ int failed;
  const cpb200_jpeg_image &e = table[blockIdx.x];
  if (!e.nscan) return;
  const Geo g = geometry(e);
  if (!fits(e, g, ws_bytes)) {
    if (threadIdx.x == 0) status[blockIdx.x] = 2;
    return;
  }
  if (e.missing_eoi) {                                      // cv2.imread decides these files
    if (threadIdx.x == 0) status[blockIdx.x] = 1;
    return;
  }
  if (threadIdx.x == 0) {
    status[blockIdx.x] = 0;
    failed = 0;
  }
  int4 *z = reinterpret_cast<int4 *>(ws + e.coef_offset);
  for (int64_t i = threadIdx.x; i < g.nblk * 8; i += blockDim.x) z[i] = make_int4(0, 0, 0, 0);
  __syncthreads();
  const cpb200_jpeg_scan *scans = reinterpret_cast<const cpb200_jpeg_scan *>(src + e.scan_offset);
  const cpb200_jpeg_huff *huff = reinterpret_cast<const cpb200_jpeg_huff *>(src + e.huff_offset);
  short *coef = reinterpret_cast<short *>(ws + e.coef_offset);
  for (int n = 0; n < e.nscan; ++n) {
    const cpb200_jpeg_scan &s = scans[n];
    // one component: its own block grid, which for luma sampled (2, x) can be a column / row short of whole MCUs
    const int c = s.comp[0], hs = c == 0 ? e.hs : 1, vs = c == 0 ? e.vs : 1;
    const int cbw = ((e.w * hs + e.hs - 1) / e.hs + 7) / 8, cbh = ((e.h * vs + e.vs - 1) / e.vs + 7) / 8;
    const int64_t total = s.ncomp > 1 ? (int64_t)g.mcux * g.mcuy : (int64_t)cbw * cbh;
    const int64_t ri = s.restart_interval ? s.restart_interval : total;
    const int64_t *seg = reinterpret_cast<const int64_t *>(src + s.seg_offset);
    for (int q = threadIdx.x; q < s.nseg; q += blockDim.x) {
      Bits r{src, seg[2 * q], seg[2 * q + 1], 0ull, 0, 0, 0};
      if (!progressive_segment(s, e, g, coef, huff, r, (int64_t)q * ri, min((int64_t)(q + 1) * ri, total), cbw)) {
        status[blockIdx.x] = 1;
        failed = 1;
        break;
      }
    }
    __syncthreads();                                        // the next scan refines what this one wrote
    if (failed) return;
  }
}

// libjpeg's jpeg_idct_islow, one pass over 8 values: CONST_BITS 13, outputs descaled by `shift`
__device__ __forceinline__ void idct8(const int (&x)[8], int (&o)[8], int shift) {
  int z2 = x[2], z3 = x[6];
  int z1 = (z2 + z3) * 4433;                                  // FIX_0_541196100
  const int t2 = z1 - z3 * 15137, t3 = z1 + z2 * 6270;        // FIX_1_847759065, FIX_0_765366865
  const int t0 = (x[0] + x[4]) * 8192, t1 = (x[0] - x[4]) * 8192;
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  int a0 = x[7], a1 = x[5], a2 = x[3], a3 = x[1];
  z1 = a0 + a3; z2 = a1 + a2; z3 = a0 + a2;
  int z4 = a1 + a3;
  const int z5 = (z3 + z4) * 9633;                            // FIX_1_175875602
  a0 *= 2446; a1 *= 16819; a2 *= 25172; a3 *= 12299;          // 0.298631336 2.053119869 3.072711026 1.501321110
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;   // 0.899976223 2.562915447 1.961570560 0.390180644
  a0 += z1 + z3; a1 += z2 + z4; a2 += z2 + z3; a3 += z1 + z4;
  const int rnd = 1 << (shift - 1);
  o[0] = (t10 + a3 + rnd) >> shift; o[7] = (t10 - a3 + rnd) >> shift;
  o[1] = (t11 + a2 + rnd) >> shift; o[6] = (t11 - a2 + rnd) >> shift;
  o[2] = (t12 + a1 + rnd) >> shift; o[5] = (t12 - a1 + rnd) >> shift;
  o[3] = (t13 + a0 + rnd) >> shift; o[4] = (t13 - a0 + rnd) >> shift;
}

// a dequantised coefficient or pass-1 output beyond this is flagged (jpeg.IDCT_RANGE): below it every sum and product
// of libjpeg-turbo's 16-bit SIMD IDCT fits int16, so its saturating and wrapping arithmetic agrees with these 32-bit
// passes; no encoder writes such blocks, corrupt or hostile files can
constexpr int kIdctRange = 16383;

// grid (block groups, image) x 256 threads: 8 lanes per 8x8 block, lane r takes column r (pass 1, through shared
// memory) then row r (pass 2); the warps of an image stride over all its blocks, 4 per warp at a time.  A block with a
// value outside +-kIdctRange sets the image's status to 1 (the caller decodes it on the host)
__global__ void __launch_bounds__(256) jpeg_idct_kernel(const cpb200_jpeg_image *__restrict__ table,
                                                        unsigned char *__restrict__ ws, size_t ws_bytes,
                                                        int *__restrict__ status) {
  __shared__ int sh[8][4][64];
  const cpb200_jpeg_image &e = table[blockIdx.y];
  const Geo g = geometry(e);
  if (!fits(e, g, ws_bytes) || e.missing_eoi) return;
  const short *coef = reinterpret_cast<const short *>(ws + e.coef_offset);
  unsigned char *planes = ws + e.plane_offset;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, grp = lane >> 3, r = lane & 7;
  const int64_t step = (int64_t)gridDim.x * 8 * 4;
  for (int64_t base = ((int64_t)blockIdx.x * 8 + warp) * 4; base < g.nblk; base += step) {
    const int64_t blk = base + grp;
    const bool active = blk < g.nblk;
    int c = 0;
    if (active) {
      c = blk >= g.base[2] && e.ncomp == 3 ? 2 : blk >= g.base[1] && e.ncomp == 3 ? 1 : 0;
      int x[8], o[8];
      bool out = false;
#pragma unroll
      for (int k = 0; k < 8; ++k) {   // flagged blocks go on with the 16-bit product, so no 32-bit sum overflows
        const int p = coef[blk * 64 + k * 8 + r] * e.qt[c][k * 8 + r];
        out |= abs(p) > kIdctRange;
        x[k] = (short)p;
      }
      idct8(x, o, 11);                                        // CONST_BITS - PASS1_BITS
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        sh[warp][grp][k * 8 + r] = o[k];
        out |= abs(o[k]) > kIdctRange;
      }
      if (out) status[blockIdx.y] = 1;
    }
    __syncwarp();
    if (active) {
      int x[8], o[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) x[k] = sh[warp][grp][r * 8 + k];
      idct8(x, o, 18);                                        // CONST_BITS + PASS1_BITS + 3
      const int64_t cbase = pick(g.base, c), li = blk - cbase;
      const int bw = pick(g.bw, c);
      const int by = (int)(li / bw), bx = (int)(li - (int64_t)by * bw);
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        lo |= (uint32_t)min(max(o[k] + 128, 0), 255) << (8 * k);
        hi |= (uint32_t)min(max(o[k + 4] + 128, 0), 255) << (8 * k);
      }
      *reinterpret_cast<uint2 *>(planes + cbase * 64 + (int64_t)(by * 8 + r) * bw * 8 + bx * 8) = make_uint2(lo, hi);
    }
    __syncwarp();
  }
}

// chroma sample of a (1, 1)-sampled plane at full-resolution (y, x), as libjpeg-turbo's upsamplers: fancy h2v1 / h2v2
// triangle filters with their alternating biases (plain box replication when the plane is at most 2 samples wide),
// fancy h1v2; edge columns and the context rows above the first and below the last real row repeat that row / column
__device__ __forceinline__ int chroma(const unsigned char *__restrict__ P, int pitch, int cw, int ch, int hs, int vs,
                                      int y, int x) {
  if (hs == 1 && vs == 1) return P[(int64_t)y * pitch + x];
  if (hs == 2 && cw <= 2) return P[(int64_t)(y / vs) * pitch + (x >> 1)];
  if (vs == 2) {
    const int k = y >> 1, f = (y & 1) ? min(k + 1, ch - 1) : max(k - 1, 0);
    const unsigned char *near = P + (int64_t)k * pitch, *far = P + (int64_t)f * pitch;
    if (hs == 1) return (3 * near[x] + far[x] + ((y & 1) ? 2 : 1)) >> 2;
    const int j = x >> 1, j2 = (x & 1) ? min(j + 1, cw - 1) : max(j - 1, 0);
    const int c0 = 3 * near[j] + far[j], c1 = 3 * near[j2] + far[j2];
    return (3 * c0 + c1 + ((x & 1) ? 7 : 8)) >> 4;
  }
  const unsigned char *row = P + (int64_t)y * pitch;
  const int j = x >> 1, j2 = (x & 1) ? min(j + 1, cw - 1) : max(j - 1, 0);
  return (3 * row[j] + row[j2] + ((x & 1) ? 2 : 1)) >> 2;
}

// grid (pixel blocks, image) x 256 threads: one thread per output pixel in row-major order of the oriented image
__global__ void __launch_bounds__(256) jpeg_color_kernel(const cpb200_jpeg_image *__restrict__ table,
                                                         const unsigned char *__restrict__ ws, size_t ws_bytes,
                                                         unsigned char *__restrict__ dst) {
  const cpb200_jpeg_image &e = table[blockIdx.y];
  const Geo g = geometry(e);
  if (!fits(e, g, ws_bytes) || e.missing_eoi) return;
  const int h = e.h, w = e.w, o = e.orientation;
  const int ow = o >= 5 ? h : w;
  const int64_t total = (int64_t)h * w;
  const unsigned char *P0 = ws + e.plane_offset;
  const unsigned char *P1 = P0 + g.base[1] * 64, *P2 = P0 + g.base[2] * 64;
  const int cw = (w + e.hs - 1) / e.hs, ch = (h + e.vs - 1) / e.vs;
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
    const int y = P0[(int64_t)sy * g.bw[0] * 8 + sx];
    int b = y, gg = y, r = y;
    if (e.ncomp == 3) {
      const int cb = chroma(P1, g.bw[1] * 8, cw, ch, e.hs, e.vs, sy, sx) - 128;
      const int cr = chroma(P2, g.bw[2] * 8, cw, ch, e.hs, e.vs, sy, sx) - 128;
      // jdcolor.c: 16-bit fixed point, ONE_HALF rounding, arithmetic shifts
      r = y + ((91881 * cr + 32768) >> 16);
      gg = y + ((-46802 * cr - 22554 * cb + 32768) >> 16);
      b = y + ((116130 * cb + 32768) >> 16);
    }
    unsigned char *px = out + i * 3;
    px[0] = (unsigned char)min(max(b, 0), 255);
    px[1] = (unsigned char)min(max(gg, 0), 255);
    px[2] = (unsigned char)min(max(r, 0), 255);
  }
}

}  // namespace

extern "C" int cpb200_jpeg_decode_batch(const unsigned char *src, const cpb200_jpeg_image *table, int B, void *workspace,
                                        size_t workspace_bytes, unsigned char *dst, int *status, void *stream) {
  if (!src || !table || !workspace || !dst || !status || B < 1)
    return cpb::fail(CPB200_ERR_ARG, "jpeg_decode_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "jpeg_decode_batch: B = %d images exceed one launch (max 65535)", B);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  jpeg_entropy_kernel<<<B, 32, 0, st>>>(src, table, ws, workspace_bytes, status);
  int rc = cpb::check_launch("jpeg_entropy_kernel");
  if (rc) return rc;
  jpeg_progressive_kernel<<<B, 32, 0, st>>>(src, table, ws, workspace_bytes, status);
  rc = cpb::check_launch("jpeg_progressive_kernel");
  if (rc) return rc;
  // the sizes live on the device: enough blocks per image to fill the GPU for one large image, fewer as B grows
  const dim3 grid((unsigned)std::max(1, 132 * 8 / B), (unsigned)B);
  jpeg_idct_kernel<<<grid, 256, 0, st>>>(table, ws, workspace_bytes, status);
  rc = cpb::check_launch("jpeg_idct_kernel");
  if (rc) return rc;
  jpeg_color_kernel<<<grid, 256, 0, st>>>(table, ws, workspace_bytes, dst);
  return cpb::check_launch("jpeg_color_kernel");
}

// wgmma 3x3 / stride-1 / pad-1 convolution with HALO REUSE (bf16 NHWC, fp32 accumulate in registers).
//
// The tap-per-stage kernel (net_tc.cu) fetches nine shifted 128-pixel windows per tile and channel
// slab: 9 x 128 row requests through L2 for data that overlaps 89 %.  Here ONE (16+2) x (8+2) halo
// box per slab is brought in by TMA (180 pixel rows) and all nine taps read it in place through
// shifted wgmma shared-memory descriptors:
//     tile = 16 rows x 8 columns of output pixels  ->  A row m = (th, tw) = (m / 8, m % 8);
//     every 8-row core-matrix group of the A operand is therefore one tile row, so tap (r, s) is
//         start address = halo + ((r * 10 + s) * pixel_bytes)      (+ 32 B per K step of 16)
//         stride between 8-row groups (SBO) = 10 * pixel_bytes     (one halo row of pixels)
// which is NOT a multiple of the 1024-byte swizzle repeat; it works because the hardware applies the
// 128B/64B/32B swizzle XOR to absolute shared-memory address bits.  The second consumer warpgroup's 64 rows
// start 8 halo rows later.  TMA's out-of-bounds zero fill provides the conv padding for the halo border.
//
// Weights: slab-major [tap][K-slab][Cout_pad][BK] bf16 via 3-D TMA; when the whole filter bank fits beside the halo
// ring it is loaded ONCE per CTA and stays resident (e.g. 64->64: 72 KB), otherwise it streams
// through its own ring.  Warps: 0-7 = two consumer warpgroups (wgmma + epilogue), 8 = halo producer, 9 = weight
// producer; persistent CTAs.
//
// Split-operand precisions (P = 2, act_dtype CPB200_BF16X2 / CPB200_F16X2; tc_common.cuh): activations and weights arrive
// as hi / lo 16-bit planes.  The halo ring is plane-granular (the planes of a slab are two consecutive stages, TMA batch
// coordinate n and n + B); a weight stage holds the hi tile immediately followed by the lo tile (tc::mma_stage,
// tc::epilogue_pair).
#include <type_traits>
#include "tc_common.cuh"
#include <memory>

using namespace tc;

namespace {

constexpr int C3_CONS = 256;                  // two consumer warpgroups
constexpr int C3_THREADS = C3_CONS + 64;      // + halo producer warp + weight producer warp
constexpr int TW = 8, TH = 16;
constexpr int MAX_NA = 16, MAX_NB = 8;

struct alignas(64) C3Args {
  CUtensorMap amap, bmap;
  int cin, slabs, BK;
  int B, Ho, Wo, tiles_h, tiles_w, n_tiles, total_tiles;
  int cout, cout_store;
  int na, nb, b_resident;
  int kh, kw, taps, hw;        // filter size, kh*kw, halo width in pixels (TW + kw - 1)
  unsigned a_stage_bytes, b_stage_bytes, a_tx_bytes, b_tx_bytes;
  void *dst;
  const void *res;
  const float *bias;
  unsigned flags, swizzle_bits;
  // split-operand mode (P = 2)
  unsigned fmt;                // 0 = bf16 planes, 1 = fp16 planes
  float acc_scale;             // accumulator multiplier (inverse of the host's power-of-two weight scale)
  long long dst_plane;         // elements between the hi and lo planes of dst / res
  unsigned b_tile_bytes;       // bytes of one weight tile (BN x BK x 2); a P = 2 weight stage is [hi tile | lo tile]
};

template <int BN, int P>
__global__ void __launch_bounds__(C3_THREADS, 1) conv3x3_tc_kernel(const __grid_constant__ C3Args a) {
  static_assert(P == 1 || BN <= 128, "split operands: two BN-column accumulators per thread");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base, b_base = smem_base + a.na * a.a_stage_bytes;
  __shared__ __align__(8) uint64_t bars[2 * MAX_NA + 2 * MAX_NB + 1];
  const uint32_t afull0 = smem_u32(&bars[0]), aempty0 = smem_u32(&bars[MAX_NA]);
  const uint32_t bfull0 = smem_u32(&bars[2 * MAX_NA]), bempty0 = smem_u32(&bars[2 * MAX_NA + MAX_NB]);
  const uint32_t ball = smem_u32(&bars[2 * MAX_NA + 2 * MAX_NB]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == C3_CONS) {
    tmap_prefetch(&a.amap); tmap_prefetch(&a.bmap);
    for (int s = 0; s < MAX_NA; ++s) { mbar_init(afull0 + 8 * s, 1); mbar_init(aempty0 + 8 * s, C3_CONS / 32); }
    for (int s = 0; s < MAX_NB; ++s) { mbar_init(bfull0 + 8 * s, 1); mbar_init(bempty0 + 8 * s, C3_CONS / 32); }
    mbar_init(ball, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t pix_bytes = a.BK * 2;

  auto tile_at = [&](int it, int &n, int &h0, int &w0, int &nt) -> bool {
    int t = blockIdx.x + it * gridDim.x;
    if (t >= a.total_tiles) return false;
    nt = t % a.n_tiles; int pt = t / a.n_tiles;
    const int tw = pt % a.tiles_w; pt /= a.tiles_w;
    const int th = pt % a.tiles_h; n = pt / a.tiles_h;
    h0 = th * TH; w0 = tw * TW;
    return true;
  };

  if (warp == C3_CONS / 32) {
    // =============================== halo producer ===============================
    if (elect_one()) {
      int sa = 0; uint32_t pha = 0;
      int n, h0, w0, nt;
      for (int it = 0; tile_at(it, n, h0, w0, nt); ++it) {
        for (int sl = 0; sl < a.slabs; ++sl) {
#pragma unroll
          for (int pl = 0; pl < P; ++pl) {                 // plane-granular stages: hi then lo (batch coordinate n + B)
            mbar_wait(aempty0 + 8 * sa, pha ^ 1);
            mbar_expect_tx(afull0 + 8 * sa, a.a_tx_bytes);
            tma_load_4d(a_base + sa * a.a_stage_bytes, &a.amap, afull0 + 8 * sa, sl * a.BK, w0 - (a.kw >> 1), h0 - (a.kh >> 1), n + pl * a.B);
            if (++sa == a.na) { sa = 0; pha ^= 1; }
          }
        }
      }
    }
  } else if (warp == C3_CONS / 32 + 1) {
    // =============================== weight producer ===============================
    if (elect_one()) {
      const int wplane = a.taps * a.slabs;                 // weight blocks per plane
      if (a.b_resident) {
        mbar_expect_tx(ball, (uint32_t)P * a.taps * a.slabs * a.b_tx_bytes);
        for (int sl = 0; sl < a.slabs; ++sl)
          for (int tap = 0; tap < a.taps; ++tap)
#pragma unroll
            for (int pl = 0; pl < P; ++pl)
              tma_load_3d(b_base + (sl * a.taps + tap) * a.b_stage_bytes + pl * a.b_tile_bytes, &a.bmap, ball, 0, 0,
                          pl * wplane + tap * a.slabs + sl);
      } else {
        int sb = 0; uint32_t phb = 0;
        int n, h0, w0, nt;
        for (int it = 0; tile_at(it, n, h0, w0, nt); ++it) {
          for (int sl = 0; sl < a.slabs; ++sl)
            for (int tap = 0; tap < a.taps; ++tap) {
              mbar_wait(bempty0 + 8 * sb, phb ^ 1);
              mbar_expect_tx(bfull0 + 8 * sb, P * a.b_tile_bytes);
#pragma unroll
              for (int pl = 0; pl < P; ++pl)
                tma_load_3d(b_base + sb * a.b_stage_bytes + pl * a.b_tile_bytes, &a.bmap, bfull0 + 8 * sb, 0, nt * BN,
                            pl * wplane + tap * a.slabs + sl);
              if (++sb == a.nb) { sb = 0; phb ^= 1; }
            }
        }
      }
    }
  } else if (warp < C3_CONS / 32) {
    // =============================== consumers: wgmma + epilogue ===============================
    // Per slab the halo plane(s) are waited for once, then every tap issues its products.  Streamed weights: one weight stage
    // per (slab, tap), released once the MMAs of the next one are queued; resident weights: nothing to wait for but the halo.
    // The halo stages of a slab are released after its last tap.
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const uint32_t bf = (P == 1 || a.fmt == 0) ? 1u : 0u;
    const int ksteps = a.BK / 16;
    const uint64_t dA = desc_sbo(0u, a.hw * pix_bytes, a.swizzle_bits), dB = desc_sbo(0u, 8 * pix_bytes, a.swizzle_bits);
    const uint32_t pstep = pix_bytes >> 4;
    const uint32_t a_lo14 = ((a_base & 0x3FFFFu) >> 4) + (uint32_t)wg * 8u * (uint32_t)a.hw * pstep;   // 8 halo rows per warpgroup
    const uint32_t b_lo14 = (b_base & 0x3FFFFu) >> 4;
    const uint32_t astep = a.a_stage_bytes >> 4, bstep = a.b_stage_bytes >> 4, rowstep = (uint32_t)a.hw * pstep;
    const uint32_t btile = a.b_tile_bytes >> 4;                                  // W_lo follows W_hi in a weight stage
    const uint32_t act = a.flags & CPB_ACT_MASK;
    const int form = (a.flags & CPB200_FLAG_OUT_F32) ? OUT_F32 : OUT_16;      // c3_eligible: no NCHW output
    float acc[BN / 2], acc2[P == 2 ? BN / 2 : 1];
    acc_zero(acc, acc2);
    int sa = 0; uint32_t pha = 0; int sb = 0; uint32_t phb = 0;
    if (a.b_resident) mbar_wait(ball, 0);
    int n, h0, w0, nt;
    for (int it = 0; tile_at(it, n, h0, w0, nt); ++it) {
      uint32_t accf = 0u;                                  // 0 for the tile's very first MMA, 1 afterwards
      int prev_b = -1;                                     // streamed weight stage whose MMAs may still be running
      for (int sl = 0; sl < a.slabs; ++sl) {
        const int sa_h = sa; const uint32_t pha_h = pha;
        if (++sa == a.na) { sa = 0; pha ^= 1; }
        int sa_l = sa_h; uint32_t pha_l = pha_h;
        if constexpr (P == 2) {
          sa_l = sa; pha_l = pha;
          if (++sa == a.na) { sa = 0; pha ^= 1; }
        }
        mbar_wait(afull0 + 8 * sa_h, pha_h);
        if constexpr (P == 2) mbar_wait(afull0 + 8 * sa_l, pha_l);
        const uint64_t ah0 = dA + (a_lo14 + (uint32_t)sa_h * astep), al0 = dA + (a_lo14 + (uint32_t)sa_l * astep);
        for (int tap = 0; tap < a.taps; ++tap) {
          const int r = tap / a.kw, q2 = tap - r * a.kw;
          const uint32_t toff = (uint32_t)r * rowstep + (uint32_t)q2 * pstep;
          uint64_t bd;
          if (a.b_resident) {
            bd = dB + (b_lo14 + (uint32_t)(sl * a.taps + tap) * bstep);
          } else {
            mbar_wait(bfull0 + 8 * sb, phb);
            bd = dB + (b_lo14 + (uint32_t)sb * bstep);
          }
          const uint64_t adh = ah0 + toff, adl = al0 + toff;
          wg_fence();
          mma_stage<BN, P>(acc, acc2, adh, adl, bd, bd + btile, ksteps, accf, bf);
          accf = 1u;
          wg_commit();
          wg_wait<1>();
          if (!a.b_resident) {
            if (prev_b >= 0 && lane == 0) mbar_arrive(bempty0 + 8 * prev_b);
            prev_b = sb;
            if (++sb == a.nb) { sb = 0; phb ^= 1; }
          }
        }
        wg_wait<0>();
        if (lane == 0) {
          if (prev_b >= 0) mbar_arrive(bempty0 + 8 * prev_b);
          mbar_arrive(aempty0 + 8 * sa_h);
          if constexpr (P == 2) mbar_arrive(aempty0 + 8 * sa_l);
        }
        prev_b = -1;
      }
      acc_fence(acc); acc_fence(acc2);
      // ---- epilogue: straight from the accumulator registers ----
      const int n0 = nt * BN;
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) {
        const int row = wg * 64 + frag_row(t, j), nb = n0 + frag_col(t, j);
        const int ho = h0 + (row >> 3), wo = w0 + (row & 7);
        if (ho >= a.Ho || wo >= a.Wo || nb >= a.cout) continue;
        const bool has1 = nb + 1 < a.cout;
        const float b0 = a.bias ? __ldg(a.bias + nb) : 0.f, b1 = (a.bias && has1) ? __ldg(a.bias + nb + 1) : 0.f;
        const size_t pix = ((size_t)n * a.Ho + ho) * a.Wo + wo;
        epilogue_pair<P>(acc, acc2, j, b0, b1, a.acc_scale, act, form, a.dst, a.res, pix * a.cout_store + nb, a.dst_plane, has1, a.fmt);
      }
    }
  }
}

struct C3Op : cpb::Prepared {
  C3Op() : Prepared(cpb::Route::HALO) {}
  C3Args args;
  int BN, P;
  size_t smem;
};

template <int BN, int P>
int launch_c3(const C3Op &t, const C3Args &args, cudaStream_t st) {
  return launch<conv3x3_tc_kernel<BN, P>>("conv3x3_tc_kernel", args.total_tiles, C3_THREADS, t.smem, st, args);
}

}  // namespace

namespace cpb {

bool c3_eligible(const cpb200_op &op) {
  const bool geom = (op.kh == 3 && op.kw == 3) || (op.kh == 7 && op.kw == 1) || (op.kh == 1 && op.kw == 7) || (op.kh == 5 && op.kw == 5);
  return op.type == CPB200_OP_CONV && geom && op.stride == 1 && op.pad_h == op.kh / 2 && op.pad_w == op.kw / 2 &&
         op.nsrc == 1 && op.cin[0] % 16 == 0 && (op.src_pitch[0] == 0 || op.src_pitch[0] == op.cin[0]) && op.Wo >= 8 && op.Ho >= 8 &&
         op.H == op.Ho && op.W == op.Wo &&
         op.out_sy == 1 && op.out_sx == 1 && !op.out_oy && !op.out_ox && op.Hd == op.Ho && op.Wd == op.Wo &&
         !(op.flags & CPB200_FLAG_OUT_NCHW_F32) && tc_dtype(op.act_dtype) &&
         ((op.flags & CPB200_FLAG_OUT_F32) || op.cout % 16 == 0);
}

int c3_prepare(const cpb200_op &op, Prepared **out) {
  std::unique_ptr<C3Op> t(new C3Op());
  C3Args &a = t->args;
  memset(&a, 0, sizeof(a));
  const Prec pr = prec_of(op);
  const Slab sl = slab_for(op.cin, 1);
  const int P = pr.P, cin = op.cin[0], bk = sl.bk;
  t->P = P;
  a.fmt = pr.fmt; a.acc_scale = pr.acc_scale;
  a.dst_plane = (long long)op.B * op.Ho * op.Wo * op.cout;
  a.cin = cin; a.BK = bk; a.slabs = cin / bk;
  a.swizzle_bits = sl.layout;
  a.B = op.B; a.Ho = op.Ho; a.Wo = op.Wo;
  a.tiles_h = (op.Ho + TH - 1) / TH; a.tiles_w = (op.Wo + TW - 1) / TW;
  const int BN = bn_for(op.cout, P);
  t->BN = BN;
  a.n_tiles = (op.cout + BN - 1) / BN;
  a.cout = op.cout; a.cout_store = op.cout;
  a.total_tiles = op.B * a.tiles_h * a.tiles_w * a.n_tiles;
  a.flags = op.flags;
  a.kh = op.kh; a.kw = op.kw; a.taps = op.kh * op.kw; a.hw = TW + op.kw - 1;
  const int hh = TH + op.kh - 1;
  a.a_tx_bytes = (unsigned)(a.hw * hh * bk * 2);
  a.a_stage_bytes = (a.a_tx_bytes + 1023u) & ~1023u;       // one plane of one slab's halo
  a.b_tx_bytes = BN * bk * 2;
  a.b_tile_bytes = a.b_tx_bytes;
  a.b_stage_bytes = ((unsigned)P * a.b_tx_bytes + 1023u) & ~1023u;      // P = 2: [hi tile | lo tile]
  // dynamic shared memory: 227 KB per CTA minus the barriers and the alignment slack
  const size_t budget = 220 * 1024;
  a.na = 3;
  if (a.a_stage_bytes <= 12 * 1024) a.na = (a.a_stage_bytes <= 6 * 1024) ? 16 : 8;   // small halos: deeper ring hides TMA latency
  if (P == 2 && a.na < 4) a.na = 4;                         // two slabs' worth of planes in flight
  const size_t resident_bytes = (size_t)a.taps * a.slabs * a.b_stage_bytes;
  int na_res = a.na;
  while (na_res > 2 && na_res * (size_t)a.a_stage_bytes + resident_bytes > budget) --na_res;
  if (a.n_tiles == 1 && na_res >= (P == 2 ? 3 : a.na) && na_res * (size_t)a.a_stage_bytes + resident_bytes <= budget) {
    a.na = na_res;
    a.b_resident = 1; a.nb = a.taps * a.slabs;
    t->smem = a.na * (size_t)a.a_stage_bytes + resident_bytes + 1024;
  } else {
    a.b_resident = 0;
    const int min_b = P == 2 ? 2 : 3;                       // weight stages wanted beside the halo ring
    if (P == 1 && a.na * (size_t)a.a_stage_bytes + min_b * (size_t)a.b_stage_bytes > budget) a.na = 2;
    while (P == 2 && a.na > 2 && a.na * (size_t)a.a_stage_bytes + min_b * (size_t)a.b_stage_bytes > budget) a.na -= 2;
    if (P == 2 && (a.na & 1)) --a.na;                       // streamed weights consume the planes in pairs
    int nb = (int)((budget - a.na * (size_t)a.a_stage_bytes) / a.b_stage_bytes);
    if (nb > MAX_NB) nb = MAX_NB;
    if (nb < 2 || a.na < 2) return fail(CPB200_ERR_ARG, "tc3: tile does not fit shared memory");
    a.nb = nb;
    t->smem = a.na * (size_t)a.a_stage_bytes + nb * (size_t)a.b_stage_bytes + 1024;
  }
  const cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)a.hw, (cuuint32_t)hh, 1}, estr[4] = {1, 1, 1, 1};
  if (int rc = encode_act_map(&a.amap, op.src[0], cin, cin, op.W, op.H, op.B, P, pr.fmt, sl.swizzle, box, estr, "tc3")) return rc;
  if (int rc = encode_weight_map(&a.bmap, op.weight, pr.fmt, bk, (op.cout + 15) / 16 * 16, BN, (long long)a.taps * a.slabs * P,
                                 sl.swizzle, "tc3"))
    return rc;
  *out = t.release();
  return CPB200_OK;
}

int c3_run(const Prepared &p, const cpb200_op &op, cudaStream_t st) {
  const C3Op &t = static_cast<const C3Op &>(p);
  C3Args args = t.args;
  args.dst = op.dst; args.res = op.res; args.bias = op.bias;
#define C3_CASE(N)                                                                                   \
  case N: return t.P == 2 ? launch_c3<N, 2>(t, args, st) : launch_c3<N, 1>(t, args, st);
  switch (t.BN) {
    C3_CASE(16) C3_CASE(32) C3_CASE(64) C3_CASE(128)
    case 256: if (t.P == 1) return launch_c3<256, 1>(t, args, st); break;
  }
#undef C3_CASE
  return fail(CPB200_ERR_STATE, "tc3: bad BN");
}

}  // namespace cpb

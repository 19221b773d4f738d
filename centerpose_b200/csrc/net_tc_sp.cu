// Small-channel 3x3 convolutions (Cin = 16 or 32, stride 1 or 2, pad 1) on wgmma with SIMT-fed operands.
//
// Why not TMA here: a tiled TMA box is fetched row by row, one request per (pixel row of the box).  With 16 or 32
// channels a request is only 32 / 64 bytes, so the halo-reuse kernel (csrc/net_tc3.cu, 180 requests per tile) and the
// tap-per-stage kernel (csrc/net_tc.cu, 9 x 128 requests per tile for stride 2) would spend most of a tile waiting for
// the copy engine.  Here producer THREADS fetch the halo with coalesced 16-byte loads (a tile row is one contiguous
// 320..1088-byte segment of the NHWC tensor) and store it straight into the swizzled K-major layout the wgmma descriptors
// read — the same scheme as the stem (csrc/net_stem_tc.cu): next tile's loads in flight while this tile is stored.
//
//   halo     stride 1: 18 x 10 pixels, row R = hy*10 + hx;  tap (r,s) = window starting (r*10 + s) rows later,
//            8-row-group stride 10 rows (as in net_tc3.cu).
//            stride 2: 33 x 17 pixels split into four parity planes of 17 x 9 (R = plane*153 + (hy/2)*9 + hx/2)
//            so that the 8 pixels of an output row are again 8 CONSECUTIVE operand rows: tap (r,s) = plane
//            (r&1, s&1), window offset ((r/2)*9 + s/2) rows, group stride 9 rows.
//   swizzle  32-byte (C=16) / 64-byte (C=32) pattern applied on absolute shared-memory address bits
//            (chunk bit(s) [4..] ^= address bits [7..]); stage bases are 1024-aligned.
//   weights  the ordinary tensor-core packing [tap][1 slab][N][C] bf16 (plan.py::_pack_conv_tc, bk = C), swizzled while being
//            copied to shared memory once per CTA.
//   warps    0-7 two consumer warpgroups (rows 0-63 / 64-127 of the tile: wgmma + epilogue), 8-15 producers.
//   split    P = 2 (CPB200_BF16X2 / CPB200_F16X2, tc_common.cuh): the stage ring is plane-granular — a tile occupies two
//            consecutive stages (hi halo, lo halo), fetched as two units of the producers' load pipeline; weights sit in
//            shared memory as [tap][hi tile | lo tile]; A_hi x W_hi goes to one accumulator array, A_hi x W_lo and
//            A_lo x W_hi to a second one; the epilogue adds them, applies
//            acc_scale / bias / residual / activation in fp32 and stores the hi and lo planes.
#include "tc_common.cuh"

#include <cstdlib>

namespace {

using namespace tc;

constexpr int SP_TH = 16, SP_TW = 8;
constexpr int SP_CONS = 256;                              // two consumer warpgroups
constexpr int SP_PT = 256;                                // producer threads
constexpr int SP_THREADS = SP_CONS + SP_PT;

struct SpArgs {
  const __nv_bfloat16 *x;      // (B,H,W,C)            [P = 2: hi plane, lo plane x_plane elements later; 16-bit either format]
  const __nv_bfloat16 *w;      // [9][N][C]            [P = 2: [plane][9][N][C]]
  const __nv_bfloat16 *res;    // optional (B,Ho,Wo,N) [planes y_plane apart]
  __nv_bfloat16 *y;            // (B,Ho,Wo,N)          [planes y_plane apart]
  const float *bias;
  int B, H, W, Ho, Wo;
  int tiles_h, tiles_w, total_tiles;
  uint32_t act;
  uint32_t fmt;                // split mode: 0 = bf16 planes, 1 = fp16 planes
  float acc_scale;
  long long x_plane, y_plane;
};

template <int C, int S>
struct SpGeom {
  static constexpr int PIX_B = C * 2;                     // bytes per pixel row of the operand
  static constexpr int CH = PIX_B / 16;                   // 16-byte chunks per pixel
  static constexpr int HH = (SP_TH - 1) * S + 3, HW = (SP_TW - 1) * S + 3;       // halo extent in input pixels
  static constexpr int PLANE_W = (S == 1) ? HW : (HW + 1) / 2;                   // operand rows per halo row (per plane)
  static constexpr int PLANE_H = (S == 1) ? HH : (HH + 1) / 2;
  static constexpr int PLANE_ROWS = PLANE_W * PLANE_H;
  static constexpr int ROWS = (S == 1) ? PLANE_ROWS : 4 * PLANE_ROWS;
  static constexpr int STAGE_BYTES = ((ROWS * PIX_B + 1023) / 1024) * 1024;
  static constexpr int NCHUNK = HH * HW * CH;             // 16-byte chunks fetched per tile
  static constexpr int NLD = (NCHUNK + SP_PT - 1) / SP_PT;
  static constexpr uint32_t SWMASK = (C == 16) ? 1u : 3u;
  static constexpr uint32_t LAYOUT = (C == 16) ? 3u : 2u; // wgmma layout type: 32-byte / 64-byte swizzle
  static constexpr int NSTAGE = (STAGE_BYTES <= 12 * 1024) ? 6 : (STAGE_BYTES <= 20 * 1024 ? 5 : 4);
  // split mode: plane-granular stages, as many as fit beside the two weight planes (at most 8, at least 3)
  template <int N_>
  struct Split {
    static constexpr int K_ = (200 * 1024 - 2 * 9 * N_ * PIX_B) / STAGE_BYTES;
    static constexpr int NSTAGE = K_ > 8 ? 8 : K_;
  };
};

__device__ __forceinline__ uint32_t sp_swz(uint32_t off, uint32_t mask) {      // offset within a 1024-aligned region
  return off ^ (((off >> 7) & mask) << 4);
}

template <int C, int N, int S, int P>
__global__ void __launch_bounds__(SP_THREADS, 1) conv_sp_kernel(const SpArgs a) {
  using G = SpGeom<C, S>;
  constexpr int NSTAGE = P == 2 ? G::template Split<N>::NSTAGE : G::NSTAGE;
  static_assert(NSTAGE >= 3 && NSTAGE <= 8, "stage ring does not fit");
  constexpr int B_TILE_BYTES = N * G::PIX_B;               // one plane of one tap
  constexpr int B_TAP_BYTES = P * B_TILE_BYTES;            // [hi tile | lo tile]
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = smem_base + NSTAGE * G::STAGE_BYTES;
  __shared__ __align__(8) uint64_t bars[2 * 8];
  __shared__ float s_bias[N];
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[8]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(full0 + 8 * s, SP_PT); mbar_init(empty0 + 8 * s, SP_CONS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // rows the producers never write (plane padding of the stride-2 layout) must hold finite values: zero everything once
  for (int i = threadIdx.x; i < NSTAGE * G::STAGE_BYTES / 16; i += SP_THREADS)
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(a_base + i * 16), "r"(0u) : "memory");
  for (int i = threadIdx.x; i < 9 * B_TAP_BYTES / 16; i += SP_THREADS) {          // weights: dense [plane][tap][n][c] -> swizzled [tap][plane][n][c]
    const uint4 v = __ldg(reinterpret_cast<const uint4 *>(a.w) + i);
    constexpr int TILE_CH = B_TILE_BYTES / 16;
    const int blk = i / TILE_CH, within = i - blk * TILE_CH;                      // blk = plane * 9 + tap
    const int pl = blk / 9, tap = blk - 9 * pl;
    const uint32_t dst = b_base + sp_swz((uint32_t)((tap * P + pl) * TILE_CH + within) * 16u, G::SWMASK);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  for (int i = threadIdx.x; i < N; i += SP_THREADS) s_bias[i] = a.bias ? __ldg(a.bias + i) : 0.f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  auto decode_tile = [&](int t, int &n, int &h0, int &w0) {
    const int tw = t % a.tiles_w; t /= a.tiles_w;
    const int th = t % a.tiles_h; n = t / a.tiles_h;
    h0 = th * SP_TH; w0 = tw * SP_TW;
  };

  if (warp >= SP_CONS / 32) {
    // =============================== producers ===============================
    const int p = threadIdx.x - SP_CONS;
    // chunk i = (hy*HW + hx)*CH + j of the halo: source offset (elements, relative to the halo origin) is tile
    // dependent only through (hi0, wi0); destination offset inside a stage is fixed -> precomputed.
    uint32_t doff[G::NLD];
    int hyx[G::NLD];                                        // hy << 16 | hx << 8 | j, or -1
#pragma unroll
    for (int q = 0; q < G::NLD; ++q) {
      const int i = p + q * SP_PT;
      if (i < G::NCHUNK) {
        const int j = i % G::CH, px = i / G::CH;
        const int hx = px % G::HW, hy = px / G::HW;
        int R;
        if (S == 1) R = hy * G::PLANE_W + hx;
        else R = ((hy & 1) * 2 + (hx & 1)) * G::PLANE_ROWS + (hy >> 1) * G::PLANE_W + (hx >> 1);
        doff[q] = sp_swz((uint32_t)(R * G::PIX_B + j * 16), G::SWMASK);
        hyx[q] = (hy << 16) | (hx << 8) | j;
      } else {
        doff[q] = 0; hyx[q] = -1;
      }
    }
    uint4 pre[G::NLD];
    auto fetch = [&](int t, int pl) {
      int n, h0, w0; decode_tile(t, n, h0, w0);
      const int hi0 = h0 * S - 1, wi0 = w0 * S - 1;
      const __nv_bfloat16 *xin = a.x + (size_t)n * a.H * a.W * C + (P == 2 ? (size_t)pl * a.x_plane : 0);
#pragma unroll
      for (int q = 0; q < G::NLD; ++q) {
        const int hy = hyx[q] >> 16, hx = (hyx[q] >> 8) & 255, j = hyx[q] & 255;
        const int hi = hi0 + hy, wi = wi0 + hx;
        const bool ok = hyx[q] >= 0 && hi >= 0 && hi < a.H && wi >= 0 && wi < a.W;
        pre[q] = ok ? __ldg(reinterpret_cast<const uint4 *>(xin + ((size_t)hi * a.W + wi) * C) + j) : make_uint4(0u, 0u, 0u, 0u);
      }
    };
    int vs = 0;
    if ((int)blockIdx.x < a.total_tiles) fetch(blockIdx.x, 0);
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
#pragma unroll
      for (int pl = 0; pl < P; ++pl, ++vs) {                 // a tile = P consecutive plane stages
        const int stage = vs % NSTAGE;
        const uint32_t phase = (uint32_t)(vs / NSTAGE) & 1u;
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t sa = a_base + stage * G::STAGE_BYTES;
#pragma unroll
        for (int q = 0; q < G::NLD; ++q)
          if (hyx[q] >= 0)
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sa + doff[q]), "r"(pre[q].x), "r"(pre[q].y), "r"(pre[q].z),
                         "r"(pre[q].w) : "memory");
        // the next unit's loads fly while the consumers work on this one
        if (pl + 1 < P) fetch(t, pl + 1);
        else if (t + (int)gridDim.x < a.total_tiles) fetch(t + gridDim.x, 0);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(full0 + 8 * stage);
      }
    }
  } else {
    // =============================== consumers: wgmma + epilogue ===============================
    const int wg = warp >> 2, tq = threadIdx.x & 127;
    const uint32_t bf = (P == 1 || a.fmt == 0) ? 1u : 0u;
    float acc[N / 2], acc2[P == 2 ? N / 2 : 1];                 // hi x W_hi | hi x W_lo + lo x W_hi (split operands)
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (P == 2 ? N / 2 : 1); ++i) acc2[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
#pragma unroll
      for (int pl = 0; pl < P; ++pl) {
        mbar_wait(full0 + 8 * stage, phase);
        // this warpgroup's 64 rows = 8 output rows of the tile = 8 operand row groups further on
        const uint64_t ad0 = desc_sbo(a_base + stage * G::STAGE_BYTES + wg * 8 * G::PLANE_W * G::PIX_B, G::PLANE_W * G::PIX_B, G::LAYOUT);
        const uint64_t bd0 = desc_sbo(b_base, 8 * G::PIX_B, G::LAYOUT);
        wg_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const int r = tap / 3, s = tap % 3;
          const int row0 = (S == 1) ? (r * G::PLANE_W + s)
                                    : (((r & 1) * 2 + (s & 1)) * G::PLANE_ROWS + (r >> 1) * G::PLANE_W + (s >> 1));
#pragma unroll
          for (int k = 0; k < C / 16; ++k) {
            const uint64_t ad = ad0 + (uint32_t)(row0 * (G::PIX_B >> 4) + 2 * k), bd = bd0 + (uint32_t)(tap * (B_TAP_BYTES >> 4) + 2 * k);
            const uint32_t first = (pl > 0 || tap > 0 || k > 0) ? 1u : 0u;
            if constexpr (P == 1) wgmma_k16<N>(acc, ad, bd, first, 1u);
            else if (pl == 0) {
              wgmma_k16<N>(acc, ad, bd, first, bf);                              // A_hi x W_hi
              wgmma_k16<N>(acc2, ad, bd + (uint32_t)(B_TILE_BYTES >> 4), first, bf);   // A_hi x W_lo
            } else {
              wgmma_k16<N>(acc2, ad, bd, 1u, bf);                                // A_lo x W_hi
            }
          }
        }
        wg_commit();
        wg_wait<0>();
        if (lane == 0) mbar_arrive(empty0 + 8 * stage);
        if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
      }
      acc_fence(acc); acc_fence(acc2);
      int n, h0, w0; decode_tile(t, n, h0, w0);
#pragma unroll
      for (int j = 0; j < N / 4; ++j) {
        const int m = wg * 64 + frag_row(tq, j), c = frag_col(tq, j);
        const int ho = h0 + (m >> 3), wo = w0 + (m & 7);
        if (ho >= a.Ho || wo >= a.Wo) continue;
        float v0 = acc[2 * j], v1 = acc[2 * j + 1];
        if constexpr (P == 2) { v0 += acc2[2 * j]; v1 += acc2[2 * j + 1]; }
        const float f0 = P == 2 ? fmaf(v0, a.acc_scale, s_bias[c]) : v0 + s_bias[c];
        const float f1 = P == 2 ? fmaf(v1, a.acc_scale, s_bias[c + 1]) : v1 + s_bias[c + 1];
        const size_t pix = ((size_t)n * a.Ho + ho) * a.Wo + wo;
        store_pair16<P>(a.y, a.res, pix * N + c, a.y_plane, f0, f1, a.act, a.fmt);
      }
    }
  }
}

template <int C, int N, int S, int P>
int launch_sp(const cpb200_op &op, cudaStream_t st) {
  using G = SpGeom<C, S>;
  constexpr int NSTAGE = P == 2 ? G::template Split<N>::NSTAGE : G::NSTAGE;
  SpArgs a;
  a.x = static_cast<const __nv_bfloat16 *>(op.src[0]); a.w = static_cast<const __nv_bfloat16 *>(op.weight);
  a.res = static_cast<const __nv_bfloat16 *>(op.res); a.y = static_cast<__nv_bfloat16 *>(op.dst); a.bias = op.bias;
  a.B = op.B; a.H = op.H; a.W = op.W; a.Ho = op.Ho; a.Wo = op.Wo;
  a.tiles_h = (op.Ho + SP_TH - 1) / SP_TH; a.tiles_w = (op.Wo + SP_TW - 1) / SP_TW;
  a.total_tiles = op.B * a.tiles_h * a.tiles_w;
  a.act = op.flags & CPB_ACT_MASK;
  a.fmt = op.act_dtype == CPB200_F16X2 ? 1u : 0u;
  a.acc_scale = op.acc_scale != 0.f ? op.acc_scale : 1.f;
  a.x_plane = (long long)op.B * op.H * op.W * C;
  a.y_plane = (long long)op.B * op.Ho * op.Wo * N;
  const size_t smem = 1024 + (size_t)NSTAGE * G::STAGE_BYTES + (size_t)P * 9 * N * G::PIX_B;
  static SmemAttrCache cache;
  if (int rc = ensure_smem(conv_sp_kernel<C, N, S, P>, smem, cache)) return rc;
  const int sms = tc::num_sms();
  const int grid = a.total_tiles < sms ? a.total_tiles : sms;
  conv_sp_kernel<C, N, S, P><<<grid, SP_THREADS, smem, st>>>(a);
  return cpb::check_launch("conv_sp_kernel");
}

template <int C, int S>
int dispatch_n(const cpb200_op &op, cudaStream_t st) {
  const bool split = op.act_dtype != CPB200_BF16;
  switch (op.cout) {
    case 16: return split ? launch_sp<C, 16, S, 2>(op, st) : launch_sp<C, 16, S, 1>(op, st);
    case 32: return split ? launch_sp<C, 32, S, 2>(op, st) : launch_sp<C, 32, S, 1>(op, st);
    case 64: return split ? launch_sp<C, 64, S, 2>(op, st) : launch_sp<C, 64, S, 1>(op, st);
  }
  return cpb::fail(CPB200_ERR_ARG, "conv_sp: cout %d", op.cout);
}

}  // namespace

namespace cpb {

bool sp_eligible(const cpb200_op &op) {
  static const bool enabled = []() { const char *e = getenv("CPB200_SP"); return !(e && e[0] == '0'); }();
  return enabled && op.type == CPB200_OP_CONV && (op.flags & CPB200_FLAG_TC) &&
         (op.act_dtype == CPB200_BF16 || op.act_dtype == CPB200_BF16X2 || op.act_dtype == CPB200_F16X2) && op.nsrc == 1 &&
         (op.src_pitch[0] == 0 || op.src_pitch[0] == op.cin[0]) &&
         (op.cin[0] == 16 || op.cin[0] == 32) && (op.cout == 16 || op.cout == 32 || op.cout == 64) && op.kh == 3 && op.kw == 3 &&
         op.pad_h == 1 && op.pad_w == 1 && (op.stride == 1 || op.stride == 2) &&
         op.Ho == (op.H + 2 - 3) / op.stride + 1 && op.Wo == (op.W + 2 - 3) / op.stride + 1 &&
         op.out_sy == 1 && op.out_sx == 1 && !op.out_oy && !op.out_ox && op.Hd == op.Ho && op.Wd == op.Wo &&
         !(op.flags & (CPB200_FLAG_OUT_NCHW_F32 | CPB200_FLAG_OUT_F32)) && op.Wo >= 8;
}

int sp_run(const cpb200_op &op, cudaStream_t st) {
  if (!sp_eligible(op)) return fail(CPB200_ERR_ARG, "conv_sp: unsupported shape");
  if (op.cin[0] == 16) return op.stride == 1 ? dispatch_n<16, 1>(op, st) : dispatch_n<16, 2>(op, st);
  return op.stride == 1 ? dispatch_n<32, 1>(op, st) : dispatch_n<32, 2>(op, st);
}

}  // namespace cpb

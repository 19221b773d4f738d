// wgmma / TMA implicit-GEMM convolution for sm_90a (bf16 NHWC activations, fp32 accumulate in registers).
//
//   M tile  = 128 output pixels = a TH x TW rectangle of one image (8x16, or 16x8 for narrow maps); two consumer warpgroups
//             own rows 0-63 and 64-127 (wgmma m64nNk16 each)
//   N tile  = BN output channels (16..256)
//   K loop  = filter taps x concatenated inputs x channel slabs of BK (64/32/16 = one swizzle atom)
//
// A operand: for tap (r,s) the 128 x BK slab is the input window
//   x[n, h0*stride + r - pad : .. : stride, w0*stride + s - pad : .. : stride, c0 : c0+BK]
// fetched by ONE 4-D TMA tiled load (box {BK, TW, TH, 1}, element strides {1,stride,stride,1});
// TMA zero-fills out-of-bounds coordinates, which IS the convolution's zero padding, and lands the
// box in shared memory as 128 rows of BK bf16 in the 128B/64B/32B-swizzled K-major layout the wgmma
// shared-memory descriptor expects — no im2col buffer exists anywhere.
// B operand: weights packed slab-major [tap][K-slab][Cout_pad][BK] bf16 (K-major), 3-D TMA box {BK, BN, 1}.
// `Root` concatenations are K-slabs from up to four tensor maps (no torch.cat copy).
//
// Warp roles (persistent CTAs, one per SM): warps 0-7 = two consumer warpgroups (wgmma issue, then the epilogue straight
// from the accumulator registers: +bias (+residual) -> activation -> store), warp 8 = TMA producer (DCN: warps 8-15 gather
// the A tile, one lane of warp 8 also issues the weight loads); a STAGES-deep smem ring
// with full/empty mbarriers feeds the tensor cores, and a stage is released as soon as the MMAs of the NEXT stage are queued.
//
// Split-operand precisions (P = 2, CPB200_BF16X2 / CPB200_F16X2, see tc_common.cuh): a stage is
// [A_hi | A_lo | W_hi | W_lo]; per stage the consumers issue the three products of every K step (tc::mma_stage).  The DCN gather blends the four corners of BOTH planes in fp32 and re-splits the sample.
//
// Pointwise convs (pw_eligible: 1x1 / stride 1 / pad 0 with an NHWC output) run as one 1 x (B*H*W) "image": a tile is 128
// consecutive pixels of the flattened map (TH 1 x TW 128, one 2-D box per K slab), the ring fills the whole opt-in shared
// memory so that several tiles of A stay in flight across an epilogue, and the epilogue stores 16 bytes per lane and
// plane (TcArgs::vec8: tc::quad_rows8 + tc::epilogue_vec8).  The products and the epilogue arithmetic are the same as
// with 2-D tiles, so the outputs are too; CPB200_NO_PW=1 (read at prepare) keeps these ops on 2-D tiles.
#include <cstdlib>
#include <type_traits>
#include "tc_common.cuh"
#include <mutex>
#include <memory>

namespace {

constexpr int CONS_THREADS = 256;      // two consumer warpgroups
constexpr int TC_THREADS = CONS_THREADS + 32;        // + TMA producer warp
constexpr int TILE_M = 128;
constexpr int MAX_STAGES = 16;

struct alignas(64) TcArgs {
  CUtensorMap amap[4];
  CUtensorMap bmap;
  int cin[4];
  int nsrc;
  int kh, kw, stride, pad_h, pad_w;
  int B, Ho, Wo;
  int TH, TW, tiles_h, tiles_w, n_tiles;
  int cout, cout_store;       // cout_store: channel pitch of dst/res
  int BK, stages, total_tiles;
  void *dst;
  const void *res;
  const float *bias;
  unsigned flags;
  unsigned swizzle_bits;      // wgmma layout type for the chosen BK
  // deformable conv (DCN) only: A tiles are gathered by producer warps instead of TMA
  const __nv_bfloat16 *dcn_src;   // (B,H,W,Cin) bf16
  const float *dcn_om;            // (B,H,W,27) fp32: 18 offsets (dy,dx per tap) | 9 mask logits
  int H, W, om_pitch;
  int Hd, Wd, sy, sx, oy, ox;     // strided output mapping (dense ConvTranspose2d parity sub-convs)
  int out_ch_off, out_ch_total;   // NCHW fp32 output: channel slice of dst
  // split-operand mode (P = 2)
  unsigned fmt;                   // 0 = bf16 planes, 1 = fp16 planes
  float acc_scale;                // accumulator multiplier (inverse of the host's power-of-two weight scale)
  long long dst_plane;            // elements between the hi and lo planes of dst / res
  long long src_plane;            // DCN: elements between the planes of dcn_src
  int wplane;                     // weight blocks (tap x K-slab) per plane
  unsigned vec8;                  // 16-byte epilogue (pointwise convs: NHWC output, cout % 16 == 0, 16-byte aligned dst / res)
};

using namespace tc;

constexpr int DCN_GW = 8;                       // gather-producer warps
constexpr int DCN_ROWS = 128 / DCN_GW;          // operand rows per gather warp
constexpr int DCN_THREADS = CONS_THREADS + DCN_GW * 32;   // 16 warps: 4 per scheduler partition leave 128 registers a thread

struct __align__(16) DcnPrm { int off[4]; uint32_t wt[4]; };   // element offsets; corner weights: packed bf16x2 (w,w), or fp32 bits when P = 2

template <int BN, bool DCN, int P>
__global__ void __launch_bounds__(DCN ? DCN_THREADS : TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcArgs a) {
  static_assert(P == 1 || BN <= 128, "split operands: two BN-column accumulators per thread");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages x (A planes | B planes)]
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_bytes = TILE_M * a.BK * 2, b_bytes = BN * a.BK * 2;
  const uint32_t stage_bytes = P * a_bytes + ((P * b_bytes + 1023u) & ~1023u);
  __shared__ __align__(8) uint64_t bars[2 * MAX_STAGES];
  __shared__ DcnPrm s_prm[DCN ? DCN_GW : 1][DCN ? 9 : 1][DCN ? DCN_ROWS : 1];
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[MAX_STAGES]);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == CONS_THREADS) {
    if (!DCN) for (int s = 0; s < a.nsrc; ++s) tmap_prefetch(&a.amap[s]);
    tmap_prefetch(&a.bmap);
    for (int s = 0; s < a.stages; ++s) { mbar_init(full0 + 8 * s, DCN ? 1 + DCN_GW : 1); mbar_init(empty0 + 8 * s, CONS_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int taps = a.kh * a.kw;
  int kblocks_per_tap = 0;
  for (int s = 0; s < a.nsrc; ++s) kblocks_per_tap += a.cin[s] / a.BK;
  const int kblocks = taps * kblocks_per_tap;

  auto decode_tile = [&](int t, int &n, int &h0, int &w0, int &nt) {
    nt = t % a.n_tiles; t /= a.n_tiles;
    const int tw = t % a.tiles_w; t /= a.tiles_w;
    const int th = t % a.tiles_h; n = t / a.tiles_h;
    h0 = th * a.TH; w0 = tw * a.TW;
  };

  if (!DCN && warp == CONS_THREADS / 32) {
    // =============================== TMA producer ===============================
    if (elect_one()) {
      int stage = 0; uint32_t phase = 0;
      for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        int n, h0, w0, nt; decode_tile(t, n, h0, w0, nt);
        for (int tap = 0; tap < taps; ++tap) {
          const int r = tap / a.kw, s_ = tap % a.kw;
          const int hi = h0 * a.stride + r - a.pad_h, wi = w0 * a.stride + s_ - a.pad_w;
          int cb = 0;
          for (int s = 0; s < a.nsrc; ++s) {
            for (int c0 = 0; c0 < a.cin[s]; c0 += a.BK) {
              mbar_wait(empty0 + 8 * stage, phase ^ 1);
              const uint32_t sa = smem_base + stage * stage_bytes, sb = sa + P * a_bytes;
              mbar_expect_tx(full0 + 8 * stage, P * (a_bytes + b_bytes));
#pragma unroll
              for (int pl = 0; pl < P; ++pl) tma_load_4d(sa + pl * a_bytes, &a.amap[s], full0 + 8 * stage, c0, wi, hi, n + pl * a.B);
#pragma unroll
              for (int pl = 0; pl < P; ++pl)
                tma_load_3d(sb + pl * b_bytes, &a.bmap, full0 + 8 * stage, 0, nt * BN,
                            pl * a.wplane + tap * kblocks_per_tap + (cb + c0) / a.BK);
              if (++stage == a.stages) { stage = 0; phase ^= 1; }
            }
            cb += a.cin[s];
          }
        }
      }
    }
  } else if (DCN && warp >= CONS_THREADS / 32) {
    // =============================== DCN gather producers ===============================
    // A[row = pixel][k = channel] of tap t is  sigmoid(mask_t) * bilinear(x, p + tap_t + offset_t)
    // (dcn_v2_im2col_cuda.cu:25-54,125-195), rounded to bf16 and stored straight into the 128B-swizzled
    // K-major tile the wgmma descriptor reads (16-byte chunk j of row r lives at chunk j ^ (r & 7)).
    // Per tile each warp first turns the 27 offset/mask values of its pixels into (4 corner offsets, 4 corner weights) for
    // all 9 taps (one round trip to global memory instead of one per tap); per stage every thread fetches the 4 corners of
    // one 16-byte chunk of DCN_ROWS / 4 rows, and the loads of the NEXT unit of work are issued before this one's results
    // are stored.  P = 2 (split operands): corners come from both planes, are summed and blended in fp32 with fp32 weights
    // (expf, not ex2.approx, for the mask), and the sample is re-split into the hi / lo A tiles.
    constexpr int NI = DCN_ROWS / 4;                       // rows per thread and stage
    const int gw = warp - CONS_THREADS / 32;               // rows [DCN_ROWS*gw, DCN_ROWS*(gw+1))
    // the weight tile of a stage: loaded by one lane of gather warp 0 once the stage is free (its expect_tx is the
    // barrier's extra arrival)
    auto load_b = [&](int stage_, int nt_, int tap, int c0) {
      if (gw != 0 || lane != 0) return;
      const uint32_t sb = smem_base + stage_ * stage_bytes + P * a_bytes;
      mbar_expect_tx(full0 + 8 * stage_, P * b_bytes);
#pragma unroll
      for (int pl = 0; pl < P; ++pl)
        tma_load_3d(sb + pl * b_bytes, &a.bmap, full0 + 8 * stage_, 0, nt_ * BN, pl * a.wplane + tap * kblocks_per_tap + c0 / a.BK);
    };
    int stage = 0; uint32_t phase = 0;
    const int Cin = a.cin[0];
    const int slabs = Cin >> 6;
    const int nk = 9 * slabs;
    const int chunk = lane & 7, rsub = lane >> 3;
    const __nv_bfloat16 *srcc = a.dcn_src + chunk * 8;
    const int px = lane & 7, tg = lane >> 3;               // pixel of the warp's group of 8, tap group {0,1,2} {3,4} {5,6} {7,8}
    const int tap0 = tg == 0 ? 0 : 1 + 2 * tg, ntap = tg == 0 ? 3 : 2;
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
      int n, h0, w0, nt; decode_tile(t, n, h0, w0, nt);
      __syncwarp();                                        // previous tile's readers are done with s_prm
#pragma unroll 1
      for (int pg = 0; pg < DCN_ROWS / 8; ++pg) {
        const int rp = gw * DCN_ROWS + pg * 8 + px;
        const int ho = h0 + rp / a.TW, wo = w0 + rp % a.TW;
        const bool okp = ho < a.Ho && wo < a.Wo;
        const float *om = a.dcn_om + (((size_t)n * a.H + ho) * a.W + wo) * a.om_pitch;
        float oh[3], ow[3], ml[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int tap = tap0 + i;
          const bool ld = okp && i < ntap;
          oh[i] = ld ? __ldg(om + 2 * tap) : 0.f; ow[i] = ld ? __ldg(om + 2 * tap + 1) : 0.f; ml[i] = ld ? __ldg(om + 18 + tap) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          if (i < ntap) {
            const int tap = tap0 + i;
            DcnPrm pr;
#pragma unroll
            for (int c = 0; c < 4; ++c) { pr.off[c] = 0; pr.wt[c] = 0u; }
            if (okp) {
              const float mk = P == 2 ? 1.0f / (1.0f + expf(-ml[i])) : 1.0f / (1.0f + __expf(-ml[i]));
              const float h_im = (float)(ho - 1 + tap / 3) + oh[i], w_im = (float)(wo - 1 + tap % 3) + ow[i];
              if (h_im > -1.f && w_im > -1.f && h_im < (float)a.H && w_im < (float)a.W) {
                const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
                const int h_high = h_low + 1, w_high = w_low + 1;
                const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
                const int rowb = n * a.H;
                auto pk = [](float w) {
                  if constexpr (P == 2) return __float_as_uint(w);
                  __nv_bfloat162 b = __float2bfloat162_rn(w); return *reinterpret_cast<uint32_t *>(&b);
                };
                constexpr int OS = P == 2 ? 2 : 1;       // P = 2 gathers with 32-bit BYTE offsets from the tensor base
                if (h_low >= 0 && w_low >= 0) { pr.off[0] = ((rowb + h_low) * a.W + w_low) * Cin * OS; pr.wt[0] = pk(hh * hw * mk); }
                if (h_low >= 0 && w_high <= a.W - 1) { pr.off[1] = ((rowb + h_low) * a.W + w_high) * Cin * OS; pr.wt[1] = pk(hh * lw * mk); }
                if (h_high <= a.H - 1 && w_low >= 0) { pr.off[2] = ((rowb + h_high) * a.W + w_low) * Cin * OS; pr.wt[2] = pk(lh * hw * mk); }
                if (h_high <= a.H - 1 && w_high <= a.W - 1) { pr.off[3] = ((rowb + h_high) * a.W + w_high) * Cin * OS; pr.wt[3] = pk(lh * lw * mk); }
              }
            }
            s_prm[gw][tap][pg * 8 + px] = pr;
          }
        }
      }
      __syncwarp();
      if constexpr (P == 1) {
        uint4 v[2][4];
        uint32_t w[2][4];
        auto issue = [&](int tap, int c0, int h) {           // rows (2h, 2h + 1) of this thread
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const DcnPrm q = s_prm[gw][tap][(2 * h + i) * 4 + rsub];
#pragma unroll
            for (int c = 0; c < 4; ++c) {       // invalid corners: weight 0, offset 0 (a safe address)
              v[i][c] = __ldg(reinterpret_cast<const uint4 *>(srcc + (size_t)(unsigned)q.off[c] + c0));
              w[i][c] = q.wt[c];
            }
          }
        };
        int tap_c = 0, c0_c = 0;
        issue(0, 0, 0);
        for (int k = 0; k < nk; ++k) {
          int tap_n = tap_c, c0_n = c0_c + 64;
          if (c0_n >= Cin) { c0_n = 0; ++tap_n; }
          mbar_wait(empty0 + 8 * stage, phase ^ 1);
          load_b(stage, nt, tap_c, c0_c);
          const uint32_t sa = smem_base + stage * stage_bytes;
#pragma unroll
          for (int h = 0; h < NI / 2; ++h) {
            uint4 o[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              __nv_bfloat162 acc2[4];
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const __nv_bfloat162 w2 = *reinterpret_cast<const __nv_bfloat162 *>(&w[i][c]);
                const __nv_bfloat162 *vv = reinterpret_cast<const __nv_bfloat162 *>(&v[i][c]);
#pragma unroll
                for (int j = 0; j < 4; ++j) acc2[j] = (c == 0) ? __hmul2(w2, vv[j]) : __hfma2(w2, vv[j], acc2[j]);
              }
              o[i] = *reinterpret_cast<const uint4 *>(acc2);
            }
            if (h + 1 < NI / 2) issue(tap_c, c0_c, h + 1);     // the next unit's corners fly across the stores / fence / wait
            else if (k + 1 < nk) issue(tap_n, c0_n, 0);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int row = gw * DCN_ROWS + (2 * h + i) * 4 + rsub;
              const uint32_t dst = sa + row * 128 + ((chunk ^ (row & 7)) << 4);
              asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(o[i].x), "r"(o[i].y), "r"(o[i].z), "r"(o[i].w) : "memory");
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(full0 + 8 * stage);       // one arrival per gather warp
          if (++stage == a.stages) { stage = 0; phase ^= 1; }
          tap_c = tap_n; c0_c = c0_n;
        }
      } else {
        uint4 vh[4], vl[4];
        float wq[4];
        // addresses = uniform tensor base + a 32-bit byte offset (one integer add per load; the host checks < 4 GiB)
        const char *srcb = reinterpret_cast<const char *>(a.dcn_src);
        const uint32_t lane_b = (uint32_t)chunk * 16u, plane_b = (uint32_t)(a.src_plane * 2);
        auto issue = [&](int tap, int c0, int i) {
          const DcnPrm q = s_prm[gw][tap][i * 4 + rsub];
          const uint32_t cb = lane_b + (uint32_t)c0 * 2u;
#pragma unroll
          for (int c = 0; c < 4; ++c) {         // invalid corners: weight 0, offset 0 (a safe address)
            const uint32_t e = (uint32_t)q.off[c] + cb;
            vh[c] = __ldg(reinterpret_cast<const uint4 *>(srcb + e));
            vl[c] = __ldg(reinterpret_cast<const uint4 *>(srcb + (e + plane_b)));
            wq[c] = __uint_as_float(q.wt[c]);
          }
        };
        int tap_c = 0, c0_c = 0;                             // (tap, channel offset) of the current stage
        issue(0, 0, 0);
        for (int k = 0; k < nk; ++k) {
          int tap_n = tap_c, c0_n = c0_c + 64;
          if (c0_n >= Cin) { c0_n = 0; ++tap_n; }
          mbar_wait(empty0 + 8 * stage, phase ^ 1);
          load_b(stage, nt, tap_c, c0_c);
          const uint32_t sa = smem_base + stage * stage_bytes;
#pragma unroll
          for (int i = 0; i < NI; ++i) {
            float f[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] = 0.f;
            uint32_t oh[4], ol[4];
            if (a.fmt) {
              // fp16 planes: sample = sum_c w_c * hi_c (fp32 FMAs on the unpacked hi plane) + sum_c w_c * lo_c.  The second sum is
              // 2^-11 of the first, so packed fp16 FMAs on the lo plane as stored (weights rounded to fp16: error 2^-11 of
              // 2^-11) leave the sample good to 2^-22 — and save the lo plane's unpack and the hi + lo adds.
              __half2 s2[4];
#pragma unroll
              for (int j = 0; j < 4; ++j) s2[j] = __float2half2_rn(0.f);
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const uint32_t hw_[4] = {vh[c].x, vh[c].y, vh[c].z, vh[c].w};
                const uint32_t lw_[4] = {vl[c].x, vl[c].y, vl[c].z, vl[c].w};
                const __half2 w2 = __float2half2_rn(wq[c]);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float2 x = __half22float2(*reinterpret_cast<const __half2 *>(&hw_[j]));
                  f[2 * j] = fmaf(wq[c], x.x, f[2 * j]); f[2 * j + 1] = fmaf(wq[c], x.y, f[2 * j + 1]);
                  s2[j] = __hfma2(w2, *reinterpret_cast<const __half2 *>(&lw_[j]), s2[j]);
                }
              }
              // the registers are free again: the next unit's corners fly while this one is split and stored
              if (i + 1 < NI) issue(tap_c, c0_c, i + 1);
              else if (k + 1 < nk) issue(tap_n, c0_n, 0);
#pragma unroll
              for (int j = 0; j < 4; ++j) {                  // |blend| <= max|x|: no saturation needed
                const __half2 h = __floats2half2_rn(f[2 * j], f[2 * j + 1]);
                const float2 hf = __half22float2(h);
                const __half2 l = __hadd2(__floats2half2_rn(f[2 * j] - hf.x, f[2 * j + 1] - hf.y), s2[j]);
                oh[j] = *reinterpret_cast<const uint32_t *>(&h); ol[j] = *reinterpret_cast<const uint32_t *>(&l);
              }
            } else {
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const uint32_t hw_[4] = {vh[c].x, vh[c].y, vh[c].z, vh[c].w};
                const uint32_t lw_[4] = {vl[c].x, vl[c].y, vl[c].z, vl[c].w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float2 x = join2(hw_[j], lw_[j], 0u);
                  f[2 * j] = fmaf(wq[c], x.x, f[2 * j]); f[2 * j + 1] = fmaf(wq[c], x.y, f[2 * j + 1]);
                }
              }
              if (i + 1 < NI) issue(tap_c, c0_c, i + 1);
              else if (k + 1 < nk) issue(tap_n, c0_n, 0);
#pragma unroll
              for (int j = 0; j < 4; ++j) split2_bounded(f[2 * j], f[2 * j + 1], 0u, oh[j], ol[j]);
            }
            const int row = gw * DCN_ROWS + i * 4 + rsub;
            const uint32_t dst = sa + row * 128 + ((chunk ^ (row & 7)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(oh[0]), "r"(oh[1]), "r"(oh[2]), "r"(oh[3]) : "memory");
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst + a_bytes), "r"(ol[0]), "r"(ol[1]), "r"(ol[2]), "r"(ol[3]) : "memory");
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(full0 + 8 * stage);       // one arrival per gather warp
          if (++stage == a.stages) { stage = 0; phase ^= 1; }
          tap_c = tap_n; c0_c = c0_n;
        }
      }
    }
  } else if (warp < CONS_THREADS / 32) {
    // =============================== consumers: wgmma + epilogue ===============================
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const uint32_t bf = (P == 1 || a.fmt == 0) ? 1u : 0u;
    const uint32_t row_bytes = a.BK * 2;
    const uint64_t dT = make_desc(0u, row_bytes, a.swizzle_bits);
    const uint32_t base14 = (smem_base & 0x3FFFFu) >> 4, sstep = stage_bytes >> 4;
    const uint32_t aoff = (uint32_t)wg * ((64u * row_bytes) >> 4);           // this warpgroup's 64 rows of A
    const uint32_t aplane = a_bytes >> 4, bplane = b_bytes >> 4, boff = (uint32_t)(P * a_bytes) >> 4;
    const int ksteps = a.BK / 16;
    const uint32_t act = a.flags & CPB_ACT_MASK;
    const int form = out_form(a.flags);
    float acc[BN / 2], acc2[P == 2 ? BN / 2 : 1];
    acc_zero(acc, acc2);
    int stage = 0; uint32_t phase = 0;
    for (int tt = blockIdx.x; tt < a.total_tiles; tt += gridDim.x) {
      int prev = -1;                                       // stage whose MMAs may still be running
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(full0 + 8 * stage, phase);
        const uint64_t sd = dT + (base14 + (uint32_t)stage * sstep);
        const uint64_t ad = sd + aoff, bd = sd + boff;
        wg_fence();
        mma_stage<BN, P>(acc, acc2, ad, ad + aplane, bd, bd + bplane, ksteps, kb > 0 ? 1u : 0u, bf);
        wg_commit();
        wg_wait<1>();                                      // the previous stage's MMAs have retired: release it
        if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
        prev = stage;
        if (++stage == a.stages) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      acc_fence(acc); acc_fence(acc2);
      if (prev >= 0 && lane == 0) mbar_arrive(empty0 + 8 * prev);
      int n, h0, w0, nt; decode_tile(tt, n, h0, w0, nt);
      const int n0 = nt * BN;
      if (a.vec8) {
        // after quad_rows8, lane q owns row r0 + 8 (q & 1) and 8-column block q >> 1 of each 16-column group
        const int q = t & 3, row = wg * 64 + frag_row(t, q & 1);
        const int ho = h0 + row / a.TW, wo = w0 + row % a.TW;
        const int pix = ho < a.Ho && wo < a.Wo ? (n * a.Hd + ho) * a.Wd + wo : -1;     // < 2^31: pw_eligible
#pragma unroll
        for (int g = 0; g < BN / 16; ++g) {
          float2 v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {                   // registers 8g + 2u, +1: row r0 + 8 (u & 1), block 2g + (u >> 1)
            const int r = 8 * g + 2 * u, c = n0 + 16 * g + 8 * (u >> 1) + 2 * (t & 3);
            const bool hb = a.bias && c < a.cout;         // cout % 16 == 0: c < cout implies c + 1 < cout
            const float b0 = hb ? __ldg(a.bias + c) : 0.f, b1 = hb ? __ldg(a.bias + c + 1) : 0.f;
            if constexpr (P == 2) v[u] = make_float2(fmaf(acc[r] + acc2[r], a.acc_scale, b0), fmaf(acc[r + 1] + acc2[r + 1], a.acc_scale, b1));
            else v[u] = make_float2(acc[r] + b0, acc[r + 1] + b1);
          }
          quad_rows8(v, q);
          const int c = n0 + 16 * g + 8 * (q >> 1);
          if (pix < 0 || c >= a.cout) continue;
          epilogue_vec8<P>(v, act, form, a.dst, a.res, (size_t)pix * a.cout_store + c, a.dst_plane, a.fmt);
        }
        continue;
      }
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) {                   // pairs of adjacent columns of this thread's fragment
        const int row = wg * 64 + frag_row(t, j), nb = n0 + frag_col(t, j);
        const int ho = h0 + row / a.TW, wo = w0 + row % a.TW;
        if (ho >= a.Ho || wo >= a.Wo || nb >= a.cout) continue;
        const bool has1 = nb + 1 < a.cout;
        const float b0 = a.bias ? __ldg(a.bias + nb) : 0.f, b1 = (a.bias && has1) ? __ldg(a.bias + nb + 1) : 0.f;
        const int y = ho * a.sy + a.oy, x = wo * a.sx + a.ox;     // strided output lattice of the deconv parity convs
        // NCHW: the head outputs, a channel slice of dst
        const size_t e = form == OUT_NCHW ? (((size_t)n * a.out_ch_total + a.out_ch_off + nb) * a.Hd + y) * a.Wd + x
                                          : (((size_t)n * a.Hd + y) * a.Wd + x) * a.cout_store + nb;
        const long long plane = form == OUT_NCHW ? (long long)a.Hd * a.Wd : a.dst_plane;
        epilogue_pair<P>(acc, acc2, j, b0, b1, a.acc_scale, act, form, a.dst, a.res, e, plane, has1, a.fmt);
      }
    }
  }
}

// ------------------------------------------------------------------------------- host side
struct TcOp : cpb::Prepared {
  TcOp() : Prepared(cpb::Route::TAP) {}
  TcArgs args;
  int BN, P;
  bool dcn;
  size_t smem;
};

template <int BN, bool DCN, int P>
int launch_tc(const TcOp &t, const TcArgs &args, cudaStream_t st) {
  return launch<conv_tc_kernel<BN, DCN, P>>(DCN ? "dcn_tc_kernel" : "conv_tc_kernel", args.total_tiles,
                                            DCN ? DCN_THREADS : TC_THREADS, t.smem, st, args);
}

}  // namespace

namespace tc {
EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}
int cur_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}
int num_sms() {
  static std::atomic<int> n[MAX_DEVICES];          // zero-initialised; per device (a process may drive several GPUs)
  const int dev = cur_device();
  if (dev < 0 || dev >= MAX_DEVICES) return 132;
  int v = n[dev].load(std::memory_order_relaxed);
  if (!v) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

bool tc_dtype(int d) { return d == CPB200_BF16 || d == CPB200_BF16X2 || d == CPB200_F16X2; }

Prec prec_of(const cpb200_op &op) {
  return {op.act_dtype == CPB200_BF16 ? 1 : 2, op.act_dtype == CPB200_F16X2 ? 1u : 0u, op.acc_scale != 0.f ? op.acc_scale : 1.f};
}

Slab slab_for(const int *cin, int nsrc) {
  int bk = 64;
  for (int s = 0; s < nsrc; ++s)
    if (cin[s] % 64) bk = (cin[s] % 32 == 0) ? (bk < 32 ? bk : 32) : 16;
  if (bk == 64) return {64, CU_TENSOR_MAP_SWIZZLE_128B, 1u};
  if (bk == 32) return {32, CU_TENSOR_MAP_SWIZZLE_64B, 2u};
  return {16, CU_TENSOR_MAP_SWIZZLE_32B, 3u};
}

int bn_for(int cout, int P) {
  int BN = 16;
  while (BN < cout && BN < 256) BN <<= 1;
  return P == 2 && BN > 128 ? 128 : BN;
}

int encode_act_map(CUtensorMap *map, const void *src, int C, int pitch, int W, int H, int B, int P, uint32_t fmt,
                   CUtensorMapSwizzle sw, const cuuint32_t (&box)[4], const cuuint32_t (&estr)[4], const char *what) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return cpb::fail(CPB200_ERR_STATE, "%s: cuTensorMapEncodeTiled unavailable", what);
  const cuuint64_t p = (cuuint64_t)pitch;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B * P};
  const cuuint64_t strides[3] = {p * 2, (cuuint64_t)W * p * 2, (cuuint64_t)H * W * p * 2};
  CUresult r = enc(map, fmt ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(src), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cpb::fail(CPB200_ERR_CUDA, "%s: cuTensorMapEncodeTiled(activations) failed: %d", what, (int)r);
  return CPB200_OK;
}

int encode_weight_map(CUtensorMap *map, const void *w, uint32_t fmt, int bk, int rows, int box_rows, long long blocks,
                      CUtensorMapSwizzle sw, const char *what) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return cpb::fail(CPB200_ERR_STATE, "%s: cuTensorMapEncodeTiled unavailable", what);
  const cuuint64_t dims[3] = {(cuuint64_t)bk, (cuuint64_t)rows, (cuuint64_t)blocks};
  const cuuint64_t strides[2] = {(cuuint64_t)bk * 2, (cuuint64_t)rows * bk * 2};
  const cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, fmt ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(w), dims,
                   strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cpb::fail(CPB200_ERR_CUDA, "%s: cuTensorMapEncodeTiled(weights) failed: %d", what, (int)r);
  return CPB200_OK;
}
}  // namespace tc

namespace cpb {

// CPB200_NO_PW=1 keeps pointwise convs on 2-D tiles (read when the program is prepared): both compute the same bits, so
// tests and timings can compare them in one process.
static bool pw_eligible(const cpb200_op &op) {
  if (const char *e = getenv("CPB200_NO_PW")) if (e[0] == '1') return false;
  if (op.type != CPB200_OP_CONV || op.kh != 1 || op.kw != 1 || op.stride != 1 || op.pad_h != 0 || op.pad_w != 0) return false;
  if (op.out_sy != 1 || op.out_sx != 1 || op.out_oy != 0 || op.out_ox != 0 || op.Hd != op.Ho || op.Wd != op.Wo) return false;
  if (op.H != op.Ho || op.W != op.Wo || (op.flags & CPB200_FLAG_OUT_NCHW_F32) || op.cout % 16) return false;
  return (long long)op.B * op.Ho * op.Wo < (1LL << 31);
}

int tap_prepare(const cpb200_op &op, Prepared **out) {
  const bool dcn = op.type == CPB200_OP_DCN;
  if (op.type != CPB200_OP_CONV && !dcn) return fail(CPB200_ERR_ARG, "tc: only CONV / DCN ops run on the tensor-core path");
  if (dcn && (op.kh != 3 || op.kw != 3 || op.stride != 1 || op.pad_h != 1 || op.pad_w != 1 || op.nsrc != 1 ||
              op.cin[0] % 64 || !op.aux || op.H != op.Ho || op.W != op.Wo))
    return fail(CPB200_ERR_ARG, "tc: DCN needs 3x3/s1/p1, one input with C %% 64 == 0 and the offset/mask tensor");
  if (!tc_dtype(op.act_dtype)) return fail(CPB200_ERR_ARG, "tc: bf16 or split (bf16x2 / fp16x2) activations required");
  if (op.stride < 1 || op.stride > 2) return fail(CPB200_ERR_ARG, "tc: stride %d", op.stride);
  if (op.Wo < 8 || op.Ho < 1) return fail(CPB200_ERR_ARG, "tc: output too small");
  int cin_total = 0;
  for (int s = 0; s < op.nsrc; ++s) {
    if (op.cin[s] % 16) return fail(CPB200_ERR_ARG, "tc: cin %d not a multiple of 16", op.cin[s]);
    cin_total += op.cin[s];
  }
  if (!(op.flags & (CPB200_FLAG_OUT_F32 | CPB200_FLAG_OUT_NCHW_F32)) && (op.cout % 16))
    return fail(CPB200_ERR_ARG, "tc: 16-bit output needs cout %% 16 == 0");
  const Prec pr = prec_of(op);
  const Slab sl = slab_for(op.cin, op.nsrc);
  const int P = pr.P, bk = sl.bk;
  const long long src_plane = (long long)op.B * op.H * op.W * op.cin[0];
  if (dcn && P == 2 && src_plane * 4 >= (1LL << 32))
    return fail(CPB200_ERR_ARG, "tc: split-precision DCN input must stay below 4 GiB (32-bit gather offsets)");
  // the bf16 gather builds its corner offsets in elements as signed ints: B*H*W*Cin must stay below 2^31
  if (dcn && P == 1 && src_plane >= (1LL << 31))
    return fail(CPB200_ERR_ARG, "tc: bf16 DCN input must stay below 2^31 elements (32-bit gather offsets)");
  const bool pw = !dcn && pw_eligible(op);
  int BN = bn_for(op.cout, P);
  // DCN: the gather warps leave 120 registers per thread, so a consumer holds at most 64 accumulator registers
  if (dcn && BN > 128 / P) BN = 128 / P;
  const size_t a_bytes = (size_t)P * TILE_M * bk * 2, b_bytes = ((size_t)P * BN * bk * 2 + 1023) / 1024 * 1024;
  // the DCN variant keeps 37 KB of sampling parameters in static smem; a pointwise conv takes the whole opt-in 227 KB
  // (less the alignment pad): every stage more is one more K block of A in flight across an epilogue
  const size_t budget = dcn ? 176 * 1024 : pw ? 226 * 1024 : 200 * 1024;
  int stages = (int)(budget / (a_bytes + b_bytes));
  if (stages > (pw ? MAX_STAGES : 8)) stages = pw ? MAX_STAGES : 8;
  if (dcn && stages > 4) stages = 4;      // leave the rest of the 256 KB to L1: the 9 taps x 4 corners re-read one ~30 KB footprint
  if (stages < 2) return fail(CPB200_ERR_ARG, "tc: tile does not fit shared memory");

  std::unique_ptr<TcOp> t(new TcOp());
  TcArgs &a = t->args;
  memset(&a, 0, sizeof(a));
  t->P = P; t->BN = BN; t->dcn = dcn;
  t->smem = stages * (a_bytes + b_bytes) + 1024;
  a.fmt = pr.fmt; a.acc_scale = pr.acc_scale;
  for (int s = 0; s < op.nsrc; ++s) a.cin[s] = op.cin[s];
  a.nsrc = op.nsrc; a.BK = bk; a.swizzle_bits = sl.layout; a.stages = stages;
  a.kh = op.kh; a.kw = op.kw; a.stride = op.stride; a.pad_h = op.pad_h; a.pad_w = op.pad_w;
  a.B = op.B; a.Ho = op.Ho; a.Wo = op.Wo;
  a.TW = op.Wo >= 16 ? 16 : 8; a.TH = TILE_M / a.TW;
  a.Hd = op.Hd; a.Wd = op.Wd;
  int map_w = op.W, map_h = op.H;
  if (pw) {                 // one 1 x (B*H*W) image of 1 x 128 tiles
    a.B = 1; a.Ho = a.Hd = map_h = 1; a.Wo = a.Wd = map_w = op.B * op.Ho * op.Wo;
    a.TW = TILE_M; a.TH = 1;
    a.vec8 = 1;
  }
  a.tiles_h = (a.Ho + a.TH - 1) / a.TH; a.tiles_w = (a.Wo + a.TW - 1) / a.TW;
  a.dcn_src = static_cast<const __nv_bfloat16 *>(op.src[0]);
  a.H = op.H; a.W = op.W; a.om_pitch = op.aux_pitch > 0 ? op.aux_pitch : 27;
  a.sy = op.out_sy; a.sx = op.out_sx; a.oy = op.out_oy; a.ox = op.out_ox;
  a.n_tiles = (op.cout + BN - 1) / BN;
  a.cout = op.cout; a.cout_store = op.cout;
  a.out_ch_off = op.out_ch_off; a.out_ch_total = op.out_ch_total;
  a.total_tiles = a.B * a.tiles_h * a.tiles_w * a.n_tiles;
  a.flags = op.flags;
  a.dst_plane = (long long)op.B * op.Hd * op.Wd * op.cout;
  a.src_plane = src_plane;
  a.wplane = op.kh * op.kw * (cin_total / bk);
  for (int s = 0; s < op.nsrc && !dcn; ++s) {
    // a channel slice of a wider tensor: op.src[s] already points at the slice
    const cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)(a.TW * op.stride), (cuuint32_t)(a.TH * op.stride), 1};
    const cuuint32_t estr[4] = {1, (cuuint32_t)op.stride, (cuuint32_t)op.stride, 1};
    if (int rc = encode_act_map(&a.amap[s], op.src[s], op.cin[s], op.src_pitch[s] > 0 ? op.src_pitch[s] : op.cin[s], map_w, map_h,
                                a.B, P, pr.fmt, sl.swizzle, box, estr, "tc"))
      return rc;
  }
  if (int rc = encode_weight_map(&a.bmap, op.weight, pr.fmt, bk, (op.cout + 15) / 16 * 16, BN, (long long)P * a.wplane, sl.swizzle, "tc"))
    return rc;
  *out = t.release();
  return CPB200_OK;
}

int tap_run(const Prepared &p, const cpb200_op &op, cudaStream_t st) {
  const TcOp &t = static_cast<const TcOp &>(p);
  // input activations and weights are baked into the tensor maps; the rest comes from the live op (tc_common.cuh: Route)
  TcArgs args = t.args;
  args.dst = op.dst; args.res = op.res; args.bias = op.bias;
  args.dcn_om = static_cast<const float *>(op.aux);
  if (args.vec8 && ((reinterpret_cast<uintptr_t>(op.dst) | reinterpret_cast<uintptr_t>(op.res)) & 15))
    return fail(CPB200_ERR_ARG, "tc: a pointwise conv's dst and res must be 16-byte aligned (16-byte epilogue stores)");
#define TC_CASE(N, D)                                                                                  \
  case N: return t.P == 2 ? launch_tc<N, D, 2>(t, args, st) : launch_tc<N, D, 1>(t, args, st);
  if (t.dcn) {
    switch (t.BN) {
      TC_CASE(16, true) TC_CASE(32, true) TC_CASE(64, true)
      case 128: if (t.P == 1) return launch_tc<128, true, 1>(t, args, st); break;
    }
  } else {
    switch (t.BN) {
      TC_CASE(16, false) TC_CASE(32, false) TC_CASE(64, false) TC_CASE(128, false)
      case 256: if (t.P == 1) return launch_tc<256, false, 1>(t, args, st); break;
    }
  }
#undef TC_CASE
  return fail(CPB200_ERR_STATE, "tc: bad BN");
}

}  // namespace cpb

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
// [A_hi | A_lo | W_hi | W_lo]; per K step the consumers issue three N = BN products: A_hi x W_hi into one accumulator array,
// A_hi x W_lo and A_lo x W_hi into a second one (added in the epilogue).  Separate arrays keep the wgmma of one K step
// independent of each other, so ptxas does not serialise them.
// The DCN gather blends the four corners of BOTH planes in fp32 and re-splits the sample.
#include <type_traits>
#include "tc_common.cuh"
#include <mutex>
#include <cstdlib>

namespace {

constexpr int CONS_THREADS = 256;      // two consumer warpgroups
constexpr int TC_THREADS = CONS_THREADS + 32;        // + TMA producer warp
constexpr int TILE_M = 128;

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
  __shared__ __align__(8) uint64_t bars[2 * 8];
  __shared__ DcnPrm s_prm[DCN ? DCN_GW : 1][DCN ? 9 : 1][DCN ? DCN_ROWS : 1];
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[8]);

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
    const bool out_f32 = a.flags & CPB200_FLAG_OUT_F32;
    const bool out_nchw = a.flags & CPB200_FLAG_OUT_NCHW_F32;
    float acc[BN / 2], acc2[P == 2 ? BN / 2 : 1];                 // hi x W_hi | hi x W_lo + lo x W_hi (split operands)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (P == 2 ? BN / 2 : 1); ++i) acc2[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    for (int tt = blockIdx.x; tt < a.total_tiles; tt += gridDim.x) {
      int prev = -1;                                       // stage whose MMAs may still be running
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(full0 + 8 * stage, phase);
        const uint64_t sd = dT + (base14 + (uint32_t)stage * sstep);
        const uint64_t ad = sd + aoff, bd = sd + boff;
        wg_fence();
        for (int k = 0; k < ksteps; ++k) {
          const uint32_t first = (kb > 0 || k > 0) ? 1u : 0u;
          if constexpr (P == 1) {
            wgmma_k16<BN>(acc, ad + 2 * k, bd + 2 * k, first, 1u);
          } else {
            wgmma_k16<BN>(acc, ad + 2 * k, bd + 2 * k, first, bf);                     // A_hi x W_hi
            wgmma_k16<BN>(acc2, ad + 2 * k, bd + bplane + 2 * k, first, bf);           // A_hi x W_lo
            // A_lo x W_hi joins the other small term (see net_tc3.cu: the fp32 accumulator truncates per instruction in
            // proportion to its magnitude)
            wgmma_k16<BN>(acc2, ad + aplane + 2 * k, bd + 2 * k, 1u, bf);
          }
        }
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
#pragma unroll
      for (int j = 0; j < BN / 4; ++j) {                   // pairs of adjacent columns of this thread's fragment
        const int row = wg * 64 + frag_row(t, j), nb = n0 + frag_col(t, j);
        const int ho = h0 + row / a.TW, wo = w0 + row % a.TW;
        if (ho >= a.Ho || wo >= a.Wo || nb >= a.cout) continue;
        float v0 = acc[2 * j], v1 = acc[2 * j + 1];
        if constexpr (P == 2) { v0 += acc2[2 * j]; v1 += acc2[2 * j + 1]; }
        const bool has1 = nb + 1 < a.cout;
        const float b0 = a.bias ? __ldg(a.bias + nb) : 0.f, b1 = (a.bias && has1) ? __ldg(a.bias + nb + 1) : 0.f;
        const float f0 = P == 2 ? fmaf(v0, a.acc_scale, b0) : v0 + b0, f1 = P == 2 ? fmaf(v1, a.acc_scale, b1) : v1 + b1;
        const size_t pix = ((size_t)n * a.Hd + (ho * a.sy + a.oy)) * a.Wd + (wo * a.sx + a.ox);
        if (out_nchw) {
          // head outputs: NCHW fp32 channel slice of dst
          float *o = static_cast<float *>(a.dst) +
                     (((size_t)n * a.out_ch_total + a.out_ch_off + nb) * a.Hd + (ho * a.sy + a.oy)) * a.Wd + (wo * a.sx + a.ox);
          const size_t plane = (size_t)a.Hd * a.Wd;
          o[0] = P == 2 ? cpb::act_fn(f0, act) : cpb::act_out<__nv_bfloat16>(f0, act);
          if (has1) o[plane] = P == 2 ? cpb::act_fn(f1, act) : cpb::act_out<__nv_bfloat16>(f1, act);
        } else if (out_f32) {
          float *o = static_cast<float *>(a.dst) + pix * a.cout_store + nb;
          o[0] = cpb::act_out<__nv_bfloat16>(f0, act);
          if (has1) o[1] = cpb::act_out<__nv_bfloat16>(f1, act);
        } else {
          store_pair16<P>(a.dst, a.res, pix * a.cout_store + nb, a.dst_plane, f0, f1, act, a.fmt);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------- host side
struct TcOp {
  TcArgs args;
  int BN, P;
  bool dcn;
  void *c3 = nullptr;      // halo-reuse 3x3 kernel handle (net_tc3.cu) when that path was chosen
  int grid;
  size_t smem;
};


template <int BN, bool DCN, int P>
int launch_tc(const TcOp &t, const TcArgs &args, cudaStream_t st) {
  static SmemAttrCache cache;
  if (int rc = ensure_smem(conv_tc_kernel<BN, DCN, P>, t.smem, cache)) return rc;
  conv_tc_kernel<BN, DCN, P><<<t.grid, DCN ? DCN_THREADS : TC_THREADS, t.smem, st>>>(args);
  return cpb::check_launch(DCN ? "dcn_tc_kernel" : "conv_tc_kernel");
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
}  // namespace tc

namespace cpb {

bool c3_eligible(const cpb200_op &op);
void *c3_prepare(const cpb200_op &op, int *rc);
void c3_release(void *h);
int c3_run(const void *h, const cpb200_op &op, cudaStream_t st);

static bool halo_enabled() {
  const char *e = getenv("CPB200_TC_HALO");
  return !(e && e[0] == '0');
}

int tc_prepare_op(cpb200_op &op) {
  if (halo_enabled() && c3_eligible(op)) {
    int rc = CPB200_OK;
    void *h = c3_prepare(op, &rc);
    if (!h) return rc;
    TcOp *t = new TcOp();
    t->c3 = h;
    op.tc = t;
    return CPB200_OK;
  }
  const bool dcn = op.type == CPB200_OP_DCN;
  if (op.type != CPB200_OP_CONV && !dcn) return fail(CPB200_ERR_ARG, "tc: only CONV / DCN ops run on the tensor-core path");
  if (dcn && (op.kh != 3 || op.kw != 3 || op.stride != 1 || op.pad_h != 1 || op.pad_w != 1 || op.nsrc != 1 ||
              op.cin[0] % 64 || !op.aux || op.H != op.Ho || op.W != op.Wo))
    return fail(CPB200_ERR_ARG, "tc: DCN needs 3x3/s1/p1, one input with C %% 64 == 0 and the offset/mask tensor");
  if (op.act_dtype != CPB200_BF16 && op.act_dtype != CPB200_BF16X2 && op.act_dtype != CPB200_F16X2)
    return fail(CPB200_ERR_ARG, "tc: bf16 or split (bf16x2 / fp16x2) activations required");
  if (op.stride < 1 || op.stride > 2) return fail(CPB200_ERR_ARG, "tc: stride %d", op.stride);
  if (op.Wo < 8 || op.Ho < 1) return fail(CPB200_ERR_ARG, "tc: output too small");
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(CPB200_ERR_STATE, "tc: cuTensorMapEncodeTiled unavailable");
  const int g_num_sms = tc::num_sms();
  TcOp *t = new TcOp();
  TcArgs &a = t->args;
  memset(&a, 0, sizeof(a));
  const int P = op.act_dtype == CPB200_BF16 ? 1 : 2;
  t->P = P;
  a.fmt = op.act_dtype == CPB200_F16X2 ? 1u : 0u;
  a.acc_scale = op.acc_scale != 0.f ? op.acc_scale : 1.f;
  int cin_total = 0, bk = 64;
  for (int s = 0; s < op.nsrc; ++s) {
    const int c = op.cin[s];
    if (c % 16) { delete t; return fail(CPB200_ERR_ARG, "tc: cin %d not a multiple of 16", c); }
    if (c % 64) bk = (c % 32 == 0) ? (bk < 32 ? bk : 32) : 16;
    a.cin[s] = c; cin_total += c;
  }
  a.nsrc = op.nsrc; a.BK = bk;
  const CUtensorMapSwizzle sw = bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  a.swizzle_bits = bk == 64 ? 1u : bk == 32 ? 2u : 3u;
  a.kh = op.kh; a.kw = op.kw; a.stride = op.stride; a.pad_h = op.pad_h; a.pad_w = op.pad_w;
  a.B = op.B; a.Ho = op.Ho; a.Wo = op.Wo;
  a.TW = op.Wo >= 16 ? 16 : 8; a.TH = TILE_M / a.TW;
  a.tiles_h = (op.Ho + a.TH - 1) / a.TH; a.tiles_w = (op.Wo + a.TW - 1) / a.TW;
  int BN = 16;
  while (BN < op.cout && BN < 256) BN <<= 1;
  if (P == 2 && BN > 128) BN = 128;            // split operands: two accumulator halves of BN columns each (2 * BN <= 256)
  // DCN: the gather warps leave 120 registers per thread, so a consumer holds at most 64 accumulator registers
  if (dcn && BN > 128 / P) BN = 128 / P;
  t->BN = BN; t->dcn = dcn;
  a.dcn_src = static_cast<const __nv_bfloat16 *>(op.src[0]); a.dcn_om = static_cast<const float *>(op.aux);
  a.H = op.H; a.W = op.W; a.om_pitch = op.aux_pitch > 0 ? op.aux_pitch : 27;
  a.Hd = op.Hd; a.Wd = op.Wd; a.sy = op.out_sy; a.sx = op.out_sx; a.oy = op.out_oy; a.ox = op.out_ox;
  a.n_tiles = (op.cout + BN - 1) / BN;
  a.cout = op.cout; a.cout_store = op.cout;
  if (!(op.flags & (CPB200_FLAG_OUT_F32 | CPB200_FLAG_OUT_NCHW_F32)) && (op.cout % 16)) { delete t; return fail(CPB200_ERR_ARG, "tc: 16-bit output needs cout %% 16 == 0"); }
  a.out_ch_off = op.out_ch_off; a.out_ch_total = op.out_ch_total;
  a.total_tiles = op.B * a.tiles_h * a.tiles_w * a.n_tiles;
  a.dst = op.dst; a.res = op.res; a.bias = op.bias; a.flags = op.flags;
  a.dst_plane = (long long)op.B * op.Hd * op.Wd * op.cout;
  a.src_plane = (long long)op.B * op.H * op.W * op.cin[0];
  if (dcn && P == 2 && a.src_plane * 4 >= (1LL << 32)) { delete t;
    return fail(CPB200_ERR_ARG, "tc: split-precision DCN input must stay below 4 GiB (32-bit gather offsets)"); }
  a.wplane = op.kh * op.kw * (cin_total / bk);
  const size_t a_bytes = (size_t)P * TILE_M * bk * 2, b_bytes = ((size_t)P * BN * bk * 2 + 1023) / 1024 * 1024;
  const size_t budget = dcn ? 176 * 1024 : 200 * 1024;     // the DCN variant keeps 37 KB of sampling parameters in static smem
  int stages = (int)(budget / (a_bytes + b_bytes));
  if (stages > 8) stages = 8;
  if (dcn && stages > 4) stages = 4;      // leave the rest of the 256 KB to L1: the 9 taps x 4 corners re-read one ~30 KB footprint
  if (stages < 2) { delete t; return fail(CPB200_ERR_ARG, "tc: tile does not fit shared memory"); }
  a.stages = stages;
  t->smem = stages * (a_bytes + b_bytes) + 1024;
  t->grid = a.total_tiles < g_num_sms ? a.total_tiles : g_num_sms;
  const CUtensorMapDataType dt = a.fmt ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;

  for (int s = 0; s < op.nsrc && !dcn; ++s) {
    // a channel slice of a wider tensor: `pitch` elements between pixels, op.src[s] already points at the slice.
    // Split activations: the lo plane follows the hi plane of the (parent) tensor, i.e. a batch of 2B images.
    const cuuint64_t pitch = op.src_pitch[s] > 0 ? (cuuint64_t)op.src_pitch[s] : (cuuint64_t)op.cin[s];
    const cuuint64_t dims[4] = {(cuuint64_t)op.cin[s], (cuuint64_t)op.W, (cuuint64_t)op.H, (cuuint64_t)op.B * P};
    const cuuint64_t strides[3] = {pitch * 2, (cuuint64_t)op.W * pitch * 2, (cuuint64_t)op.H * op.W * pitch * 2};
    const cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)(a.TW * op.stride), (cuuint32_t)(a.TH * op.stride), 1};
    const cuuint32_t estr[4] = {1, (cuuint32_t)op.stride, (cuuint32_t)op.stride, 1};
    CUresult r = enc(&a.amap[s], dt, 4, const_cast<void *>(op.src[s]), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { delete t; return fail(CPB200_ERR_CUDA, "tc: cuTensorMapEncodeTiled(A[%d]) failed: %d", s, (int)r); }
  }
  {
    // weights are packed slab-major [plane][tap][K-slab][cout_pad][bk] (plan.py::_pack_conv_tc): a box is one dense run
    const int cout_pad = (op.cout + 15) / 16 * 16;
    const cuuint64_t dims[3] = {(cuuint64_t)bk, (cuuint64_t)cout_pad, (cuuint64_t)(op.kh * op.kw) * (cuuint64_t)(cin_total / bk) * P};
    const cuuint64_t strides[2] = {(cuuint64_t)bk * 2, (cuuint64_t)cout_pad * bk * 2};
    const cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)BN, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&a.bmap, dt, 3, const_cast<void *>(op.weight), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { delete t; return fail(CPB200_ERR_CUDA, "tc: cuTensorMapEncodeTiled(B) failed: %d", (int)r); }
  }
  op.tc = t;
  return CPB200_OK;
}

int tc_release_op(cpb200_op &op) {
  TcOp *t = static_cast<TcOp *>(op.tc);
  if (t && t->c3) c3_release(t->c3);
  delete t;
  op.tc = nullptr;
  return CPB200_OK;
}

int tc_run_op(const cpb200_op &op, cudaStream_t st) {
  const TcOp *t = static_cast<const TcOp *>(op.tc);
  if (!t) return fail(CPB200_ERR_STATE, "tc: op not prepared");
  if (t->c3) return c3_run(t->c3, op, st);
  // dst / res / bias / the DCN offset tensor are taken from the live op: the model binds new output tensors every
  // forward (include/centerpose_b200.h); input activations and weights were baked into the tensor maps at prepare.
  TcArgs args = t->args;
  args.dst = op.dst; args.res = op.res; args.bias = op.bias;
  args.dcn_om = static_cast<const float *>(op.aux);
#define TC_CASE(N, D)                                                                                  \
  case N: return t->P == 2 ? launch_tc<N, D, 2>(*t, args, st) : launch_tc<N, D, 1>(*t, args, st);
  if (t->dcn) {
    switch (t->BN) {
      TC_CASE(16, true) TC_CASE(32, true) TC_CASE(64, true)
      case 128: if (t->P == 1) return launch_tc<128, true, 1>(*t, args, st); break;
    }
    return fail(CPB200_ERR_STATE, "tc: DCN supports cout tiles of 16..128 (bf16) / 16..64 (split) only");
  }
  switch (t->BN) {
    TC_CASE(16, false) TC_CASE(32, false) TC_CASE(64, false) TC_CASE(128, false)
    case 256: if (t->P == 1) return launch_tc<256, false, 1>(*t, args, st); break;
  }
#undef TC_CASE
  return fail(CPB200_ERR_STATE, "tc: bad BN");
}

}  // namespace cpb

// All keypoint heads in one kernel: per head  out = conv1x1(relu(conv3x3(x)))  with the hidden map kept in registers.
//
// Unfused, every head's 3x3 conv writes a (B, H, W, hidden) map (split precisions: two 16-bit planes) that its 1x1 conv
// reads back once; at DLA-34 512x512 B=32 that round trip is 2 x 537 MB per head.  Here a CTA owns a 16 x 8 pixel tile:
//   * the (16+2) x (8+2) input halo of every K slab is loaded ONCE per tile by TMA and read by all nine taps of every head
//     through shifted wgmma descriptors (the halo scheme of net_tc3.cu);
//   * per head and per chunk of 128 hidden channels the 3x3 GEMM runs exactly as conv3x3_tc_kernel does (slab outer, tap
//     inner, then k steps; split precisions: A_hi x W_hi into `acc`, A_hi x W_lo + A_lo x W_hi into `acc2`);
//   * the chunk epilogue (acc_scale, bias, ReLU, the hi / lo split or the bf16 round) runs on the accumulator registers,
//     and the results ARE the A operand of the 1x1 GEMM: the 64 x 16 column block k of a wgmma accumulator has the
//     thread / register layout of the A register fragment of wgmma k16 (tc_common.cuh frag_row / frag_col), so the 1x1
//     products are register-A ("RS") wgmmas with the chunk's 1x1 weights in shared memory;
//   * the 1x1 accumulators (N = the head's channels padded to 16, at most 48) collect the chunks in the k order of
//     conv_tc_kernel, and the head epilogue stores NCHW fp32 like conv_tc_kernel's out_nchw branch.
// The same products are summed in the same order as the unfused 3x3 + 1x1 pair, so the head maps are bit-identical.
//
// Warps: warpgroup 0 = producers (warp 0 halo, warp 1 weights: the 3x3 weight tiles and each chunk's 1x1 weights
// through one ring), warpgroups 1-2 = consumers (rows 0-63 / 64-127 of the tile).  A consumer holds 128 hidden-chunk
// accumulators, 48 head accumulators and the 64 fragment registers of the chunk, so the producers give their registers
// away (setmaxnreg).
#include "tc_common.cuh"
#include <memory>

using namespace tc;

namespace {

constexpr int HD_THREADS = 384;
constexpr int HD_CONS = 256;
constexpr int HD_MAX = 8;                      // heads per op
constexpr int HD_CHUNK = 128;                  // hidden channels per chunk
constexpr int HD_MAXN = 48;                    // widest head (channels padded to 16)
constexpr int HD_MAX_NB = 8;
constexpr int TW = 8, TH = 16, HW = TW + 2, HH = TH + 2;

struct alignas(64) HdArgs {
  CUtensorMap amap, wmap3, wmap1[HD_MAX];
  int nheads, hid, chunks, slabs, BK;
  int B, Ho, Wo, tiles_h, tiles_w, total_tiles;
  int nh, nb;                    // halo buffers (each holds every slab / plane of a tile), weight stages
  unsigned halo_stage_bytes, halo_tx_bytes, halo_buf_bytes, w_stage_bytes, w3_tile_bytes;
  unsigned swizzle_bits, fmt;
  const float *bias3;            // [head][hid]
  int cout[HD_MAX], npad[HD_MAX];
  const float *bias1[HD_MAX];
  float scale3[HD_MAX], scale1[HD_MAX];
  float *dst[HD_MAX];
};

template <int R>
__device__ __forceinline__ void reg_fence(uint32_t (&r)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// The 1x1 products of one hidden chunk: 8 k steps of 16 channels, weights [slab of 64][plane][N rows][64] (128B swizzle).
template <int N, int P>
__device__ __forceinline__ void heads_1x1(float (&out)[HD_MAXN / 2], float (&out2)[P == 2 ? HD_MAXN / 2 : 1],
                                          const uint32_t (&ahi)[32], const uint32_t (&alo)[P == 2 ? 32 : 1],
                                          uint32_t w_lo14, bool first_chunk, uint32_t bf) {
  const uint64_t dW = desc_sbo(0u, 1024u, 1u);
  constexpr uint32_t blk = (N * 128) >> 4;       // one (slab, plane) block
#pragma unroll
  for (int kk = 0; kk < HD_CHUNK / 16; ++kk) {
    const uint32_t s2 = kk >> 2, koff = 2u * (kk & 3);
    const uint64_t bh = dW + (w_lo14 + s2 * P * blk + koff), bl = bh + blk;
    const uint32_t first = (first_chunk && kk == 0) ? 0u : 1u;
    const uint32_t fh[4] = {ahi[4 * kk], ahi[4 * kk + 1], ahi[4 * kk + 2], ahi[4 * kk + 3]};
    if constexpr (P == 1) {
      mma_step_rs<N, 1>(out, out2, fh, fh, bh, bl, first, bf);
    } else {
      const uint32_t fl[4] = {alo[4 * kk], alo[4 * kk + 1], alo[4 * kk + 2], alo[4 * kk + 3]};
      mma_step_rs<N, 2>(out, out2, fh, fl, bh, bl, first, bf);
    }
  }
}

template <int P>
__global__ void __launch_bounds__(HD_THREADS, 1) heads_tc_kernel(const __grid_constant__ HdArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t h_base = smem_base, w_base = smem_base + a.nh * a.halo_buf_bytes;
  __shared__ __align__(8) uint64_t bars[4 + 2 * HD_MAX_NB];
  const uint32_t hfull0 = smem_u32(&bars[0]), hempty0 = smem_u32(&bars[2]);
  const uint32_t wfull0 = smem_u32(&bars[4]), wempty0 = smem_u32(&bars[4 + HD_MAX_NB]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tmap_prefetch(&a.amap); tmap_prefetch(&a.wmap3);
    for (int s = 0; s < 2; ++s) { mbar_init(hfull0 + 8 * s, 1); mbar_init(hempty0 + 8 * s, HD_CONS / 32); }
    for (int s = 0; s < HD_MAX_NB; ++s) { mbar_init(wfull0 + 8 * s, 1); mbar_init(wempty0 + 8 * s, HD_CONS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto tile_at = [&](int it, int &n, int &h0, int &w0) -> bool {
    int t = blockIdx.x + it * gridDim.x;
    if (t >= a.total_tiles) return false;
    const int tw = t % a.tiles_w; t /= a.tiles_w;
    const int th = t % a.tiles_h; n = t / a.tiles_h;
    h0 = th * TH; w0 = tw * TW;
    return true;
  };

  // warpgroup index made warp-uniform for the compiler (setmaxnreg must be executed by whole warpgroups)
  const int wgi = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);
  if (wgi == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && elect_one()) {
      // =============================== halo producer ===============================
      int s = 0; uint32_t ph = 0;
      int n, h0, w0;
      for (int it = 0; tile_at(it, n, h0, w0); ++it) {
        mbar_wait(hempty0 + 8 * s, ph ^ 1);
        mbar_expect_tx(hfull0 + 8 * s, (uint32_t)(a.slabs * P) * a.halo_tx_bytes);
        for (int sl = 0; sl < a.slabs; ++sl)
#pragma unroll
          for (int pl = 0; pl < P; ++pl)
            tma_load_4d(h_base + s * a.halo_buf_bytes + (sl * P + pl) * a.halo_stage_bytes, &a.amap, hfull0 + 8 * s,
                        sl * a.BK, w0 - 1, h0 - 1, n + pl * a.B);
        if (++s == a.nh) { s = 0; ph ^= 1; }
      }
    } else if (warp == 1 && elect_one()) {
      // =============================== weight producer ===============================
      for (int h = 0; h < a.nheads; ++h) tmap_prefetch(&a.wmap1[h]);
      const int wplane = 9 * a.slabs;                      // 3x3 weight blocks per head and plane
      const int slabs1 = a.hid / 64;                       // 1x1 weight blocks per plane
      int sb = 0; uint32_t phb = 0;
      int n, h0, w0;
      for (int it = 0; tile_at(it, n, h0, w0); ++it) {
        for (int h = 0; h < a.nheads; ++h) {
          for (int c = 0; c < a.chunks; ++c) {
            for (int sl = 0; sl < a.slabs; ++sl)
              for (int tap = 0; tap < 9; ++tap) {
                mbar_wait(wempty0 + 8 * sb, phb ^ 1);
                mbar_expect_tx(wfull0 + 8 * sb, P * a.w3_tile_bytes);
#pragma unroll
                for (int pl = 0; pl < P; ++pl)
                  tma_load_3d(w_base + sb * a.w_stage_bytes + pl * a.w3_tile_bytes, &a.wmap3, wfull0 + 8 * sb, 0, c * HD_CHUNK,
                              (h * P + pl) * wplane + tap * a.slabs + sl);
                if (++sb == a.nb) { sb = 0; phb ^= 1; }
              }
            const uint32_t blk = (uint32_t)a.npad[h] * 128u;
            mbar_wait(wempty0 + 8 * sb, phb ^ 1);
            mbar_expect_tx(wfull0 + 8 * sb, 2u * P * blk);
            for (int s2 = 0; s2 < 2; ++s2)
#pragma unroll
              for (int pl = 0; pl < P; ++pl)
                tma_load_3d(w_base + sb * a.w_stage_bytes + (s2 * P + pl) * blk, &a.wmap1[h], wfull0 + 8 * sb, 0, 0,
                            pl * slabs1 + c * 2 + s2);
            if (++sb == a.nb) { sb = 0; phb ^= 1; }
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    // =============================== consumers ===============================
    const int wg = (warp >> 2) - 1, t = threadIdx.x & 127;
    const uint32_t bf = (P == 1 || a.fmt == 0) ? 1u : 0u;
    const int ksteps = a.BK / 16;
    const uint32_t pix_bytes = a.BK * 2, pstep = pix_bytes >> 4, rowstep = HW * pstep;
    const uint64_t dA = desc_sbo(0u, HW * pix_bytes, a.swizzle_bits), dB = desc_sbo(0u, 8 * pix_bytes, a.swizzle_bits);
    const uint32_t a_lo14 = ((h_base & 0x3FFFFu) >> 4) + (uint32_t)wg * 8u * rowstep;      // 8 halo rows per warpgroup
    const uint32_t w_lo14 = (w_base & 0x3FFFFu) >> 4;
    const uint32_t hstage = a.halo_stage_bytes >> 4, hbufstep = a.halo_buf_bytes >> 4;
    const uint32_t wstep = a.w_stage_bytes >> 4, wtile = a.w3_tile_bytes >> 4;
    // The accumulators are (re)defined where each chunk / head starts: the MMAs' first instruction overwrites them
    // anyway, and a fresh definition ends the previous chunk's values once they are converted, so the 3x3 accumulators
    // do not stay live beside the fragments and the head accumulators during the 1x1 products.
    float acc[HD_CHUNK / 2], acc2[P == 2 ? HD_CHUNK / 2 : 1];
    float out[HD_MAXN / 2], out2[P == 2 ? HD_MAXN / 2 : 1];
    int hs = 0; uint32_t phh = 0; int sb = 0; uint32_t phb = 0;
    int n, h0, w0;
    for (int it = 0; tile_at(it, n, h0, w0); ++it) {
      mbar_wait(hfull0 + 8 * hs, phh);
      const uint32_t hbuf = a_lo14 + (uint32_t)hs * hbufstep;
      for (int h = 0; h < a.nheads; ++h) {
        const int npad = a.npad[h];
        acc_zero(out, out2);
        for (int c = 0; c < a.chunks; ++c) {
          acc_zero(acc, acc2);
          // ---- 3x3 GEMM of hidden channels [c * 128, c * 128 + 128) ----
          uint32_t accf = 0u;
          int prev = -1;
          for (int sl = 0; sl < a.slabs; ++sl) {
            const uint64_t ah0 = dA + (hbuf + (uint32_t)(sl * P) * hstage), al0 = ah0 + (P == 2 ? hstage : 0u);
            for (int tap = 0; tap < 9; ++tap) {
              const int r = tap / 3, q = tap - r * 3;
              const uint32_t toff = (uint32_t)r * rowstep + (uint32_t)q * pstep;
              mbar_wait(wfull0 + 8 * sb, phb);
              const uint64_t bd = dB + (w_lo14 + (uint32_t)sb * wstep);
              const uint64_t adh = ah0 + toff, adl = al0 + toff;
              wg_fence();
              for (int k = 0; k < ksteps; ++k)
                mma_step<HD_CHUNK, P>(acc, acc2, adh, adl, bd, bd + wtile, k, k == 0 ? accf : 1u, bf);
              accf = 1u;
              wg_commit();
              wg_wait<1>();
              if (prev >= 0 && lane == 0) mbar_arrive(wempty0 + 8 * prev);
              prev = sb;
              if (++sb == a.nb) { sb = 0; phb ^= 1; }
            }
          }
          wg_wait<0>();
          if (lane == 0) mbar_arrive(wempty0 + 8 * prev);
          acc_fence(acc); acc_fence(acc2);
          // ---- chunk epilogue: what conv3x3_tc_kernel's epilogue_pair stores, kept as 1x1 A fragments ----
          uint32_t ahi[32], alo[P == 2 ? 32 : 1];
          const float *b3 = a.bias3 + h * a.hid + c * HD_CHUNK;
          const float s3 = a.scale3[h];
#pragma unroll
          for (int j = 0; j < HD_CHUNK / 4; ++j) {
            const int col = frag_col(t, j);
            const float b0 = __ldg(b3 + col), b1 = __ldg(b3 + col + 1);
            if constexpr (P == 2) {
              const float f0 = fmaf(acc[2 * j] + acc2[2 * j], s3, b0), f1 = fmaf(acc[2 * j + 1] + acc2[2 * j + 1], s3, b1);
              split2(cpb::act_fast(f0, CPB200_FLAG_RELU), cpb::act_fast(f1, CPB200_FLAG_RELU), a.fmt, ahi[j], alo[j]);
            } else {
              const __nv_bfloat162 v = __floats2bfloat162_rn(cpb::act_out<__nv_bfloat16>(acc[2 * j] + b0, CPB200_FLAG_RELU),
                                                             cpb::act_out<__nv_bfloat16>(acc[2 * j + 1] + b1, CPB200_FLAG_RELU));
              ahi[j] = *reinterpret_cast<const uint32_t *>(&v);
            }
          }
          // ---- 1x1 GEMM of the chunk into the head's accumulators ----
          mbar_wait(wfull0 + 8 * sb, phb);
          const uint32_t w1 = w_lo14 + (uint32_t)sb * wstep;
          wg_fence();
          if (npad == 16) heads_1x1<16, P>(out, out2, ahi, alo, w1, c == 0, bf);
          else if (npad == 32) heads_1x1<32, P>(out, out2, ahi, alo, w1, c == 0, bf);
          else heads_1x1<48, P>(out, out2, ahi, alo, w1, c == 0, bf);
          wg_commit();
          wg_wait<0>();
          reg_fence(ahi); reg_fence(alo);                   // the MMAs read them asynchronously
          if (lane == 0) mbar_arrive(wempty0 + 8 * sb);
          if (++sb == a.nb) { sb = 0; phb ^= 1; }
        }
        acc_fence(out); acc_fence(out2);
        // ---- head epilogue: NCHW fp32, as conv_tc_kernel stores it ----
        const int cout = a.cout[h];
        const float *b1p = a.bias1[h];
        const float s1 = a.scale1[h];
        float *dst = a.dst[h];
        const long long plane = (long long)a.Ho * a.Wo;
#pragma unroll
        for (int j = 0; j < HD_MAXN / 4; ++j) {
          const int row = wg * 64 + frag_row(t, j), nb = frag_col(t, j);
          const int ho = h0 + (row >> 3), wo = w0 + (row & 7);
          if (4 * j >= npad || ho >= a.Ho || wo >= a.Wo || nb >= cout) continue;
          const bool has1 = nb + 1 < cout;
          const float b0 = __ldg(b1p + nb), b1 = has1 ? __ldg(b1p + nb + 1) : 0.f;
          epilogue_pair<P>(out, out2, j, b0, b1, s1, 0u, OUT_NCHW, dst, nullptr, (((size_t)n * cout + nb) * a.Ho + ho) * a.Wo + wo,
                           plane, has1, a.fmt);
        }
      }
      if (lane == 0) mbar_arrive(hempty0 + 8 * hs);
      if (++hs == a.nh) { hs = 0; phh ^= 1; }
    }
  }
}

struct HdOp : cpb::Prepared {
  HdOp() : Prepared(cpb::Route::HEADS) {}
  HdArgs args;
  int P;
  size_t smem;
};

}  // namespace

namespace cpb {

int heads_prepare(const cpb200_op &op, Prepared **out) {
  const cpb200_head *hd = static_cast<const cpb200_head *>(op.aux);
  const int nheads = op.aux_pitch;
  if (!hd || nheads < 1 || nheads > HD_MAX) return fail(CPB200_ERR_ARG, "heads: 1..%d head entries required", HD_MAX);
  if (!tc_dtype(op.act_dtype)) return fail(CPB200_ERR_ARG, "heads: bf16 or split (bf16x2 / fp16x2) activations required");
  if (op.nsrc != 1 || op.cin[0] % 16 || op.cin[0] > 64 || (op.src_pitch[0] != 0 && op.src_pitch[0] != op.cin[0]))
    return fail(CPB200_ERR_ARG, "heads: one dense input with C %% 16 == 0 and C <= 64 required");
  if (op.kh != 3 || op.kw != 3 || op.stride != 1 || op.pad_h != 1 || op.pad_w != 1 || op.H != op.Ho || op.W != op.Wo ||
      op.Ho < 8 || op.Wo < 8)
    return fail(CPB200_ERR_ARG, "heads: 3x3 / stride 1 / pad 1 over maps of at least 8 x 8 required");
  const int hid = hd[0].hidden;
  if (hid <= 0 || hid % HD_CHUNK) return fail(CPB200_ERR_ARG, "heads: hidden width %d is not a multiple of %d", hid, HD_CHUNK);
  std::unique_ptr<HdOp> t(new HdOp());
  HdArgs &a = t->args;
  memset(&a, 0, sizeof(a));
  const Prec pr = prec_of(op);
  const int P = pr.P;
  t->P = P;
  a.fmt = pr.fmt;
  a.nheads = nheads; a.hid = hid; a.chunks = hid / HD_CHUNK;
  int npad_max = 16;
  for (int h = 0; h < nheads; ++h) {
    if (hd[h].hidden != hid || hd[h].cout < 1 || hd[h].cout > HD_MAXN || !hd[h].weight || !hd[h].bias)
      return fail(CPB200_ERR_ARG, "heads: entry %d: same hidden width, 1..%d channels, weight and bias required", h, HD_MAXN);
    a.cout[h] = hd[h].cout; a.npad[h] = (hd[h].cout + 15) / 16 * 16;
    if (a.npad[h] > npad_max) npad_max = a.npad[h];
    a.scale3[h] = hd[h].acc_scale3 != 0.f ? hd[h].acc_scale3 : 1.f;
    a.scale1[h] = hd[h].acc_scale1 != 0.f ? hd[h].acc_scale1 : 1.f;
    // 1x1 weights as packed for a 1x1 conv over the hidden channels (K slab 64): [plane][hid / 64][npad][64]
    if (int rc = encode_weight_map(&a.wmap1[h], hd[h].weight, pr.fmt, 64, a.npad[h], a.npad[h], (long long)(hid / 64) * P,
                                   CU_TENSOR_MAP_SWIZZLE_128B, "heads (1x1)"))
      return rc;
  }
  const Slab sl = slab_for(op.cin, 1);
  const int bk = sl.bk;
  a.BK = bk; a.slabs = op.cin[0] / bk;
  a.swizzle_bits = sl.layout;
  a.B = op.B; a.Ho = op.Ho; a.Wo = op.Wo;
  a.tiles_h = (op.Ho + TH - 1) / TH; a.tiles_w = (op.Wo + TW - 1) / TW;
  a.total_tiles = op.B * a.tiles_h * a.tiles_w;
  a.halo_tx_bytes = HW * HH * bk * 2;
  a.halo_stage_bytes = (a.halo_tx_bytes + 1023u) & ~1023u;
  a.halo_buf_bytes = a.slabs * P * a.halo_stage_bytes;
  a.w3_tile_bytes = HD_CHUNK * bk * 2;
  unsigned ws = P * a.w3_tile_bytes;
  if (2u * P * npad_max * 128u > ws) ws = 2u * P * npad_max * 128u;
  a.w_stage_bytes = (ws + 1023u) & ~1023u;
  const size_t budget = 220 * 1024;
  a.nh = 2 * (size_t)a.halo_buf_bytes + 3 * (size_t)a.w_stage_bytes <= budget ? 2 : 1;
  int nb = (int)((budget - a.nh * (size_t)a.halo_buf_bytes) / a.w_stage_bytes);
  if (nb > HD_MAX_NB) nb = HD_MAX_NB;
  if (nb < 2) return fail(CPB200_ERR_ARG, "heads: tile does not fit shared memory");
  a.nb = nb;
  t->smem = a.nh * (size_t)a.halo_buf_bytes + nb * (size_t)a.w_stage_bytes + 1024;
  const cuuint32_t box[4] = {(cuuint32_t)bk, HW, HH, 1}, estr[4] = {1, 1, 1, 1};
  if (int rc = encode_act_map(&a.amap, op.src[0], op.cin[0], op.cin[0], op.W, op.H, op.B, P, pr.fmt, sl.swizzle, box, estr, "heads"))
    return rc;
  // 3x3 weights: the heads' packed 3x3 convs back to back, [head][plane][tap][K-slab][hid][bk]
  if (int rc = encode_weight_map(&a.wmap3, op.weight, pr.fmt, bk, hid, HD_CHUNK, (long long)nheads * P * 9 * a.slabs, sl.swizzle,
                                 "heads (3x3)"))
    return rc;
  *out = t.release();
  return CPB200_OK;
}

// the output pointers and biases are read from the live table: outputs may be re-bound between runs
int heads_run(const Prepared &p, const cpb200_op &op, cudaStream_t st) {
  const HdOp &t = static_cast<const HdOp &>(p);
  const cpb200_head *hd = static_cast<const cpb200_head *>(op.aux);
  HdArgs args = t.args;
  args.bias3 = op.bias;
  for (int h = 0; h < args.nheads; ++h) {
    if (!hd[h].dst) return fail(CPB200_ERR_ARG, "heads: entry %d: null dst", h);
    args.dst[h] = hd[h].dst; args.bias1[h] = hd[h].bias;
  }
  return t.P == 2 ? launch<heads_tc_kernel<2>>("heads_tc_kernel", args.total_tiles, HD_THREADS, t.smem, st, args)
                  : launch<heads_tc_kernel<1>>("heads_tc_kernel", args.total_tiles, HD_THREADS, t.smem, st, args);
}

}  // namespace cpb

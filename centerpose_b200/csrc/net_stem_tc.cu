// Tensor-core stem: 7x7 (stride 1 or 2, pad 3) convolution of the NCHW fp32 network input with Cin = 3,
// + folded BatchNorm bias + activation, NHWC bf16 output          (pose_dla_dcn.py:246-250 base_layer,
// msra_resnet.py:112-116 conv1/bn1/relu).
//
// Why: on CUDA cores the 7x7x3 -> 16 stem costs 37 632 FMAs per output pixel (1.07 ms for 32 x 512^2,
// 13 % of the DLA-34 step at half the fp32 FMA peak).  Here the im2col happens IN SHARED MEMORY: producer
// threads build the K-major bf16 operand tile straight from a staged input patch, one wgmma chain
// per 64-pixel half tile does the arithmetic, and HBM only sees the image once and the output once.  (A first
// attempt that materialised a 32-channel im2col tensor in HBM was slower than the CUDA-core kernel.)
//
//   K index  k = (c * 7 + r) * 8 + s   (s = 0..7; the 8th column has a zero weight), 168 real + 24 zero = 192
//            => every 16-byte chunk of an operand row is 8 CONSECUTIVE input pixels of one (channel, row).
//   A tile   128 pixels (8 rows x 16 cols) x 192, three 64-wide slabs in the 128-byte-swizzled wgmma layout
//            (chunk j of row m at (j ^ (m & 7)) * 16), written with st.shared.v4 + fence.proxy.async.
//   B tile   weights, pre-swizzled by the host (plan.py::_pack_stem_tc), copied to shared memory once per CTA.
//   warps    0-7 two consumer warpgroups (rows 0-63 / 64-127: wgmma + epilogue), 8-15 producers (two groups of 128,
//            alternating tiles; thread m of a group builds row m).
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int PGROUPS = 2;                     // producer groups of 128 threads, alternating tiles
constexpr int CONS = 256;                      // two consumer warpgroups
constexpr int ST_THREADS = CONS + 128 * PGROUPS;
constexpr int TH = 8, TW = 16;                 // output tile (M = 128)
constexpr int KW8 = 8, KH = 7, CIN = 3;
constexpr int NCHUNK = CIN * KH;               // 21 real 16-byte chunks per operand row
constexpr int SLABS = 3;                       // K = 192
constexpr int A_SLAB_BYTES = 128 * 128;        // 128 rows x 128 B
constexpr int A_STAGE_BYTES = SLABS * A_SLAB_BYTES;
constexpr int NSTAGE = 3;

struct StemArgs {
  const float *x;            // (B,3,H,W) fp32
  __nv_bfloat16 *y;          // (B,Ho,Wo,N) bf16   [split mode: hi plane, lo plane y_plane elements later]
  const uint4 *wimg;         // pre-swizzled B operand image: SLABS x (N x 128 B)
  const float *bias;
  int B, H, W, Ho, Wo;
  int tiles_h, tiles_w, total_tiles;
  uint32_t act;
  uint32_t fmt;              // split mode (stem_tc_h_kernel<N, 2>): 0 = bf16 planes, 1 = fp16 planes
  float acc_scale;
  long long y_plane;
};

template <int N, int S>
__global__ void __launch_bounds__(ST_THREADS, 1) stem_tc_kernel(const StemArgs a) {
  constexpr int PH = (TH - 1) * S + KH;                   // staged input rows per tile
  constexpr int PW = (TW - 1) * S + KW8;                  // staged input columns per tile
  constexpr int PP = (S == 1) ? 48 : PW + 1;              // row pitch (words): S=1 keeps the two half-warps on disjoint banks
  constexpr int B_SLAB_BYTES = N * 128;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = smem_base + NSTAGE * A_STAGE_BYTES;
  float *patch0 = reinterpret_cast<float *>(smem_raw + (smem_base - smem_u32(smem_raw)) + NSTAGE * A_STAGE_BYTES + SLABS * B_SLAB_BYTES);
  __shared__ __align__(8) uint64_t bars[2 * NSTAGE];
  __shared__ float s_bias[N];
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[NSTAGE]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- one-time setup: barriers, zeroed A stages (the 3 pad chunks stay zero), weights, bias ----
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSTAGE; ++s) { mbar_init(full0 + 8 * s, 128); mbar_init(empty0 + 8 * s, CONS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < NSTAGE * A_STAGE_BYTES / 16; i += ST_THREADS)
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(a_base + i * 16), "r"(0u) : "memory");
  for (int i = threadIdx.x; i < SLABS * B_SLAB_BYTES / 16; i += ST_THREADS) {
    const uint4 v = __ldg(a.wimg + i);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(b_base + i * 16), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  for (int i = threadIdx.x; i < N; i += ST_THREADS) s_bias[i] = a.bias ? __ldg(a.bias + i) : 0.f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  auto decode_tile = [&](int t, int &n, int &h0, int &w0) {
    const int tw = t % a.tiles_w; t /= a.tiles_w;
    const int th = t % a.tiles_h; n = t / a.tiles_h;
    h0 = th * TH; w0 = tw * TW;
  };

  if (warp >= CONS / 32) {
    // =============================== producers: patch -> swizzled K-major operand rows ===============================
    // One warp per scheduler is latency-bound on the LDS -> cvt -> STS chains, so PGROUPS groups work on alternate tiles;
    // stages are handed to the consumers in tile order.
    const int grp = (warp - CONS / 32) >> 2;
    const int m = threadIdx.x & 127;                       // operand row = tile pixel (ty, tx)
    const int ty = m >> 4, tx = m & 15;
    float *patch = patch0 + grp * (2 * CIN * PH * PP);
    const int tstep = gridDim.x * PGROUPS;
    int it = grp;                                          // index of this group's tile in the CTA's tile sequence
    int pb = 0;                                            // patch double buffer
    constexpr int NLD = (CIN * PH * PW + 127) / 128;       // patch elements per producer thread
    float pre[NLD];
    // The patch of tile i+1 is requested from global memory BEFORE tile i's operand rows are built and parked in
    // registers meanwhile: without this every tile pays a full exposed DRAM/L2 round trip.
    auto fetch = [&](int t) {
      int n, h0, w0; decode_tile(t, n, h0, w0);
      const int hi0 = h0 * S - 3, wi0 = w0 * S - 3;
      const float *xin = a.x + (size_t)n * CIN * a.H * a.W;
#pragma unroll
      for (int j = 0; j < NLD; ++j) {
        const int i = m + j * 128;
        const int col = i % PW, rr = i / PW;               // rr = c * PH + row
        const int row = rr % PH, c = rr / PH;
        const int hi = hi0 + row, wi = wi0 + col;
        const bool okl = i < CIN * PH * PW && hi >= 0 && hi < a.H && wi >= 0 && wi < a.W;
        pre[j] = okl ? __ldg(xin + ((size_t)c * a.H + hi) * a.W + wi) : 0.f;
      }
    };
    const int t_first = blockIdx.x + grp * gridDim.x;
    if (t_first < a.total_tiles) fetch(t_first);
    for (int t = t_first; t < a.total_tiles; t += tstep, it += PGROUPS) {
      const int stage = it % NSTAGE;
      const uint32_t phase = (uint32_t)(it / NSTAGE) & 1u;
      float *pbuf = patch + pb * (CIN * PH * PP);
#pragma unroll
      for (int j = 0; j < NLD; ++j) {
        const int i = m + j * 128;
        if (i < CIN * PH * PW) pbuf[(i / PW) * PP + (i % PW)] = pre[j];
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + grp) : "memory");   // patch complete (the other buffer is free: see below)
      if (t + tstep < a.total_tiles) fetch(t + tstep);
      mbar_wait(empty0 + 8 * stage, phase ^ 1);
      const uint32_t sa = a_base + stage * A_STAGE_BYTES + m * 128;
      const float *prow = pbuf + (ty * S) * PP + tx * S;
#pragma unroll
      for (int q = 0; q < NCHUNK; ++q) {
        const int c = q / KH, r = q % KH;
        const float *p = prow + (c * PH + r) * PP;
        __nv_bfloat162 h0 = __floats2bfloat162_rn(p[0], p[1]), h1 = __floats2bfloat162_rn(p[2], p[3]);
        __nv_bfloat162 h2 = __floats2bfloat162_rn(p[4], p[5]), h3 = __floats2bfloat162_rn(p[6], p[7]);
        const uint32_t dst = sa + (q >> 3) * A_SLAB_BYTES + (((q & 7) ^ (m & 7)) << 4);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(*reinterpret_cast<uint32_t *>(&h0)),
                     "r"(*reinterpret_cast<uint32_t *>(&h1)), "r"(*reinterpret_cast<uint32_t *>(&h2)),
                     "r"(*reinterpret_cast<uint32_t *>(&h3)) : "memory");
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_arrive(full0 + 8 * stage);
      // the next tile fills the OTHER patch buffer; by the time a thread returns to this one it has passed the
      // next tile's bar.sync, i.e. every producer has finished reading this buffer.
      pb ^= 1;
    }
  } else {
    // =============================== consumers: wgmma + epilogue ===============================
    const int wg = warp >> 2, tq = threadIdx.x & 127;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
      mbar_wait(full0 + 8 * stage, phase);
      const uint64_t ad0 = make_desc(a_base + stage * A_STAGE_BYTES + wg * 64 * 128, 128, 1);
      const uint64_t bd0 = make_desc(b_base, 128, 1);
      wg_fence();
#pragma unroll
      for (int sl = 0; sl < SLABS; ++sl) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_k16<N>(acc, ad0 + (uint32_t)(sl * (A_SLAB_BYTES >> 4) + 2 * k), bd0 + (uint32_t)(sl * (B_SLAB_BYTES >> 4) + 2 * k),
                       (sl > 0 || k > 0) ? 1u : 0u, 1u);
      }
      wg_commit();
      wg_wait<0>();
      acc_fence(acc);
      if (lane == 0) mbar_arrive(empty0 + 8 * stage);
      if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
      int n, h0, w0; decode_tile(t, n, h0, w0);
#pragma unroll
      for (int j = 0; j < N / 4; ++j) {
        const int m = wg * 64 + frag_row(tq, j), c = frag_col(tq, j);
        const int ho = h0 + (m >> 4), wo = w0 + (m & 15);
        if (ho >= a.Ho || wo >= a.Wo) continue;
        epilogue_pair<1>(acc, acc, j, s_bias[c], s_bias[c + 1], 1.f, a.act, OUT_16, a.y, nullptr, (((size_t)n * a.Ho + ho) * a.Wo + wo) * N + c,
                         0, true, 0u);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Stride-1 variant (DLA-34 base_layer): fold only the VERTICAL taps into the K dimension and let the wgmma
// descriptors do the horizontal ones.  Per tile (16 rows x 8 cols) the producers build, for every output row ty
// and every input column x of the 14-wide halo, ONE 64-byte vector T[ty][x][k = c*7 + r] = in[c][ty + r][x]
// (21 real values of 32) — 224 vectors instead of 128 x 21 chunks, ~8x less shared-memory traffic and cvt work.
// Horizontal tap s is then the operand window starting s vectors later: descriptor start + s * 64 B, stride
// between 8-row groups = 14 * 64 B (same shifted-window trick as csrc/net_tc3.cu; 64-byte swizzle on absolute
// address bits).  7 taps x K=32 = 14 wgmma per warpgroup and tile.
constexpr int HT_H = 16, HT_W = 8;                       // output tile, M = 128, m = ty * 8 + tx
constexpr int HP_W = HT_W + 6, HP_H = HT_H + 6;          // input patch 22 x 14 per channel
constexpr int HVEC = HT_H * HP_W;                        // 224 operand vectors per tile = producer threads
constexpr int HA_STAGE_BYTES = ((HVEC * 64 + 1023) / 1024) * 1024;
constexpr int H_GROUPS = 1;                              // producer groups (7 warps each) on alternate tiles: the consumers' 64
                                                         // accumulator registers leave room for one beside them
constexpr int H_THREADS = CONS + H_GROUPS * HVEC;        // consumers + producers
template <int N_, int P_> struct HStages { static constexpr int value = (P_ == 2 && N_ > 16) ? 4 : 6; };

// P = 2 (split operands, CPB200_BF16X2 / CPB200_F16X2): every producer thread splits its 21 fp32 input values into a hi and a
// lo 64-byte vector; a stage is [hi vectors | lo vectors], the weight image per horizontal tap [hi tile | lo tile]
// (plan.py::_pack_stem_tc_h).
template <int N, int P>
__global__ void __launch_bounds__(H_THREADS, 1) stem_tc_h_kernel(const StemArgs a) {
  constexpr int H_NSTAGE = HStages<N, P>::value;
  constexpr int HA_PLANE_BYTES = HA_STAGE_BYTES;           // one plane of a stage
  constexpr int HA_STAGE = P * HA_PLANE_BYTES;
  constexpr int B_TILE_BYTES = N * 64;
  constexpr int B_TAP_BYTES = P * B_TILE_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_base = smem_base;
  const uint32_t b_base = smem_base + H_NSTAGE * HA_STAGE;
  __shared__ __align__(8) uint64_t bars[2 * H_NSTAGE];
  __shared__ float s_bias[N];
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[H_NSTAGE]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < H_NSTAGE; ++s) { mbar_init(full0 + 8 * s, HVEC); mbar_init(empty0 + 8 * s, CONS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < H_NSTAGE * HA_STAGE / 16; i += H_THREADS)      // pad values (k >= 21) stay zero
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(a_base + i * 16), "r"(0u) : "memory");
  for (int i = threadIdx.x; i < 7 * B_TAP_BYTES / 16; i += H_THREADS) {
    const uint4 v = __ldg(a.wimg + i);
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(b_base + i * 16), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
  for (int i = threadIdx.x; i < N; i += H_THREADS) s_bias[i] = a.bias ? __ldg(a.bias + i) : 0.f;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  auto decode_tile = [&](int t, int &n, int &h0, int &w0) {
    const int tw = t % a.tiles_w; t /= a.tiles_w;
    const int th = t % a.tiles_h; n = t / a.tiles_h;
    h0 = th * HT_H; w0 = tw * HT_W;
  };

  if (warp >= CONS / 32) {
    // =============================== producers: thread v = (ty, x) builds one 64-byte vector ===============================
    // The 21 values come straight from global memory (read-only path; the 7 threads that share an input element
    // hit L1) and the NEXT tile's values are requested before this tile's vector is converted and stored, so a
    // producer thread never waits on anything but the stage's empty barrier: no CTA-level barrier, no staging
    // buffer.  What bounds a producer is the global-load round trip of its NEXT tile (~1 us under load: three
    // with one tile in flight), so H_GROUPS independent
    // groups take alternate tiles and hand their stages to the consumers in tile order.
    const int grp = (threadIdx.x - CONS) / HVEC;
    const int v = (threadIdx.x - CONS) - grp * HVEC;
    const int tstep = gridDim.x * H_GROUPS;
    const int ty = v / HP_W, x = v % HP_W;
    float f[24];
#pragma unroll
    for (int q = 0; q < 24; ++q) f[q] = 0.f;
    const size_t plane = (size_t)a.H * a.W;
    auto fetch = [&](int t) {
      int n, h0, w0; decode_tile(t, n, h0, w0);
      const int wi = w0 - 3 + x, hi0 = h0 - 3 + ty;
      const float *p0 = a.x + (size_t)n * CIN * plane + (ptrdiff_t)hi0 * a.W + wi;
      if (h0 >= 3 && h0 + HT_H + 3 <= a.H && w0 >= 3 && w0 + HT_W + 3 <= a.W) {
        // interior tile (warp-uniform): no bounds checks, pointer increments only
#pragma unroll
        for (int r = 0; r < KH; ++r) {
          const float *p = p0 + (size_t)r * a.W;
#pragma unroll
          for (int c = 0; c < CIN; ++c) f[c * KH + r] = __ldg(p + c * plane);
        }
      } else {
        const bool okw = wi >= 0 && wi < a.W;
#pragma unroll
        for (int r = 0; r < KH; ++r) {
          const int hi = hi0 + r;
          const bool okl = okw && hi >= 0 && hi < a.H;
#pragma unroll
          for (int c = 0; c < CIN; ++c) f[c * KH + r] = okl ? __ldg(p0 + (ptrdiff_t)r * a.W + c * plane) : 0.f;
        }
      }
    };
    // physical address of (vector row R = v, chunk j): 64-byte swizzle XORs address bits [4,5] with bits [7,8];
    // stage bases are 1024-aligned, so bits [7,8] of the address are (R >> 1) & 3.
    const uint32_t vrow = (uint32_t)v * 64u, sw = ((uint32_t)v >> 1) & 3u;
    const int t_first = blockIdx.x + grp * gridDim.x;
    int it = grp;                                          // index of this group's tile in the CTA's tile sequence
    if (t_first < a.total_tiles) fetch(t_first);
    for (int t = t_first; t < a.total_tiles; t += tstep, it += H_GROUPS) {
      const int stage = it % H_NSTAGE;
      const uint32_t phase = (uint32_t)(it / H_NSTAGE) & 1u;
      uint32_t pk[12], pl_[P == 2 ? 12 : 1];
#pragma unroll
      for (int q = 0; q < 12; ++q) {
        if constexpr (P == 2) {
          split2(f[2 * q], f[2 * q + 1], a.fmt, pk[q], pl_[q]);
        } else {
          __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
          pk[q] = *reinterpret_cast<uint32_t *>(&h);
        }
      }
      if (t + tstep < a.total_tiles) fetch(t + tstep);                   // in flight while we wait for the stage
      mbar_wait(empty0 + 8 * stage, phase ^ 1);
      const uint32_t sa = a_base + stage * HA_STAGE + vrow;
#pragma unroll
      for (int j = 0; j < 3; ++j)
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sa + ((j ^ sw) << 4)), "r"(pk[4 * j]), "r"(pk[4 * j + 1]),
                     "r"(pk[4 * j + 2]), "r"(pk[4 * j + 3]) : "memory");
      if constexpr (P == 2) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sa + HA_PLANE_BYTES + ((j ^ sw) << 4)), "r"(pl_[4 * j]),
                       "r"(pl_[4 * j + 1]), "r"(pl_[4 * j + 2]), "r"(pl_[4 * j + 3]) : "memory");
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_arrive(full0 + 8 * stage);
    }
  } else {
    // =============================== consumers: wgmma + epilogue ===============================
    const int wg = warp >> 2, tq = threadIdx.x & 127;
    const uint32_t bf = (P == 1 || a.fmt == 0) ? 1u : 0u;
    float acc[N / 2], acc2[P == 2 ? N / 2 : 1];
    acc_zero(acc, acc2);
    int stage = 0; uint32_t phase = 0;
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
      mbar_wait(full0 + 8 * stage, phase);
      // this warpgroup's 64 rows = output rows 8 wg .. 8 wg + 7 = 8 halo rows of vectors further on
      const uint64_t ad0 = desc_sbo(a_base + stage * HA_STAGE + wg * 8 * HP_W * 64, HP_W * 64, 2);
      const uint64_t bd0 = desc_sbo(b_base, 8 * 64, 2);
      wg_fence();
#pragma unroll
      for (int s = 0; s < 7; ++s) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint64_t ad = ad0 + (uint32_t)(s * 4), bd = bd0 + (uint32_t)(s * (B_TAP_BYTES >> 4));
          mma_step<N, P>(acc, acc2, ad, ad + (uint32_t)(HA_PLANE_BYTES >> 4), bd, bd + (uint32_t)(B_TILE_BYTES >> 4), k,
                         (s > 0 || k > 0) ? 1u : 0u, bf);
        }
      }
      wg_commit();
      wg_wait<0>();
      acc_fence(acc); acc_fence(acc2);
      if (lane == 0) mbar_arrive(empty0 + 8 * stage);
      if (++stage == H_NSTAGE) { stage = 0; phase ^= 1; }
      int n, h0, w0; decode_tile(t, n, h0, w0);
#pragma unroll
      for (int j = 0; j < N / 4; ++j) {
        const int m = wg * 64 + frag_row(tq, j), c = frag_col(tq, j);
        const int ho = h0 + (m >> 3), wo = w0 + (m & 7);
        if (ho >= a.Ho || wo >= a.Wo) continue;
        epilogue_pair<P>(acc, acc2, j, s_bias[c], s_bias[c + 1], a.acc_scale, a.act, OUT_16, a.y, nullptr,
                         (((size_t)n * a.Ho + ho) * a.Wo + wo) * N + c, a.y_plane, true, a.fmt);
      }
    }
  }
}

template <int N, int P>
int launch_stem_h(const cpb200_op &op, cudaStream_t st) {
  StemArgs a;
  const Prec pr = prec_of(op);
  a.fmt = pr.fmt; a.acc_scale = pr.acc_scale;
  a.y_plane = (long long)op.B * op.Ho * op.Wo * N;
  a.x = static_cast<const float *>(op.src[0]); a.y = static_cast<__nv_bfloat16 *>(op.dst);
  a.wimg = static_cast<const uint4 *>(op.weight); a.bias = op.bias;
  a.B = op.B; a.H = op.H; a.W = op.W; a.Ho = op.Ho; a.Wo = op.Wo;
  a.tiles_h = (op.Ho + HT_H - 1) / HT_H; a.tiles_w = (op.Wo + HT_W - 1) / HT_W;
  a.total_tiles = op.B * a.tiles_h * a.tiles_w;
  a.act = op.flags & CPB_ACT_MASK;
  const size_t smem = 1024 + (size_t)HStages<N, P>::value * P * HA_STAGE_BYTES + 7 * (size_t)P * N * 64;
  return launch<stem_tc_h_kernel<N, P>>("stem_tc_h_kernel", a.total_tiles, H_THREADS, smem, st, a);
}

template <int N, int S>
int launch_stem(const cpb200_op &op, cudaStream_t st) {
  constexpr int PH = (TH - 1) * S + KH, PW = (TW - 1) * S + KW8, PP = (S == 1) ? 48 : PW + 1;
  StemArgs a;
  a.x = static_cast<const float *>(op.src[0]); a.y = static_cast<__nv_bfloat16 *>(op.dst);
  a.wimg = static_cast<const uint4 *>(op.weight); a.bias = op.bias;
  a.B = op.B; a.H = op.H; a.W = op.W; a.Ho = op.Ho; a.Wo = op.Wo;
  a.tiles_h = (op.Ho + TH - 1) / TH; a.tiles_w = (op.Wo + TW - 1) / TW;
  a.total_tiles = op.B * a.tiles_h * a.tiles_w;
  a.act = op.flags & CPB_ACT_MASK;
  a.fmt = 0; a.acc_scale = 1.f; a.y_plane = 0;
  const size_t smem = 1024 + (size_t)NSTAGE * A_STAGE_BYTES + (size_t)SLABS * N * 128 + (size_t)PGROUPS * 2 * CIN * PH * PP * sizeof(float);
  return launch<stem_tc_kernel<N, S>>("stem_tc_kernel", a.total_tiles, ST_THREADS, smem, st, a);
}

}  // namespace

namespace cpb {

bool stem_tc_eligible(const cpb200_op &op) {
  const bool split = op.act_dtype == CPB200_BF16X2 || op.act_dtype == CPB200_F16X2;
  // split operands: the stride-1 kernel only (the stride-2 im2col stages do not fit twice; plan.py routes those through fp32)
  return op.type == CPB200_OP_STEM && (op.act_dtype == CPB200_BF16 || (split && op.stride == 1)) && op.cin[0] == 3 && op.kh == 7 && op.kw == 7 &&
         op.pad_h == 3 && op.pad_w == 3 && (op.stride == 1 || op.stride == 2) && (op.cout == 16 || op.cout == 64) &&
         op.Ho == (op.H + 6 - 7) / op.stride + 1 && op.Wo == (op.W + 6 - 7) / op.stride + 1;
}

int stem_tc_run(const cpb200_op &op, cudaStream_t st) {
  const bool split = op.act_dtype != CPB200_BF16;
  // stride 1: vertical-fold kernel (weight image = 7 taps x N rows x 64 B); stride 2: full im2col rows (3 slabs x N x 128 B)
  if (op.cout == 16 && op.stride == 1) return split ? launch_stem_h<16, 2>(op, st) : launch_stem_h<16, 1>(op, st);
  if (op.cout == 64 && op.stride == 1) return split ? launch_stem_h<64, 2>(op, st) : launch_stem_h<64, 1>(op, st);
  if (op.cout == 16) return launch_stem<16, 2>(op, st);
  return launch_stem<64, 2>(op, st);
}

}  // namespace cpb

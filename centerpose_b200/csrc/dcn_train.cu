// Modulated deformable convolution (DCNv2) for training: forward, data backward and weight backward, as the reference's
// `_ext.dcn_v2_forward` / `_ext.dcn_v2_backward` compute them (DCNv2/src/cuda/dcn_v2_cuda.cu, dcn_v2_im2col_cuda.cu),
// for the one configuration every reference backbone builds: 3x3 taps, stride 1, padding 1, dilation 1, one
// deformable group.  Tensors are the reference's: NCHW fp32 input / output, offset (B, 18, H, W) with channel 2*tap = dh
// and 2*tap+1 = dw, mask (B, 9, H, W) already a probability, weight (Co, C, 3, 3).
//
// All three passes are one tiled GEMM whose column operand is gathered on the fly, so the (C*9) x (H*W) column matrix
// never reaches HBM.  The GEMM row index of the column matrix is r = c*9 + tap, the weight's own (Co, C*9) layout.
//   forward          out[o, p]   = sum_r W[o, r] col[r, p] + bias[o]        tile Co x pixels, K = C*9
//   data backward    gcol[r, p]  = sum_o W[o, r] gout[o, p]                 tile (c, tap) x pixels, K = Co
//                    then col2im / col2im_coord on the tile, from shared memory
//   weight backward  gW[o, r]    = sum_p gout[o, p] col[r, p]               tile Co x (c, tap), K = B*H*W, split K
//
// Two inner products share every kernel, tile and accumulator layout: train_mma.cuh's 3xTF32 tensor-core split
// (TRAIN_TF32X3) and CUDA-core fp32 (TRAIN_FP32).
//
// Determinism: the forward, grad_offset, grad_mask, grad_weight and grad_bias are sums in a fixed order (no atomics);
// grad_input is scattered with fp32 atomics, as the reference and torchvision do.
#include "common.cuh"
#include "train_mma.cuh"

namespace cpb {
namespace {

using namespace train;
constexpr int TAPS = 9;
constexpr int WG_TARGET_CTAS = 264;     // weight-backward split-K aims at two CTAs per SM of a 132-SM H100
constexpr size_t WG_WS_CAP = size_t(16) << 20;  // and keeps its per-split partials under 16 MiB

// One bilinear sample of tap `tap` at output pixel (ho, wo): dmcn_im2col_bilinear's corners and weights
// (dcn_v2_im2col_cuda.cu:25-54) behind the `> -1 / < H` test of :180.  bits 0..3 = corners v1..v4 in bounds; all clear
// outside the sampling range.
struct Sample {
  int base;            // h_low * W + w_low
  int bits;
  float lh, lw, m;
};

__device__ __forceinline__ Sample make_sample(const float *off, const float *msk, int b, int tap, int p, int H, int W) {
  const int HW = H * W;
  const int ho = p / W, wo = p - ho * W;
  const size_t ob = (size_t)b * 2 * TAPS * HW;
  const float oh = off[ob + (size_t)(2 * tap) * HW + p];
  const float ow = off[ob + (size_t)(2 * tap + 1) * HW + p];
  Sample s;
  s.m = msk[((size_t)b * TAPS + tap) * HW + p];
  const float h = (float)(ho - 1 + tap / 3) + oh;
  const float w = (float)(wo - 1 + tap % 3) + ow;
  s.bits = 0;
  s.base = 0;
  s.lh = s.lw = 0.f;
  if (h > -1.f && w > -1.f && h < (float)H && w < (float)W) {
    const int hl = (int)floorf(h), wl = (int)floorf(w);
    s.lh = h - (float)hl;
    s.lw = w - (float)wl;
    s.base = hl * W + wl;
    s.bits = (hl >= 0 && wl >= 0 ? 1 : 0) | (hl >= 0 && wl + 1 <= W - 1 ? 2 : 0) |
             (hl + 1 <= H - 1 && wl >= 0 ? 4 : 0) | (hl + 1 <= H - 1 && wl + 1 <= W - 1 ? 8 : 0) | 16;
  }
  return s;
}

struct Corners { float v1, v2, v3, v4; };

__device__ __forceinline__ Corners load_corners(const float *plane, const Sample &s, int W) {
  Corners v;
  v.v1 = (s.bits & 1) ? __ldg(plane + s.base) : 0.f;
  v.v2 = (s.bits & 2) ? __ldg(plane + s.base + 1) : 0.f;
  v.v3 = (s.bits & 4) ? __ldg(plane + s.base + W) : 0.f;
  v.v4 = (s.bits & 8) ? __ldg(plane + s.base + W + 1) : 0.f;
  return v;
}

__device__ __forceinline__ float bilinear(const Corners &v, float lh, float lw) {
  const float hh = 1.f - lh, hw = 1.f - lw;
  const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
  return w1 * v.v1 + w2 * v.v2 + w3 * v.v3 + w4 * v.v4;
}

// ---- forward: out[b] = W (Co x C*9) . col[b] (C*9 x HW) + bias ------------------------------------------------------
// grid (pixel tiles of BN, Co tiles of BM, B).  The tile's 9 x BN samples are set up once; each K step gathers a
// BK x BN column slab from them.
template <int P>
__global__ void __launch_bounds__(NT) dcn_fwd_kernel(const float *__restrict__ x, const float *__restrict__ wgt,
                                                     const float *__restrict__ bias, const float *__restrict__ off,
                                                     const float *__restrict__ msk, float *__restrict__ out, int C,
                                                     int H, int W, int Co) {
  __shared__ float As[BM][AP];
  __shared__ __align__(16) float Bs[BK][BP];
  __shared__ Sample S[TAPS][BN];
  const int HW = H * W, K = C * TAPS;
  const int p0 = blockIdx.x * BN, o0 = blockIdx.y * BM, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  for (int e = tid; e < TAPS * BN; e += NT) {
    const int tap = e / BN, n = e % BN;
    if (p0 + n < HW) S[tap][n] = make_sample(off, msk, b, tap, p0 + n, H, W);
  }
  float acc[2][4][4];
  zero_acc(acc);
  const float *xb = x + (size_t)b * C * HW;
  for (int r0 = 0; r0 < K; r0 += BK) {
    __syncthreads();
    for (int e = tid; e < BM * BK; e += NT) {
      const int m = e / BK, k = e % BK;
      As[m][k] = (o0 + m < Co && r0 + k < K) ? __ldg(wgt + (size_t)(o0 + m) * K + r0 + k) : 0.f;
    }
    for (int e = tid; e < BK * BN; e += NT) {
      const int k = e / BN, n = e % BN, r = r0 + k;
      float v = 0.f;
      if (r < K && p0 + n < HW) {
        const int c = r / TAPS, tap = r - c * TAPS;
        const Sample s = S[tap][n];
        if (s.bits) v = bilinear(load_corners(xb + (size_t)c * HW, s, W), s.lh, s.lw) * s.m;
      }
      Bs[k][n] = v;
    }
    __syncthreads();
    tile_mma<P>(As, Bs, wm, wn, lane, acc);
  }
  const int gid = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int o = o0 + wm * 32 + mt * 16 + gid + 8 * h;
      if (o >= Co) continue;
      const float bo = bias[o];
      float *orow = out + ((size_t)b * Co + o) * HW;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int p = p0 + wn * 32 + nt * 8 + 2 * tig + j;
          if (p < HW) orow[p] = acc[mt][nt][2 * h + j] + bo;
        }
    }
}

// ---- data backward: gcol = W^T . gout per pixel tile, consumed from shared memory ----------------------------------
// grid (pixel tiles of BN, B).  The CTA walks the C*9 rows in chunks of BM; each chunk's gcol (BM x BN) is staged in
// shared memory and consumed by thread (half, n): pixel n, rows [half*32, half*32 + 32) of the chunk, in order.
//   grad_input  += weight_corner * (gcol * mask)   at the four corners            (col2im, :197-254)
//   grad_offset  = sum_c coordinate_weight * gcol * mask                          (col2im_coord, :256-327)
//   grad_mask    = sum_c gcol * bilinear
// The offset / mask sums of (half, tap, n) live in shared memory, owned by one thread, and the two halves are added
// once at the end: a fixed order.
struct DataSmem {
  union {
    struct {
      float As[BM][AP];
      float Bs[BK][BP];
    } g;
    float G[BM][BN + 4];
  } u;
  Sample S[TAPS][BN];
  float acc[2][3][TAPS][BN];   // [half][dh, dw, mask][tap][n]
};

template <int P>
__global__ void __launch_bounds__(NT) dcn_bwd_data_kernel(const float *__restrict__ x, const float *__restrict__ wgt,
                                                          const float *__restrict__ off, const float *__restrict__ msk,
                                                          const float *__restrict__ gout, float *__restrict__ gin,
                                                          float *__restrict__ goff, float *__restrict__ gmsk, int C,
                                                          int H, int W, int Co) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  DataSmem &sm = *reinterpret_cast<DataSmem *>(smem_raw);
  const int HW = H * W, K = C * TAPS;
  const int p0 = blockIdx.x * BN, b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  const int gid = lane >> 2, tig = lane & 3;
  for (int e = tid; e < TAPS * BN; e += NT) {
    const int tap = e / BN, n = e % BN;
    if (p0 + n < HW) sm.S[tap][n] = make_sample(off, msk, b, tap, p0 + n, H, W);
  }
  for (int e = tid; e < 2 * 3 * TAPS * BN; e += NT) (&sm.acc[0][0][0][0])[e] = 0.f;
  const float *xb = x + (size_t)b * C * HW;
  const float *gb = gout + (size_t)b * Co * HW;
  float *gib = gin + (size_t)b * C * HW;
  const int en = tid % BN, half = tid / BN;
  for (int r0 = 0; r0 < K; r0 += BM) {
    float acc[2][4][4];
    zero_acc(acc);
    for (int k0 = 0; k0 < Co; k0 += BK) {
      __syncthreads();
      for (int e = tid; e < BM * BK; e += NT) {
        const int m = e % BM, k = e / BM;
        sm.u.g.As[m][k] = (r0 + m < K && k0 + k < Co) ? __ldg(wgt + (size_t)(k0 + k) * K + r0 + m) : 0.f;
      }
      for (int e = tid; e < BK * BN; e += NT) {
        const int k = e / BN, n = e % BN;
        sm.u.g.Bs[k][n] = (k0 + k < Co && p0 + n < HW) ? __ldg(gb + (size_t)(k0 + k) * HW + p0 + n) : 0.f;
      }
      __syncthreads();
      tile_mma<P>(sm.u.g.As, sm.u.g.Bs, wm, wn, lane, acc);
    }
    __syncthreads();
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int m = wm * 32 + mt * 16 + gid, n = wn * 32 + nt * 8 + 2 * tig;
        *reinterpret_cast<float2 *>(&sm.u.G[m][n]) = make_float2(acc[mt][nt][0], acc[mt][nt][1]);
        *reinterpret_cast<float2 *>(&sm.u.G[m + 8][n]) = make_float2(acc[mt][nt][2], acc[mt][nt][3]);
      }
    __syncthreads();
    if (p0 + en < HW) {
      for (int mm = 0; mm < BM / 2; ++mm) {
        const int m = half * (BM / 2) + mm, r = r0 + m;
        if (r >= K) break;
        const int c = r / TAPS, tap = r - c * TAPS;
        const Sample s = sm.S[tap][en];
        if (!s.bits) continue;     // outside (-1, H) x (-1, W): every weight of the reference is 0
        const float g = sm.u.G[m][en];
        const float *plane = xb + (size_t)c * HW;
        const Corners v = load_corners(plane, s, W);
        const float hh = 1.f - s.lh, hw = 1.f - s.lw;
        // col2im: cur_top_grad = gcol * mask, times each corner's bilinear weight
        const float tg = g * s.m;
        float *gp = gib + (size_t)c * HW + s.base;
        if (s.bits & 1) atomicAdd(gp, hh * hw * tg);
        if (s.bits & 2) atomicAdd(gp + 1, hh * s.lw * tg);
        if (s.bits & 4) atomicAdd(gp + W, s.lh * hw * tg);
        if (s.bits & 8) atomicAdd(gp + W + 1, s.lh * s.lw * tg);
        // dmcn_get_coordinate_weight, bp_dir 0 (h) and 1 (w)
        const float cw_h = -hw * v.v1 - s.lw * v.v2 + hw * v.v3 + s.lw * v.v4;
        const float cw_w = -hh * v.v1 + hh * v.v2 - s.lh * v.v3 + s.lh * v.v4;
        sm.acc[half][0][tap][en] += cw_h * g * s.m;
        sm.acc[half][1][tap][en] += cw_w * g * s.m;
        sm.acc[half][2][tap][en] += g * bilinear(v, s.lh, s.lw);
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < TAPS * BN; e += NT) {
    const int tap = e / BN, n = e % BN, p = p0 + n;
    if (p >= HW) continue;
    goff[((size_t)b * 2 * TAPS + 2 * tap) * HW + p] = sm.acc[0][0][tap][n] + sm.acc[1][0][tap][n];
    goff[((size_t)b * 2 * TAPS + 2 * tap + 1) * HW + p] = sm.acc[0][1][tap][n] + sm.acc[1][1][tap][n];
    gmsk[((size_t)b * TAPS + tap) * HW + p] = sm.acc[0][2][tap][n] + sm.acc[1][2][tap][n];
  }
}

// ---- weight backward: partial[s] = gout (Co x pixels of split s) . col^T (pixels x C*9) -----------------------------
// grid (C*9 tiles of BN, Co tiles of BM, splits).  K runs over the flattened (b, p) pixels of the split, BK at a time;
// each step sets up the BK x 9 samples of its pixels and gathers the BK x BN column slab (pixels x (c, tap)).
template <int P>
__global__ void __launch_bounds__(NT) dcn_bwd_weight_kernel(const float *__restrict__ x, const float *__restrict__ off,
                                                            const float *__restrict__ msk,
                                                            const float *__restrict__ gout, float *__restrict__ part,
                                                            int B, int C, int H, int W, int Co, int steps_per_split) {
  __shared__ float As[BM][AP];
  __shared__ __align__(16) float Bs[BK][BP];
  __shared__ Sample S[TAPS][BK];
  const int HW = H * W, K = C * TAPS, NQ = B * HW;
  const int r0 = blockIdx.x * BN, o0 = blockIdx.y * BM, split = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  float acc[2][4][4];
  zero_acc(acc);
  const int q_begin = split * steps_per_split * BK;
  const int q_end = min(NQ, q_begin + steps_per_split * BK);
  for (int q0 = q_begin; q0 < q_end; q0 += BK) {
    __syncthreads();
    if (tid < TAPS * BK) {
      const int tap = tid / BK, k = tid % BK, q = q0 + k;
      if (q < q_end) {
        const int bq = q / HW;
        S[tap][k] = make_sample(off, msk, bq, tap, q - bq * HW, H, W);
      }
    }
    for (int e = tid; e < BM * BK; e += NT) {
      const int m = e / BK, k = e % BK, q = q0 + k;
      float v = 0.f;
      if (o0 + m < Co && q < q_end) {
        const int bq = q / HW;
        v = __ldg(gout + ((size_t)bq * Co + o0 + m) * HW + (q - bq * HW));
      }
      As[m][k] = v;
    }
    __syncthreads();
    for (int e = tid; e < BK * BN; e += NT) {
      const int k = e % BK, n = e / BK, r = r0 + n, q = q0 + k;
      float v = 0.f;
      if (r < K && q < q_end) {
        const int c = r / TAPS, tap = r - c * TAPS, bq = q / HW;
        const Sample s = S[tap][k];
        if (s.bits) v = bilinear(load_corners(x + ((size_t)bq * C + c) * HW, s, W), s.lh, s.lw) * s.m;
      }
      Bs[k][n] = v;
    }
    __syncthreads();
    tile_mma<P>(As, Bs, wm, wn, lane, acc);
  }
  const int gid = lane >> 2, tig = lane & 3;
  float *ps = part + (size_t)split * Co * K;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int o = o0 + wm * 32 + mt * 16 + gid + 8 * h;
      if (o >= Co) continue;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int r = r0 + wn * 32 + nt * 8 + 2 * tig + j;
          if (r < K) ps[(size_t)o * K + r] = acc[mt][nt][2 * h + j];
        }
    }
}

// grad_weight = sum of the split partials, in split order
__global__ void dcn_wgrad_reduce_kernel(const float *__restrict__ part, float *__restrict__ gw, int n, int splits) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float s = part[i];
    for (int k = 1; k < splits; ++k) s += part[(size_t)k * n + i];
    gw[i] = s;
  }
}

// grad_bias[o] = sum over (b, p) of gout[b, o, p]: thread-strided partial sums, then a fixed shared-memory tree.
// Each thread adds B*HW/256 values in sequence (4 096 at B = 64 on 128x128); a plain running sum drifts by some 1e-6
// relative there, so the partial sums are compensated (Kahan): each carries its rounding error into the next add.
__global__ void __launch_bounds__(NT) dcn_bgrad_kernel(const float *__restrict__ gout, float *__restrict__ gbias, int B,
                                                       int Co, int HW) {
  __shared__ float red[NT];
  const int o = blockIdx.x;
  float s = 0.f, c = 0.f;
  for (int b = 0; b < B; ++b) {
    const float *row = gout + ((size_t)b * Co + o) * HW;
    for (int p = threadIdx.x; p < HW; p += NT) {
      const float y = __fsub_rn(row[p], c);
      const float t = __fadd_rn(s, y);
      c = __fsub_rn(__fsub_rn(t, s), y);
      s = t;
    }
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = NT / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) gbias[o] = red[0];
}

struct WgradSplit { int splits, steps; };

WgradSplit wgrad_split(int B, int C, int H, int W, int Co) {
  const long long K = (long long)C * TAPS;
  const long long tiles = (long long)ceil_div((int)K, BN) * ceil_div(Co, BM);
  const long long nsteps = ((long long)B * H * W + BK - 1) / BK;
  long long s = (WG_TARGET_CTAS + tiles - 1) / tiles;
  const long long cap = (long long)(WG_WS_CAP / ((size_t)Co * K * sizeof(float)));
  s = s < cap ? s : cap;
  s = s < nsteps ? s : nsteps;
  if (s < 1) s = 1;
  const long long steps = (nsteps + s - 1) / s;
  WgradSplit w;
  w.steps = (int)steps;
  w.splits = (int)((nsteps + steps - 1) / steps);
  return w;
}

int check_shape(const char *what, int B, int C, int H, int W, int Co, int precision) {
  if (B < 1 || C < 1 || H < 1 || W < 1 || Co < 1 || B > 65535)
    return fail(CPB200_ERR_ARG, "%s: bad shape B=%d C=%d H=%d W=%d Co=%d", what, B, C, H, W, Co);
  if ((long long)B * C * H * W >= (1ll << 31) || (long long)B * 2 * TAPS * H * W >= (1ll << 31) ||
      (long long)B * Co * H * W >= (1ll << 31) || (long long)C * TAPS * Co >= (1ll << 31))
    return fail(CPB200_ERR_ARG, "%s: tensors over 2^31 elements", what);
  if (precision != TRAIN_TF32X3 && precision != TRAIN_FP32)
    return fail(CPB200_ERR_ARG, "%s: unknown precision %d", what, precision);
  return CPB200_OK;
}

size_t data_smem_bytes() { return sizeof(DataSmem); }

}  // namespace
}  // namespace cpb

using namespace cpb;

extern "C" size_t cpb200_dcn_train_workspace_bytes(int B, int C, int H, int W, int Co) {
  if (check_shape("dcn_train_workspace_bytes", B, C, H, W, Co, 0) != CPB200_OK) return 0;
  const WgradSplit s = wgrad_split(B, C, H, W, Co);
  return (size_t)s.splits * Co * C * TAPS * sizeof(float);
}

extern "C" int cpb200_dcn_train_forward(const float *input, const float *weight, const float *bias,
                                        const float *offset, const float *mask, float *output, int B, int C, int H,
                                        int W, int Co, int precision, void *stream) {
  if (int st = check_shape("dcn_train_forward", B, C, H, W, Co, precision)) return st;
  if (!input || !weight || !bias || !offset || !mask || !output)
    return fail(CPB200_ERR_ARG, "dcn_train_forward: null pointer");
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 grid(ceil_div(H * W, BN), ceil_div(Co, BM), B);
  if (precision == TRAIN_TF32X3) {
    dcn_fwd_kernel<TRAIN_TF32X3><<<grid, NT, 0, s>>>(input, weight, bias, offset, mask, output, C, H, W, Co);
    return check_launch("dcn_fwd_kernel<tf32x3>", dcn_fwd_kernel<TRAIN_TF32X3>);
  }
  dcn_fwd_kernel<TRAIN_FP32><<<grid, NT, 0, s>>>(input, weight, bias, offset, mask, output, C, H, W, Co);
  return check_launch("dcn_fwd_kernel<fp32>", dcn_fwd_kernel<TRAIN_FP32>);
}

template <int P>
static int dcn_backward_impl(const float *input, const float *weight, const float *offset, const float *mask,
                             const float *grad_output, float *grad_input, float *grad_offset, float *grad_mask,
                             float *grad_weight, float *grad_bias, int B, int C, int H, int W, int Co, float *part,
                             WgradSplit ws, cudaStream_t s) {
  const size_t smem = data_smem_bytes();
  CPB_CUDA(cudaFuncSetAttribute(dcn_bwd_data_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CPB_CUDA(cudaMemsetAsync(grad_input, 0, (size_t)B * C * H * W * sizeof(float), s));
  const int HW = H * W, K = C * TAPS;
  dcn_bwd_data_kernel<P><<<dim3(ceil_div(HW, BN), B), NT, smem, s>>>(input, weight, offset, mask, grad_output,
                                                                      grad_input, grad_offset, grad_mask, C, H, W, Co);
  if (int st = check_launch("dcn_bwd_data_kernel", dcn_bwd_data_kernel<P>)) return st;
  dcn_bwd_weight_kernel<P><<<dim3(ceil_div(K, BN), ceil_div(Co, BM), ws.splits), NT, 0, s>>>(
      input, offset, mask, grad_output, part, B, C, H, W, Co, ws.steps);
  if (int st = check_launch("dcn_bwd_weight_kernel", dcn_bwd_weight_kernel<P>)) return st;
  const int n = Co * K;
  dcn_wgrad_reduce_kernel<<<ceil_div(n, 256) < 1024 ? ceil_div(n, 256) : 1024, 256, 0, s>>>(part, grad_weight, n,
                                                                                             ws.splits);
  if (int st = check_launch("dcn_wgrad_reduce_kernel", dcn_wgrad_reduce_kernel)) return st;
  dcn_bgrad_kernel<<<Co, NT, 0, s>>>(grad_output, grad_bias, B, Co, HW);
  return check_launch("dcn_bgrad_kernel", dcn_bgrad_kernel);
}

extern "C" int cpb200_dcn_train_backward(const float *input, const float *weight, const float *offset,
                                         const float *mask, const float *grad_output, float *grad_input,
                                         float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias,
                                         int B, int C, int H, int W, int Co, int precision, void *workspace,
                                         size_t workspace_bytes, void *stream) {
  if (int st = check_shape("dcn_train_backward", B, C, H, W, Co, precision)) return st;
  if (!input || !weight || !offset || !mask || !grad_output || !grad_input || !grad_offset || !grad_mask ||
      !grad_weight || !grad_bias || !workspace)
    return fail(CPB200_ERR_ARG, "dcn_train_backward: null pointer");
  const WgradSplit ws = wgrad_split(B, C, H, W, Co);
  const size_t need = (size_t)ws.splits * Co * C * TAPS * sizeof(float);
  if (workspace_bytes < need)
    return fail(CPB200_ERR_ARG, "dcn_train_backward: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  float *part = static_cast<float *>(workspace);
  if (precision == TRAIN_TF32X3)
    return dcn_backward_impl<TRAIN_TF32X3>(input, weight, offset, mask, grad_output, grad_input, grad_offset, grad_mask,
                                         grad_weight, grad_bias, B, C, H, W, Co, part, ws, s);
  return dcn_backward_impl<TRAIN_FP32>(input, weight, offset, mask, grad_output, grad_input, grad_offset, grad_mask,
                                     grad_weight, grad_bias, B, C, H, W, Co, part, ws, s);
}

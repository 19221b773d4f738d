// The six keypoint heads of KeypointHead (lib/models/heads/keypoint.py) for training: out_h = W2_h . relu(conv3x3(x,
// W0_h) + b0_h) + b2_h for h in HEADS order, with their backward.  Tensors are the reference's: x (B, C, H, W) NCHW
// fp32; the weights concatenated in HEADS order, W0 (6*hc, C, 3, 3), b0 (6*hc), W2 (58, hc), b2 (58); head h owns
// W2 rows [OUT_OFF[h], OUT_OFF[h + 1]).
//
// The hc x H x W hidden maps never reach HBM.  Each pass is a tiled GEMM whose column operand is gathered from NCHW
// tensors as the tile fills (integer taps, zero padding).  Hidden row j of head h is global row R = h*hc + j.
//   forward      pre[j, p] = sum_r W0[R, r] col(x)[r, p]          tile 64 hidden x 128 pixels, K = C*9
//                out[o, p] = b2[o] + sum_j W2[o, j] relu(pre + b0)[j, p], chunk by chunk from shared memory
//   backward, per chunk of images (make_plan: d_hidden of a chunk at most 256 MiB):
//     1. hidden   recompute pre with the forward's own routine; dpre = (W2^T g) * [pre + b0 > 0] into the workspace;
//                 per-CTA partials of dW2 = g . relu(pre + b0)^T, db0 = sum_p dpre and db2 = sum_p g
//     2. data     dx[c, p] = sum_{h, j, tap} W0[R, c, tap] dpre[R, p - tap]     tile 64 channels x 128 pixels,
//                 K = (heads with a gradient) * hc * 9, one owner per element
//     3. weight   dW0[R, r] = sum_p dpre[R, p] col(x)[r, p]               tile 64 rows x 128 (c, tap), K = pixels,
//                 split K; the partials are summed in split order
//
// Precision: train_mma.cuh's TRAIN_TF32X3 (3xTF32 tensor cores) or TRAIN_FP32 (CUDA cores) for the three GEMMs and the
// hidden-to-output product; dW2 and the bias sums are CUDA-core fp32 in both.  The long sums of passes 2 and 3 and
// every reduction over partials are compensated (Kahan).  Every output and gradient is a sum in a fixed order: the
// same bits on every run.
#include "common.cuh"
#include "train_mma.cuh"
#include "../../include/centerpose_b200_heads_train.h"

namespace cpb {
namespace {

using namespace train;
constexpr int TAPS = 9;
constexpr int NHEADS = 6;
constexpr int NOUT = 58;                                   // 1 + 2 + 34 + 2 + 17 + 2 output channels
constexpr int MAX_OUT = 34;                                // hps
constexpr int GROWS = 48;                                  // MAX_OUT rounded up to BK
__constant__ int OUT_OFF[NHEADS + 1] = {0, 1, 3, 37, 39, 56, 58};
constexpr size_t DH_CHUNK_BYTES = size_t(256) << 20;      // d_hidden of one image chunk, all six heads
constexpr int WG_TARGET_CTAS = 264;                        // weight-gradient split K: two CTAs per SM of a 132-SM H100
constexpr size_t WG_WS_CAP = size_t(16) << 20;             // and its per-split partials under 16 MiB

struct Shape {
  int C, H, W, hc;
};

// head h's map of the struct (a switch, not an index into the struct, keeps the parameter out of local memory)
__device__ __forceinline__ const float *head_map(const cpb200_multi_pose_heads &m, int h) {
  switch (h) {
    case 0: return m.hm;
    case 1: return m.wh;
    case 2: return m.hps;
    case 3: return m.reg;
    case 4: return m.hm_hp;
    default: return m.hp_offset;
  }
}

// ---- the hidden pre-activation of one tile: pre[j0 + m, p0 + n] for m < 64, n < 128 ----------------------------
// Used by the forward and by the backward's recompute, so the ReLU mask is the forward's bit for bit.
template <int P>
__device__ __forceinline__ void hidden_pre(const float *__restrict__ xb, const float *__restrict__ w0h, int j0,
                                           int p0, const Shape &s, float (*As)[AP], float (*Bs)[BP], int tid,
                                           float (&acc)[2][4][4]) {
  const int HW = s.H * s.W, K = s.C * TAPS;
  const int lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  zero_acc(acc);
  for (int r0 = 0; r0 < K; r0 += BK) {
    __syncthreads();
    for (int e = tid; e < BM * BK; e += NT) {
      const int m = e / BK, k = e % BK;
      As[m][k] = (j0 + m < s.hc && r0 + k < K) ? __ldg(w0h + (size_t)(j0 + m) * K + r0 + k) : 0.f;
    }
    for (int e = tid; e < BK * BN; e += NT) {
      const int k = e / BN, n = e % BN, r = r0 + k, p = p0 + n;
      float v = 0.f;
      if (r < K && p < HW) {
        const int c = r / TAPS, tap = r - c * TAPS;
        const int y = p / s.W + tap / 3 - 1, x = p % s.W + tap % 3 - 1;
        if (y >= 0 && y < s.H && x >= 0 && x < s.W) v = __ldg(xb + (size_t)c * HW + y * s.W + x);
      }
      Bs[k][n] = v;
    }
    __syncthreads();
    tile_mma<P>(As, Bs, wm, wn, lane, acc);
  }
}

// Hs[m][n] = relu(pre + b0) of the tile; rows past hc are 0.
__device__ __forceinline__ void stage_hidden(const float (&acc)[2][4][4], const float *__restrict__ b0h, int j0,
                                             int hc, int tid, float (*Hs)[BP]) {
  const int lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3, gid = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = wm * 32 + mt * 16 + gid + 8 * h;
      const float b = j0 + m < hc ? b0h[j0 + m] : 0.f;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j)
          Hs[m][wn * 32 + nt * 8 + 2 * tig + j] = fmaxf(__fadd_rn(acc[mt][nt][2 * h + j], b), 0.f);
    }
}

// ---- forward ------------------------------------------------------------------------------------------------------
// grid (pixel tiles of BN, 6 heads, B).  The CTA walks its head's hidden channels in chunks of BM: pre-activation,
// bias and ReLU into shared memory, then acc_out (outputs x pixels) += W2[:, chunk] . Hs.
struct FwdSmem {
  float As[BM][AP];
  float Bs[BK][BP];
  float Hs[BM][BP];
};

template <int P>
__global__ void __launch_bounds__(NT) heads_fwd_kernel(const float *__restrict__ x, const float *__restrict__ w0,
                                                       const float *__restrict__ b0, const float *__restrict__ w2,
                                                       const float *__restrict__ b2, cpb200_multi_pose_heads out,
                                                       Shape s) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FwdSmem &sm = *reinterpret_cast<FwdSmem *>(smem_raw);
  const int HW = s.H * s.W, K = s.C * TAPS;
  const int p0 = blockIdx.x * BN, head = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  const int o_off = OUT_OFF[head], nout = OUT_OFF[head + 1] - o_off;
  const float *xb = x + (size_t)b * s.C * HW;
  const float *w0h = w0 + (size_t)head * s.hc * K;
  float acc_out[2][4][4];
  zero_acc(acc_out);
  for (int j0 = 0; j0 < s.hc; j0 += BM) {
    float acc[2][4][4];
    hidden_pre<P>(xb, w0h, j0, p0, s, sm.As, sm.Bs, tid, acc);
    stage_hidden(acc, b0 + head * s.hc, j0, s.hc, tid, sm.Hs);
    for (int k0 = 0; k0 < BM && j0 + k0 < s.hc; k0 += BK) {
      __syncthreads();
      for (int e = tid; e < BM * BK; e += NT) {
        const int m = e / BK, k = e % BK, j = j0 + k0 + k;
        sm.As[m][k] = (m < nout && j < s.hc) ? __ldg(w2 + (size_t)(o_off + m) * s.hc + j) : 0.f;
      }
      __syncthreads();
      tile_mma<P>(sm.As, &sm.Hs[k0], wm, wn, lane, acc_out);
    }
  }
  float *ob = const_cast<float *>(head_map(out, head)) + (size_t)b * nout * HW;
  const int gid = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int o = wm * 32 + mt * 16 + gid + 8 * h;
      if (o >= nout) continue;
      const float bo = b2[o_off + o];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int p = p0 + wn * 32 + nt * 8 + 2 * tig + j;
          if (p < HW) ob[(size_t)o * HW + p] = __fadd_rn(acc_out[mt][nt][2 * h + j], bo);
        }
    }
}

// ---- backward 1: recompute the hidden tile, d_hidden and the per-CTA partials of dW2, db0, db2 -------------------
// grid (pixel tiles of BN, 6 heads, images of the chunk).  Slot (image, tile) of the partials holds, over all heads,
// dW2 (58 x hc), then db0 (6*hc), then db2 (58): slot_floats(hc) floats.
__host__ __device__ inline size_t slot_floats(int hc) { return (size_t)NOUT * hc + (size_t)NHEADS * hc + NOUT; }

struct HidSmem {
  float As[BM][AP];
  float Bs[BK][BP];
  float Hs[BM][BP];
  float G[GROWS][BP];      // g_h of the tile, rows past the head's outputs and pixels past HW are 0
};

// sum_n a[n] * b[n] over the BN pixels of a tile: BK-long FMA chains, their sums added left to right
__device__ __forceinline__ float dot_tile(const float *a, const float *b) {
  float s = 0.f;
  for (int n0 = 0; n0 < BN; n0 += BK) {
    float t = 0.f;
#pragma unroll
    for (int n = 0; n < BK; ++n) t = fmaf(a[n0 + n], b[n0 + n], t);
    s = __fadd_rn(s, t);
  }
  return s;
}

__device__ __forceinline__ float sum_tile(const float *a) {
  float s = 0.f;
  for (int n0 = 0; n0 < BN; n0 += BK) {
    float t = 0.f;
#pragma unroll
    for (int n = 0; n < BK; ++n) t = __fadd_rn(t, a[n0 + n]);
    s = __fadd_rn(s, t);
  }
  return s;
}

template <int P>
__global__ void __launch_bounds__(NT, 1) heads_bwd_hidden_kernel(const float *__restrict__ x, const float *__restrict__ w0,
                                                              const float *__restrict__ b0,
                                                              const float *__restrict__ w2,
                                                              cpb200_multi_pose_heads gout, float *__restrict__ dh,
                                                              float *__restrict__ part, int b_begin, Shape s) {
  const int head = blockIdx.y;
  const float *gh = head_map(gout, head);
  if (!gh) return;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  HidSmem &sm = *reinterpret_cast<HidSmem *>(smem_raw);
  const int HW = s.H * s.W, K = s.C * TAPS, ntiles = gridDim.x;
  const int p0 = blockIdx.x * BN, bl = blockIdx.z, b = b_begin + bl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  const int gid = lane >> 2, tig = lane & 3;
  const int o_off = OUT_OFF[head], nout = OUT_OFF[head + 1] - o_off;
  const float *xb = x + (size_t)b * s.C * HW;
  const float *w0h = w0 + (size_t)head * s.hc * K;
  float *slot = part + ((size_t)bl * ntiles + blockIdx.x) * slot_floats(s.hc);
  for (int e = tid; e < GROWS * BN; e += NT) {
    const int o = e / BN, n = e % BN, p = p0 + n;
    sm.G[o][n] = (o < nout && p < HW) ? __ldg(gh + ((size_t)b * nout + o) * HW + p) : 0.f;
  }
  __syncthreads();
  for (int o = tid; o < nout; o += NT) slot[(size_t)NOUT * s.hc + (size_t)NHEADS * s.hc + o_off + o] = sum_tile(sm.G[o]);
  for (int j0 = 0; j0 < s.hc; j0 += BM) {
    float acc[2][4][4];
    hidden_pre<P>(xb, w0h, j0, p0, s, sm.As, sm.Bs, tid, acc);
    stage_hidden(acc, b0 + head * s.hc, j0, s.hc, tid, sm.Hs);
    __syncthreads();
    // dW2[o, j0 + m] over this tile's pixels
    for (int e = tid; e < nout * BM; e += NT) {
      const int o = e / BM, m = e % BM;
      if (j0 + m < s.hc) slot[(size_t)(o_off + o) * s.hc + j0 + m] = dot_tile(sm.G[o], sm.Hs[m]);
    }
    // dpre = W2[:, chunk]^T . g, K = the head's outputs
    zero_acc(acc);
    for (int k0 = 0; k0 < nout; k0 += BK) {
      __syncthreads();
      for (int e = tid; e < BM * BK; e += NT) {
        const int m = e % BM, k = e / BM, o = k0 + k;
        sm.As[m][k] = (o < nout && j0 + m < s.hc) ? __ldg(w2 + (size_t)(o_off + o) * s.hc + j0 + m) : 0.f;
      }
      __syncthreads();
      tile_mma<P>(sm.As, &sm.G[k0], wm, wn, lane, acc);
    }
    // mask in place: each thread rewrites the Hs entries of its own fragment
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = wm * 32 + mt * 16 + gid + 8 * h;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int n = wn * 32 + nt * 8 + 2 * tig + j;
            sm.Hs[m][n] = (sm.Hs[m][n] > 0.f && p0 + n < HW) ? acc[mt][nt][2 * h + j] : 0.f;
          }
      }
    __syncthreads();
    for (int m = tid / 32; m < BM && j0 + m < s.hc; m += NT / 32) {
      float *row = dh + ((size_t)bl * NHEADS * s.hc + (size_t)head * s.hc + j0 + m) * HW;
      for (int n = lane; n < BN; n += 32)
        if (p0 + n < HW) row[p0 + n] = sm.Hs[m][n];
    }
    for (int m = tid; m < BM && j0 + m < s.hc; m += NT)
      slot[(size_t)NOUT * s.hc + (size_t)head * s.hc + j0 + m] = sum_tile(sm.Hs[m]);
  }
}

// ---- backward 2: dx = sum over the heads with a gradient of conv3x3^T(d_hidden, W0) ------------------------------
// grid (pixel tiles of BN, channel tiles of BM, images of the chunk).  K runs head by head over (j, tap); the column
// operand reads d_hidden at the flipped tap.
template <int P>
__global__ void __launch_bounds__(NT) heads_bwd_data_kernel(const float *__restrict__ w0, const float *__restrict__ dh,
                                                            float *__restrict__ dx, int active, int b_begin, Shape s) {
  __shared__ float As[BM][AP];
  __shared__ __align__(16) float Bs[BK][BP];
  const int HW = s.H * s.W, KH = s.hc * TAPS;
  const int p0 = blockIdx.x * BN, c0 = blockIdx.y * BM, bl = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  float acc[2][4][4], comp[2][4][4];
  zero_acc(acc);
  zero_acc(comp);
  for (int head = 0; head < NHEADS; ++head) {
    if (!(active >> head & 1)) continue;
    const float *dhh = dh + ((size_t)bl * NHEADS + head) * s.hc * HW;
    const float *w0h = w0 + (size_t)head * s.hc * s.C * TAPS;
    for (int r0 = 0; r0 < KH; r0 += BK) {
      __syncthreads();
      for (int e = tid; e < BM * BK; e += NT) {
        const int m = e % BM, k = e / BM, r = r0 + k;
        float v = 0.f;
        if (r < KH && c0 + m < s.C) {
          const int j = r / TAPS, tap = r - j * TAPS;
          v = __ldg(w0h + ((size_t)j * s.C + c0 + m) * TAPS + tap);
        }
        As[m][k] = v;
      }
      for (int e = tid; e < BK * BN; e += NT) {
        const int k = e / BN, n = e % BN, r = r0 + k, p = p0 + n;
        float v = 0.f;
        if (r < KH && p < HW) {
          const int j = r / TAPS, tap = r - j * TAPS;
          const int y = p / s.W + 1 - tap / 3, x = p % s.W + 1 - tap % 3;
          if (y >= 0 && y < s.H && x >= 0 && x < s.W) v = dhh[(size_t)j * HW + y * s.W + x];
        }
        Bs[k][n] = v;
      }
      __syncthreads();
      tile_mma_kahan<P>(As, Bs, wm, wn, lane, acc, comp);
    }
  }
  const int gid = lane >> 2, tig = lane & 3;
  float *dxb = dx + (size_t)(b_begin + bl) * s.C * HW;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = c0 + wm * 32 + mt * 16 + gid + 8 * h;
      if (c >= s.C) continue;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int p = p0 + wn * 32 + nt * 8 + 2 * tig + j;
          if (p < HW) dxb[(size_t)c * HW + p] = acc[mt][nt][2 * h + j];
        }
    }
}

// ---- backward 3: partial[split] = d_hidden (6*hc x pixels of the split) . col(x)^T (pixels x C*9) ----------------
// grid (C*9 tiles of BN, 6*hc tiles of BM, splits).  Rows of heads without a gradient read 0.
template <int P>
__global__ void __launch_bounds__(NT) heads_bwd_weight_kernel(const float *__restrict__ x, const float *__restrict__ dh,
                                                              float *__restrict__ part, int active, int b_begin,
                                                              int nimg, int steps_per_split, Shape s) {
  __shared__ float As[BM][AP];
  __shared__ __align__(16) float Bs[BK][BP];
  const int HW = s.H * s.W, K = s.C * TAPS, NQ = nimg * HW, NR = NHEADS * s.hc;
  const int r0 = blockIdx.x * BN, R0 = blockIdx.y * BM, split = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  float acc[2][4][4], comp[2][4][4];
  zero_acc(acc);
  zero_acc(comp);
  const int q_begin = split * steps_per_split * BK;
  const int q_end = min(NQ, q_begin + steps_per_split * BK);
  for (int q0 = q_begin; q0 < q_end; q0 += BK) {
    __syncthreads();
    for (int e = tid; e < BM * BK; e += NT) {
      const int m = e / BK, k = e % BK, q = q0 + k, R = R0 + m;
      float v = 0.f;
      if (R < NR && q < q_end && (active >> (R / s.hc) & 1)) {
        const int bq = q / HW;
        v = dh[((size_t)bq * NR + R) * HW + (q - bq * HW)];
      }
      As[m][k] = v;
    }
    for (int e = tid; e < BK * BN; e += NT) {
      const int k = e % BK, n = e / BK, r = r0 + n, q = q0 + k;
      float v = 0.f;
      if (r < K && q < q_end) {
        const int c = r / TAPS, tap = r - c * TAPS, bq = q / HW, p = q - bq * HW;
        const int y = p / s.W + tap / 3 - 1, xx = p % s.W + tap % 3 - 1;
        if (y >= 0 && y < s.H && xx >= 0 && xx < s.W)
          v = __ldg(x + ((size_t)(b_begin + bq) * s.C + c) * HW + y * s.W + xx);
      }
      Bs[k][n] = v;
    }
    __syncthreads();
    tile_mma_kahan<P>(As, Bs, wm, wn, lane, acc, comp);
  }
  const int gid = lane >> 2, tig = lane & 3;
  float *ps = part + (size_t)split * NR * K;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int R = R0 + wm * 32 + mt * 16 + gid + 8 * h;
      if (R >= NR) continue;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int r = r0 + wn * 32 + nt * 8 + 2 * tig + j;
          if (r < K) ps[(size_t)R * K + r] = acc[mt][nt][2 * h + j];
        }
    }
}

// sum over k < n of src[k * stride + i], compensated, in k order
__device__ __forceinline__ float kahan_sum(const float *src, size_t stride, int n, size_t i) {
  float s = 0.f, c = 0.f;
  for (int k = 0; k < n; ++k) {
    const float y = __fsub_rn(src[(size_t)k * stride + i], c);
    const float t = __fadd_rn(s, y);
    c = __fsub_rn(__fsub_rn(t, s), y);
    s = t;
  }
  return s;
}

// dW0 += sum of the split partials, in split order
__global__ void heads_wgrad_reduce_kernel(const float *__restrict__ part, float *__restrict__ gw0, int splits,
                                          int active, int hc, int K) {
  const size_t n = (size_t)NHEADS * hc * K;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (!(active >> (int)(i / ((size_t)hc * K)) & 1)) continue;
    gw0[i] = __fadd_rn(gw0[i], kahan_sum(part, n, splits, i));
  }
}

// dW2, db0, db2 += sum of the slots' partials, in slot order
__global__ void heads_slot_reduce_kernel(const float *__restrict__ part, float *__restrict__ gw2,
                                         float *__restrict__ gb0, float *__restrict__ gb2, int slots, int active,
                                         int hc) {
  const size_t n = slot_floats(hc), nw2 = (size_t)NOUT * hc, nb0 = (size_t)NHEADS * hc;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float *dst;
    int head;
    if (i < nw2) {
      const int o = (int)(i / hc);
      head = 0;
      while (o >= OUT_OFF[head + 1]) ++head;
      dst = gw2 + i;
    } else if (i < nw2 + nb0) {
      head = (int)((i - nw2) / hc);
      dst = gb0 + (i - nw2);
    } else {
      const int o = (int)(i - nw2 - nb0);
      head = 0;
      while (o >= OUT_OFF[head + 1]) ++head;
      dst = gb2 + o;
    }
    if (!(active >> head & 1)) continue;
    *dst = __fadd_rn(*dst, kahan_sum(part, n, slots, i));
  }
}

// ---- host --------------------------------------------------------------------------------------------------------
struct Plan {
  int chunk;               // images per chunk
  int tiles;               // pixel tiles per image
  size_t dh_floats;        // d_hidden of one chunk
  size_t part1_floats;     // hidden-pass partials of one chunk
  size_t part0_floats;     // weight-gradient partials of the chunk with the most splits
};

struct Split { int splits, steps; };

Split wgrad_split(int nimg, int C, int H, int W, int hc) {
  const long long K = (long long)C * TAPS, NR = (long long)NHEADS * hc;
  const long long tiles = ((K + BN - 1) / BN) * ((NR + BM - 1) / BM);
  const long long nsteps = ((long long)nimg * H * W + BK - 1) / BK;
  long long s = (WG_TARGET_CTAS + tiles - 1) / tiles;
  const long long cap = (long long)(WG_WS_CAP / ((size_t)NR * K * sizeof(float)));
  s = s < cap ? s : cap;
  s = s < nsteps ? s : nsteps;
  if (s < 1) s = 1;
  const long long steps = (nsteps + s - 1) / s;
  return Split{(int)((nsteps + steps - 1) / steps), (int)steps};
}

Plan make_plan(int B, int C, int H, int W, int hc) {
  Plan p;
  const size_t per_image = (size_t)NHEADS * hc * H * W * sizeof(float);
  const size_t n = DH_CHUNK_BYTES / per_image;
  p.chunk = (int)(n < 1 ? 1 : (n < (size_t)B ? n : (size_t)B));
  p.tiles = ceil_div(H * W, BN);
  p.dh_floats = (size_t)p.chunk * NHEADS * hc * H * W;
  p.part1_floats = (size_t)p.chunk * p.tiles * slot_floats(hc);
  // a short last chunk can split into more parts than a full one
  const int last = B % p.chunk ? B % p.chunk : p.chunk;
  const int splits = max(wgrad_split(p.chunk, C, H, W, hc).splits, wgrad_split(last, C, H, W, hc).splits);
  p.part0_floats = (size_t)splits * NHEADS * hc * C * TAPS;
  return p;
}

int check_shape(const char *what, int B, int C, int H, int W, int hc, int precision) {
  if (B < 1 || C < 1 || H < 1 || W < 1 || hc < 1 || B > 65535)
    return fail(CPB200_ERR_ARG, "%s: bad shape B=%d C=%d H=%d W=%d hc=%d", what, B, C, H, W, hc);
  if ((long long)B * C * H * W >= (1ll << 31) || (long long)B * MAX_OUT * H * W >= (1ll << 31) ||
      (long long)NHEADS * hc * C * TAPS >= (1ll << 31) || (long long)NHEADS * hc * H * W >= (1ll << 31))
    return fail(CPB200_ERR_ARG, "%s: tensors over 2^31 elements", what);
  if (precision != TRAIN_TF32X3 && precision != TRAIN_FP32)
    return fail(CPB200_ERR_ARG, "%s: unknown precision %d", what, precision);
  return CPB200_OK;
}

size_t workspace_floats(const Plan &p) { return p.dh_floats + p.part1_floats + p.part0_floats; }

int reduce_grid(size_t n) { return (int)(n / 256 + 1 < 2048 ? n / 256 + 1 : 2048); }

template <int P>
int forward_impl(const float *x, const float *w0, const float *b0, const float *w2, const float *b2,
                 cpb200_multi_pose_heads out, int B, Shape s, cudaStream_t st) {
  const int smem = (int)sizeof(FwdSmem);
  CPB_CUDA(cudaFuncSetAttribute(heads_fwd_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  heads_fwd_kernel<P><<<dim3(ceil_div(s.H * s.W, BN), NHEADS, B), NT, smem, st>>>(x, w0, b0, w2, b2, out, s);
  return check_launch("heads_fwd_kernel", heads_fwd_kernel<P>);
}

template <int P>
int backward_impl(const float *x, const float *w0, const float *b0, const float *w2, cpb200_multi_pose_heads gout,
                  float *gx, float *gw0, float *gb0, float *gw2, float *gb2, int B, Shape s, const Plan &pl,
                  float *ws, cudaStream_t st) {
  const int HW = s.H * s.W, K = s.C * TAPS;
  int active = 0;
  for (int h = 0; h < NHEADS; ++h)
    if ((&gout.hm)[h]) active |= 1 << h;
  CPB_CUDA(cudaMemsetAsync(gw0, 0, (size_t)NHEADS * s.hc * K * sizeof(float), st));
  CPB_CUDA(cudaMemsetAsync(gb0, 0, (size_t)NHEADS * s.hc * sizeof(float), st));
  CPB_CUDA(cudaMemsetAsync(gw2, 0, (size_t)NOUT * s.hc * sizeof(float), st));
  CPB_CUDA(cudaMemsetAsync(gb2, 0, (size_t)NOUT * sizeof(float), st));
  if (gx && !active) CPB_CUDA(cudaMemsetAsync(gx, 0, (size_t)B * s.C * HW * sizeof(float), st));
  if (!active) return CPB200_OK;
  float *dh = ws, *part1 = ws + pl.dh_floats, *part0 = part1 + pl.part1_floats;
  const int smem = (int)sizeof(HidSmem);
  CPB_CUDA(cudaFuncSetAttribute(heads_bwd_hidden_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  for (int b0i = 0; b0i < B; b0i += pl.chunk) {
    const int n = B - b0i < pl.chunk ? B - b0i : pl.chunk;
    heads_bwd_hidden_kernel<P><<<dim3(pl.tiles, NHEADS, n), NT, smem, st>>>(x, w0, b0, w2, gout, dh, part1, b0i, s);
    if (int e = check_launch("heads_bwd_hidden_kernel", heads_bwd_hidden_kernel<P>)) return e;
    if (gx) {
      heads_bwd_data_kernel<P><<<dim3(pl.tiles, ceil_div(s.C, BM), n), NT, 0, st>>>(w0, dh, gx, active, b0i, s);
      if (int e = check_launch("heads_bwd_data_kernel", heads_bwd_data_kernel<P>)) return e;
    }
    const Split sp = wgrad_split(n, s.C, s.H, s.W, s.hc);
    heads_bwd_weight_kernel<P><<<dim3(ceil_div(K, BN), ceil_div(NHEADS * s.hc, BM), sp.splits), NT, 0, st>>>(
        x, dh, part0, active, b0i, n, sp.steps, s);
    if (int e = check_launch("heads_bwd_weight_kernel", heads_bwd_weight_kernel<P>)) return e;
    const size_t n0 = (size_t)NHEADS * s.hc * K;
    heads_wgrad_reduce_kernel<<<reduce_grid(n0), 256, 0, st>>>(part0, gw0, sp.splits, active, s.hc, K);
    if (int e = check_launch("heads_wgrad_reduce_kernel", heads_wgrad_reduce_kernel)) return e;
    heads_slot_reduce_kernel<<<reduce_grid(slot_floats(s.hc)), 256, 0, st>>>(part1, gw2, gb0, gb2, n * pl.tiles,
                                                                             active, s.hc);
    if (int e = check_launch("heads_slot_reduce_kernel", heads_slot_reduce_kernel)) return e;
  }
  return CPB200_OK;
}

}  // namespace
}  // namespace cpb

using namespace cpb;

extern "C" size_t cpb200_heads_train_workspace_bytes(int B, int C, int H, int W, int hc) {
  if (check_shape("heads_train_workspace_bytes", B, C, H, W, hc, 0) != CPB200_OK) return 0;
  return workspace_floats(make_plan(B, C, H, W, hc)) * sizeof(float);
}

extern "C" int cpb200_heads_train_forward(const float *x, const float *w0, const float *b0, const float *w2,
                                          const float *b2, cpb200_multi_pose_heads out, int B, int C, int H, int W,
                                          int hc, int precision, void *stream) {
  if (int e = check_shape("heads_train_forward", B, C, H, W, hc, precision)) return e;
  if (!x || !w0 || !b0 || !w2 || !b2 || !out.hm || !out.wh || !out.hps || !out.reg || !out.hm_hp || !out.hp_offset)
    return fail(CPB200_ERR_ARG, "heads_train_forward: null pointer");
  const Shape s{C, H, W, hc};
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == TRAIN_TF32X3) return forward_impl<TRAIN_TF32X3>(x, w0, b0, w2, b2, out, B, s, st);
  return forward_impl<TRAIN_FP32>(x, w0, b0, w2, b2, out, B, s, st);
}

extern "C" int cpb200_heads_train_backward(const float *x, const float *w0, const float *b0, const float *w2,
                                           cpb200_multi_pose_heads grad_output, float *grad_x, float *grad_w0,
                                           float *grad_b0, float *grad_w2, float *grad_b2, int B, int C, int H,
                                           int W, int hc, int precision, void *workspace, size_t workspace_bytes,
                                           void *stream) {
  if (int e = check_shape("heads_train_backward", B, C, H, W, hc, precision)) return e;
  if (!x || !w0 || !b0 || !w2 || !grad_w0 || !grad_b0 || !grad_w2 || !grad_b2 || !workspace)
    return fail(CPB200_ERR_ARG, "heads_train_backward: null pointer");
  const Plan pl = make_plan(B, C, H, W, hc);
  const size_t need = workspace_floats(pl) * sizeof(float);
  if (workspace_bytes < need)
    return fail(CPB200_ERR_ARG, "heads_train_backward: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  const Shape s{C, H, W, hc};
  cudaStream_t st = (cudaStream_t)stream;
  float *ws = static_cast<float *>(workspace);
  if (precision == TRAIN_TF32X3)
    return backward_impl<TRAIN_TF32X3>(x, w0, b0, w2, grad_output, grad_x, grad_w0, grad_b0, grad_w2, grad_b2, B, s,
                                       pl, ws, st);
  return backward_impl<TRAIN_FP32>(x, w0, b0, w2, grad_output, grad_x, grad_w0, grad_b0, grad_w2, grad_b2, B, s, pl,
                                   ws, st);
}

// CUDA-core (SIMT) implementations of the fused network ops, fp32 accumulate, activations
// fp32 or bf16 NHWC.  This is the "precise" path (act_dtype = fp32 reproduces the reference's
// fp32 arithmetic up to summation order) and the fallback for layers whose shapes the
// wgmma path (net_tc.cu) does not take.  Reference semantics per op:
//   CONV          torch.nn.Conv2d + folded eval BatchNorm2d (+ residual add) (+ ReLU)
//                 e.g. pose_dla_dcn.py:43-57 (BasicBlock), :155-163 (Root: the torch.cat of
//                 the children is never materialised — each child is one K-slab), :199-204
//   STEM          pose_dla_dcn.py:226-231 base_layer (7x7, 3->16) on the NCHW fp32 image
//   MAXPOOL       pose_dla_dcn.py:196 nn.MaxPool2d(stride), msra_resnet.py:126
//   DWDECONV_ADD  pose_dla_dcn.py:361-364,374-377: depthwise ConvTranspose2d(2f, stride f,
//                 pad f/2) followed by `+ layers[i-1]`
//   DCN           DCNv2/dcn_v2.py:117-127 + DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:25-54,125-195
//                 + dcn_v2_cuda.cu:123-163: sigmoid(mask) * bilinear sample, then the GEMM —
//                 fused here: the sampled im2col tile lives in shared memory only (the
//                 reference round-trips a (B, 9C, HW) fp32 `columns` buffer through HBM).
#include "common.cuh"
#include <cuda_fp16.h>
#include <cstdlib>
#include <algorithm>

namespace {

using bf16 = __nv_bfloat16;

template <typename T> struct Act;
template <> struct Act<float> {
  __device__ static float4 ld4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
  __device__ static float ld(const float *p) { return __ldg(p); }
  __device__ static void st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
  __device__ static void st(float *p, float v) { *p = v; }
};
template <> struct Act<bf16> {
  __device__ static float4 ld4(const bf16 *p) {
    uint2 r = __ldg(reinterpret_cast<const uint2 *>(p));
    float2 a = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&r.x));
    float2 b = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  __device__ static float ld(const bf16 *p) { return __bfloat162float(*p); }
  __device__ static void st4(bf16 *p, float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 r; r.x = *reinterpret_cast<unsigned *>(&a); r.y = *reinterpret_cast<unsigned *>(&b);
    *reinterpret_cast<uint2 *>(p) = r;
  }
  __device__ static void st(bf16 *p, float v) { *p = __float2bfloat16_rn(v); }
};

// ------------------------------------------------------------------------------------------------------------
// Split-operand activations (CPB200_BF16X2 / CPB200_F16X2): a value is hi + lo, two 16-bit planes `plane` elements apart
// (include/centerpose_b200.h).  hi + lo is exact in fp32 and split(hi + lo) reproduces the value exactly, so max-pooling
// and copies are lossless; arithmetic happens in fp32 and the result is re-split.
struct Sp16 {
  __device__ static float2 up(uint32_t v, uint32_t fmt) {
    if (fmt) return __half22float2(*reinterpret_cast<const __half2 *>(&v));
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&v));
  }
  __device__ static float4 ld4(const uint16_t *p, size_t plane, uint32_t fmt) {
    const uint2 h = __ldg(reinterpret_cast<const uint2 *>(p)), l = __ldg(reinterpret_cast<const uint2 *>(p + plane));
    const float2 h0 = up(h.x, fmt), h1 = up(h.y, fmt), l0 = up(l.x, fmt), l1 = up(l.y, fmt);
    return make_float4(h0.x + l0.x, h0.y + l0.y, h1.x + l1.x, h1.y + l1.y);
  }
  __device__ static void split2(float a, float b, uint32_t fmt, uint32_t &hi, uint32_t &lo) {
    if (fmt) {
      a = fminf(fmaxf(a, -65504.f), 65504.f); b = fminf(fmaxf(b, -65504.f), 65504.f);
      const __half2 h = __floats2half2_rn(a, b);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
      hi = *reinterpret_cast<const uint32_t *>(&h); lo = *reinterpret_cast<const uint32_t *>(&l);
    } else {
      const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
      const float2 hf = __bfloat1622float2(h);
      const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
      hi = *reinterpret_cast<const uint32_t *>(&h); lo = *reinterpret_cast<const uint32_t *>(&l);
    }
  }
  __device__ static void st4(uint16_t *p, size_t plane, uint32_t fmt, float4 v) {
    uint2 h, l;
    split2(v.x, v.y, fmt, h.x, l.x); split2(v.z, v.w, fmt, h.y, l.y);
    *reinterpret_cast<uint2 *>(p) = h;
    *reinterpret_cast<uint2 *>(p + plane) = l;
  }
};


// Pointer-like handles of split activations, so the element-wise kernels below take fp32, bf16 or split tensors on
// either side through the same source: `p + n` advances both planes, io_ld4 joins hi + lo, io_st4 re-splits.
struct SpC {
  const uint16_t *p; size_t plane; uint32_t fmt;
  __host__ __device__ SpC operator+(size_t n) const { return SpC{p + n, plane, fmt}; }
  __host__ __device__ explicit operator bool() const { return p != nullptr; }
};
struct SpM {
  uint16_t *p; size_t plane; uint32_t fmt;
  __host__ __device__ SpM operator+(size_t n) const { return SpM{p + n, plane, fmt}; }
};
__device__ __forceinline__ float4 io_ld4(const float *p) { return Act<float>::ld4(p); }
__device__ __forceinline__ float4 io_ld4(const bf16 *p) { return Act<bf16>::ld4(p); }
__device__ __forceinline__ float4 io_ld4(SpC p) { return Sp16::ld4(p.p, p.plane, p.fmt); }
__device__ __forceinline__ void io_st4(float *p, float4 v) { Act<float>::st4(p, v); }
__device__ __forceinline__ void io_st4(bf16 *p, float4 v) { Act<bf16>::st4(p, v); }
__device__ __forceinline__ void io_st4(SpM p, float4 v) { Sp16::st4(p.p, p.plane, p.fmt, v); }

struct ConvArgs {
  const void *src[4];
  int cin[4];
  int pitch[4];              // elements between pixels of each input (== cin unless the input is a channel slice)
  int nsrc;
  const void *res;
  const float *aux;       // DCN: (B,H,W,aux_pitch) fp32 offsets+mask logits
  int aux_pitch;
  void *dst;
  const float *weight;    // [taps][cin_total][cout_pad]
  const float *bias;
  int B, H, W, Ho, Wo, Hd, Wd;
  int cin_total, cout, cout_pad;
  int kh, kw, stride, pad_h, pad_w;
  int out_sy, out_sx, out_oy, out_ox;
  int out_ch_off, out_ch_total;
  unsigned flags;
};

constexpr int BK = 16;

// Implicit-GEMM conv: M = B*Ho*Wo output pixels, N = cout, K = taps * cin_total.
// CTA = 256 threads computes a BM x BN tile, 4x4 outputs per thread... (TM x TN generic).
template <typename T, int BM, int BN, bool DCN>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvArgs a) {
  constexpr int TM = 4;
  constexpr int TN = (BM * BN) / (256 * TM);       // 64x64 -> 4, 128x32 -> 4, 256x16 -> 4
  static_assert(TN == 4, "tile must give 4x4 outputs per thread");
  constexpr int TX = BN / TN;                       // threads along N
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ int s_coff[DCN ? 4 : 1][DCN ? BM : 1];     // DCN: 4 corner element offsets per pixel
  __shared__ float s_cwt[DCN ? 4 : 1][DCN ? BM : 1];    // DCN: 4 corner weights (x mask x validity)

  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const long long M = (long long)a.B * a.Ho * a.Wo;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  // per-thread A-load assignment: pixel slots i = lid/4 (+64 per round), channel quad kq = lid%4
  constexpr int A_ROUNDS = BM / 64;
  int pb[A_ROUNDS], pho[A_ROUNDS], pwo[A_ROUNDS];
  bool pok[A_ROUNDS];
#pragma unroll
  for (int r = 0; r < A_ROUNDS; ++r) {
    const long long m = m0 + (tid >> 2) + 64 * r;
    pok[r] = m < M;
    const long long mm = pok[r] ? m : 0;
    pb[r] = (int)(mm / ((long long)a.Ho * a.Wo));
    const int rem = (int)(mm % ((long long)a.Ho * a.Wo));
    pho[r] = rem / a.Wo; pwo[r] = rem % a.Wo;
  }
  const int kq = tid & 3;
  const int taps = a.kh * a.kw;

  for (int tap = 0; tap < taps; ++tap) {
    const int r_ = tap / a.kw, q_ = tap % a.kw;
    if (DCN) {
      __syncthreads();
      for (int i = tid; i < BM; i += 256) {
        const long long m = m0 + i;
        int off[4] = {0, 0, 0, 0}; float wt[4] = {0.f, 0.f, 0.f, 0.f};
        if (m < M) {
          const int b = (int)(m / ((long long)a.Ho * a.Wo));
          const int rem = (int)(m % ((long long)a.Ho * a.Wo));
          const int ho = rem / a.Wo, wo = rem % a.Wo;
          const float *om = a.aux + ((size_t)m) * a.aux_pitch;
          const float oh = __ldg(om + 2 * tap), ow = __ldg(om + 2 * tap + 1);
          const float mk = 1.0f / (1.0f + expf(-__ldg(om + 18 + tap)));      // dcn_v2.py:121
          const float h_im = (float)(ho * a.stride - a.pad_h + r_) + oh;      // im2col_cuda.cu:177-178
          const float w_im = (float)(wo * a.stride - a.pad_w + q_) + ow;
          if (h_im > -1.f && w_im > -1.f && h_im < (float)a.H && w_im < (float)a.W) {   // :180
            const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
            const int h_high = h_low + 1, w_high = w_low + 1;
            const float lh = h_im - h_low, lw = w_im - w_low, hh = 1.f - lh, hw = 1.f - lw;
            const size_t rowb = (size_t)b * a.H;
            if (h_low >= 0 && w_low >= 0) { off[0] = (int)(((rowb + h_low) * a.W + w_low)); wt[0] = hh * hw * mk; }
            if (h_low >= 0 && w_high <= a.W - 1) { off[1] = (int)(((rowb + h_low) * a.W + w_high)); wt[1] = hh * lw * mk; }
            if (h_high <= a.H - 1 && w_low >= 0) { off[2] = (int)(((rowb + h_high) * a.W + w_low)); wt[2] = lh * hw * mk; }
            if (h_high <= a.H - 1 && w_high <= a.W - 1) { off[3] = (int)(((rowb + h_high) * a.W + w_high)); wt[3] = lh * lw * mk; }
          }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) { s_coff[c][i] = off[c]; s_cwt[c][i] = wt[c]; }
      }
      __syncthreads();
    }
    int cbase = 0;
    for (int s = 0; s < a.nsrc; ++s) {
      const T *src = static_cast<const T *>(a.src[s]);
      const int cs = a.cin[s], ps = a.pitch[s];
      for (int c0 = 0; c0 < cs; c0 += BK) {
        // ---- A tile: BM pixels x 16 channels ----
        float4 av[A_ROUNDS];
#pragma unroll
        for (int r = 0; r < A_ROUNDS; ++r) {
          av[r] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (!DCN) {
            const int hi = pho[r] * a.stride - a.pad_h + r_, wi = pwo[r] * a.stride - a.pad_w + q_;
            if (pok[r] && hi >= 0 && hi < a.H && wi >= 0 && wi < a.W)
              av[r] = Act<T>::ld4(src + (((size_t)pb[r] * a.H + hi) * a.W + wi) * ps + c0 + kq * 4);
          } else {
            const int i = (tid >> 2) + 64 * r;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float wgt = s_cwt[c][i];
              if (wgt != 0.f) {
                const float4 v = Act<T>::ld4(src + (size_t)s_coff[c][i] * ps + c0 + kq * 4);
                av[r].x += wgt * v.x; av[r].y += wgt * v.y; av[r].z += wgt * v.z; av[r].w += wgt * v.w;
              }
            }
          }
        }
        // ---- B tile: 16 x BN weights ----
        constexpr int B_LOADS = (BK * BN / 4 + 255) / 256;     // float4 loads per thread
        float4 bv[B_LOADS];
#pragma unroll
        for (int l = 0; l < B_LOADS; ++l) {
          const int e = tid + 256 * l;
          const int k = e / (BN / 4), nq = e % (BN / 4);
          bv[l] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (k < BK && n0 + nq * 4 < a.cout_pad)
            bv[l] = __ldg(reinterpret_cast<const float4 *>(
                a.weight + ((size_t)tap * a.cin_total + cbase + c0 + k) * a.cout_pad + n0 + nq * 4));
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < A_ROUNDS; ++r) {
          const int i = (tid >> 2) + 64 * r;
          As[kq * 4 + 0][i] = av[r].x; As[kq * 4 + 1][i] = av[r].y;
          As[kq * 4 + 2][i] = av[r].z; As[kq * 4 + 3][i] = av[r].w;
        }
#pragma unroll
        for (int l = 0; l < B_LOADS; ++l) {
          const int e = tid + 256 * l;
          const int k = e / (BN / 4), nq = e % (BN / 4);
          if (k < BK) *reinterpret_cast<float4 *>(&Bs[k][nq * 4]) = bv[l];
        }
        __syncthreads();
        // blocked summation: each 16-deep chunk is reduced on its own, then added to the running
        // sum — error grows with K/16 + 16 instead of K (matters for K = 9*512 in fp32 parity mode)
        float part[TM][TN];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) part[i][j] = 0.f;
#pragma unroll
        for (int k = 0; k < BK; ++k) {
          const float4 a4 = *reinterpret_cast<const float4 *>(&As[k][ty * TM]);
          const float4 b4 = *reinterpret_cast<const float4 *>(&Bs[k][tx * TN]);
          const float ar[4] = {a4.x, a4.y, a4.z, a4.w}, br[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) part[i][j] = fmaf(ar[i], br[j], part[i][j]);
        }
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] += part[i][j];
      }
      cbase += cs;
    }
  }

  // ---- epilogue ----
  const uint32_t act = a.flags & CPB_ACT_MASK;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long m = m0 + ty * TM + i;
    if (m >= M) continue;
    const int b = (int)(m / ((long long)a.Ho * a.Wo));
    const int rem = (int)(m % ((long long)a.Ho * a.Wo));
    const int ho = rem / a.Wo, wo = rem % a.Wo;
    const int hd = ho * a.out_sy + a.out_oy, wd = wo * a.out_sx + a.out_ox;
    const size_t pix = ((size_t)b * a.Hd + hd) * a.Wd + wd;
    float v[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      v[j] = acc[i][j] + ((a.bias && n < a.cout) ? __ldg(a.bias + n) : 0.f);
    }
    const int nb = n0 + tx * TN;
    if (a.flags & CPB200_FLAG_OUT_NCHW_F32) {
      float *o = static_cast<float *>(a.dst);
#pragma unroll
      for (int j = 0; j < TN; ++j)
        if (nb + j < a.cout) {
          float x = v[j]; x = cpb::act_out<T>(x, act);
          o[(((size_t)b * a.out_ch_total + a.out_ch_off + nb + j) * a.Hd + hd) * a.Wd + wd] = x;
        }
    } else if (a.flags & CPB200_FLAG_OUT_F32) {
      float *o = static_cast<float *>(a.dst) + pix * a.cout;
#pragma unroll
      for (int j = 0; j < TN; ++j)
        if (nb + j < a.cout) { float x = v[j]; x = cpb::act_out<T>(x, act); o[nb + j] = x; }
    } else {
      T *o = static_cast<T *>(a.dst) + pix * a.cout;
      const T *rs = a.res ? static_cast<const T *>(a.res) + pix * a.cout : nullptr;
      if (nb + TN <= a.cout && (a.cout & 3) == 0) {
        float4 x = make_float4(v[0], v[1], v[2], v[3]);
        if (rs) { float4 r4 = Act<T>::ld4(rs + nb); x.x += r4.x; x.y += r4.y; x.z += r4.z; x.w += r4.w; }
        if (act) { x.x = cpb::act_out<T>(x.x, act); x.y = cpb::act_out<T>(x.y, act); x.z = cpb::act_out<T>(x.z, act); x.w = cpb::act_out<T>(x.w, act); }
        Act<T>::st4(o + nb, x);
      } else {
#pragma unroll
        for (int j = 0; j < TN; ++j)
          if (nb + j < a.cout) {
            float x = v[j];
            if (rs) x += Act<T>::ld(rs + nb + j);
            x = cpb::act_out<T>(x, act);
            Act<T>::st(o + nb + j, x);
          }
      }
    }
  }
}

// ---- STEM: NCHW fp32 (B,Cin<=4,H,W) -> NHWC (B,Ho,Wo,Cout<=64), direct conv, bias + ReLU ----
// weight layout: [kh*kw*cin][cout] fp32 in shared memory.  One thread = PX consecutive output
// pixels of one row x all couts: every weight vector fetched from shared memory feeds PX pixels
// (PX*COUT FMAs per COUT/4 LDS.128), the input row segment is read once into registers.
template <typename T, int COUT, int PX, int STRIDE, int KW>
__global__ void __launch_bounds__(128) stem_kernel(const float *__restrict__ x, T *__restrict__ y,
                                                   const float *__restrict__ w, const float *__restrict__ bias,
                                                   int B, int Cin, int H, int W, int Ho, int Wo,
                                                   int kh, int pad_h, int pad_w, uint32_t act) {
  extern __shared__ float sw[];                      // kh*KW*cin*COUT
  const int nw = kh * KW * Cin * COUT;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int WG = Wo / PX;                            // pixel groups per row (Wo % PX == 0 checked by the host)
  const long long M = (long long)B * Ho * WG;
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int b = (int)(m / ((long long)Ho * WG));
  const int rem = (int)(m % ((long long)Ho * WG));
  const int ho = rem / WG, wo0 = (rem % WG) * PX;
  float acc[PX][COUT];
#pragma unroll
  for (int p = 0; p < PX; ++p)
#pragma unroll
    for (int n = 0; n < COUT; ++n) acc[p][n] = bias ? __ldg(bias + n) : 0.f;
  constexpr int SEG = (PX - 1) * STRIDE + KW;        // input columns feeding PX outputs
  const int wi0 = wo0 * STRIDE - pad_w;
  for (int r = 0; r < kh; ++r) {
    const int hi = ho * STRIDE - pad_h + r;
    if (hi < 0 || hi >= H) continue;
    for (int c = 0; c < Cin; ++c) {
      const float *row = x + (((size_t)b * Cin + c) * H + hi) * W;
      float in[SEG];
#pragma unroll
      for (int i = 0; i < SEG; ++i) { const int wi = wi0 + i; in[i] = (wi >= 0 && wi < W) ? __ldg(row + wi) : 0.f; }
#pragma unroll
      for (int q = 0; q < KW; ++q) {
        const float4 *wp = reinterpret_cast<const float4 *>(sw + ((r * KW + q) * Cin + c) * COUT);
#pragma unroll
        for (int n4 = 0; n4 < COUT / 4; ++n4) {
          const float4 w4 = wp[n4];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const float v = in[p * STRIDE + q];
            acc[p][4 * n4] = fmaf(v, w4.x, acc[p][4 * n4]); acc[p][4 * n4 + 1] = fmaf(v, w4.y, acc[p][4 * n4 + 1]);
            acc[p][4 * n4 + 2] = fmaf(v, w4.z, acc[p][4 * n4 + 2]); acc[p][4 * n4 + 3] = fmaf(v, w4.w, acc[p][4 * n4 + 3]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    T *o = y + ((((size_t)b * Ho + ho) * Wo) + wo0 + p) * COUT;
#pragma unroll
    for (int n = 0; n < COUT; n += 4) {
      float4 v = make_float4(acc[p][n], acc[p][n + 1], acc[p][n + 2], acc[p][n + 3]);
      if (act) { v.x = cpb::act_out<T>(v.x, act); v.y = cpb::act_out<T>(v.y, act); v.z = cpb::act_out<T>(v.z, act); v.w = cpb::act_out<T>(v.w, act); }
      Act<T>::st4(o + n, v);
    }
  }
}

// ---- IM2COL_W: NCHW fp32 (B,cin,H,W) -> NHWC (B,H,W,COUT): channel s*cin+c = x[c,h,w+s-pad], zero padded ----
template <typename T, int COUT>
__global__ void __launch_bounds__(256) im2col_w_kernel(const float *__restrict__ x, T *__restrict__ y, int B, int Cin,
                                                       int H, int W, int kw, int pad) {
  const long long M = (long long)B * H * W;
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int w = (int)(m % W);
  const int h = (int)((m / W) % H);
  const int b = (int)(m / ((long long)W * H));
  float v[COUT];
#pragma unroll
  for (int i = 0; i < COUT; ++i) v[i] = 0.f;
  for (int c = 0; c < Cin; ++c) {
    const float *row = x + (((size_t)b * Cin + c) * H + h) * W;
    for (int s_ = 0; s_ < kw; ++s_) {
      const int wi = w + s_ - pad;
      const float val = (wi >= 0 && wi < W) ? __ldg(row + wi) : 0.f;
      const int ch = s_ * Cin + c;
#pragma unroll
      for (int i = 0; i < COUT; ++i) if (i == ch) v[i] = val;      // static indexing keeps v[] in registers
    }
  }
  T *o = y + (size_t)m * COUT;
#pragma unroll
  for (int i = 0; i < COUT; i += 4) Act<T>::st4(o + i, make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]));
}

// ---- MAXPOOL k x k / stride / pad, NHWC, 4 channels per thread ----
template <typename T>
__global__ void maxpool_kernel(const T *__restrict__ x, T *__restrict__ y, int B, int H, int W, int C,
                               int Ho, int Wo, int k, int stride, int pad) {
  const int C4 = C >> 2;
  const long long total = (long long)B * Ho * Wo * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    long long p = i / C4;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < k; ++r) {
      const int hi = ho * stride - pad + r;
      if (hi < 0 || hi >= H) continue;
      for (int q = 0; q < k; ++q) {
        const int wi = wo * stride - pad + q;
        if (wi < 0 || wi >= W) continue;
        const float4 v = Act<T>::ld4(x + (((size_t)b * H + hi) * W + wi) * C + c4 * 4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    Act<T>::st4(y + (((size_t)b * Ho + ho) * Wo + wo) * C + c4 * 4, m);
  }
}

// ---- depthwise ConvTranspose2d(k=2f, stride f, pad f/2) + skip add, NHWC ----
// out[b,ho,wo,c] = skip[b,ho,wo,c] + sum_{kh,kw : (ho+p-kh)%f==0, (wo+p-kw)%f==0} x[b,(ho+p-kh)/f,(wo+p-kw)/f,c] * w[kh,kw,c]
// One CTA = one output row (b, ho); thread = (wo, group of VEC channels), VEC*sizeof(T) = 16 bytes.  The
// k*k*C filter taps sit in shared memory; no integer division in the inner loop.
template <typename T, int VEC>
__global__ void __launch_bounds__(256) dwdeconv_add_kernel(const T *__restrict__ x, const T *__restrict__ skip, T *__restrict__ y,
                                                           const float *__restrict__ w, int H, int W, int C, int Ho, int Wo,
                                                           int k, int f, int pad, int lf, int lcv) {
  // f and C / VEC are powers of two (lf = log2 f, lcv = log2(C / VEC), or -1 -> generic division):
  // the per-element index arithmetic is shifts and masks only.
  extern __shared__ float sw[];                       // [k*k][C]
  for (int i = threadIdx.x; i < k * k * C; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int CV = C / VEC;
  const int b = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  const int kh0 = (ho + pad) % f;
  const T *xb = x + (size_t)b * H * W * C;
  const bool fast = lf >= 0 && lcv >= 0;
  for (int i = threadIdx.x; i < Wo * CV; i += blockDim.x) {
    const int wo = fast ? (i >> lcv) : (i / CV), cv = i - wo * CV;
    const size_t opix = (((size_t)b * Ho + ho) * Wo + wo) * C + cv * VEC;
    float acc[VEC];
#pragma unroll
    for (int q = 0; q < VEC; q += 4) {
      float4 s4 = skip ? Act<T>::ld4(skip + opix + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[q] = s4.x; acc[q + 1] = s4.y; acc[q + 2] = s4.z; acc[q + 3] = s4.w;
    }
    const int kw0 = fast ? ((wo + pad) & (f - 1)) : ((wo + pad) % f);
    for (int khh = kh0; khh < k; khh += f) {
      const int hn = ho + pad - khh;
      const int hi = fast ? (hn >> lf) : (hn / f);
      if (hn < 0 || hi >= H) continue;
      for (int kww = kw0; kww < k; kww += f) {
        const int wn = wo + pad - kww;
        const int wi = fast ? (wn >> lf) : (wn / f);
        if (wn < 0 || wi >= W) continue;
        const T *xp = xb + ((size_t)hi * W + wi) * C + cv * VEC;
        const float *wp = sw + (khh * k + kww) * C + cv * VEC;
#pragma unroll
        for (int q = 0; q < VEC; q += 4) {
          const float4 v = Act<T>::ld4(xp + q);
          const float4 ww = *reinterpret_cast<const float4 *>(wp + q);
          acc[q] = fmaf(v.x, ww.x, acc[q]); acc[q + 1] = fmaf(v.y, ww.y, acc[q + 1]);
          acc[q + 2] = fmaf(v.z, ww.z, acc[q + 2]); acc[q + 3] = fmaf(v.w, ww.w, acc[q + 3]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < VEC; q += 4) Act<T>::st4(y + opix + q, make_float4(acc[q], acc[q + 1], acc[q + 2], acc[q + 3]));
  }
}

// Fast path for the shapes IDAUp uses (k == 2f, f and C/VEC powers of two, 256 % (f * C/VEC) == 0): every item a
// thread visits in one output row has the same channel group and the same column parity class, so its four
// (kh, kw) tap weight vectors are loaded into registers ONCE per CTA instead of 8 LDS.128 per item.
template <typename T, int VEC>
__global__ void __launch_bounds__(256) dwdeconv_add_fast_kernel(const T *__restrict__ x, const T *__restrict__ skip, T *__restrict__ y,
                                                                const float *__restrict__ w, int H, int W, int C, int Ho, int Wo,
                                                                int k, int f, int pad, int lf, int lcv) {
  const int CV = C / VEC;
  const int b = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  const int i0 = threadIdx.x;
  const int wo_first = i0 >> lcv, cv = i0 & (CV - 1);
  const int kh0 = (ho + pad) & (f - 1), kw0 = (wo_first + pad) & (f - 1);
  float wt[2][2][VEC];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float *wp = w + (size_t)((kh0 + a * f) * k + kw0 + c * f) * C + cv * VEC;
#pragma unroll
      for (int q = 0; q < VEC; q += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(wp + q));
        wt[a][c][q] = v.x; wt[a][c][q + 1] = v.y; wt[a][c][q + 2] = v.z; wt[a][c][q + 3] = v.w;
      }
    }
  const T *xb = x + (size_t)b * H * W * C + cv * VEC;
  const int hn0 = ho + pad - kh0;                               // >= 0; tap a reads input row (hn0 >> lf) - a
  const int hi0 = hn0 >> lf;
  const size_t orow = ((size_t)b * Ho + ho) * Wo;
  for (int i = i0; i < Wo * CV; i += 256) {
    const int wo = i >> lcv;
    const size_t opix = (orow + wo) * C + cv * VEC;
    float acc[VEC];
#pragma unroll
    for (int q = 0; q < VEC; q += 4) {
      float4 s4 = skip ? Act<T>::ld4(skip + opix + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[q] = s4.x; acc[q + 1] = s4.y; acc[q + 2] = s4.z; acc[q + 3] = s4.w;
    }
    const int wi0 = (wo + pad - kw0) >> lf;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int hi = hi0 - a;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int wi = wi0 - c;
        if (wi < 0 || wi >= W) continue;
        const T *xp = xb + ((size_t)hi * W + wi) * C;
#pragma unroll
        for (int q = 0; q < VEC; q += 4) {
          const float4 v = Act<T>::ld4(xp + q);
          acc[q] = fmaf(v.x, wt[a][c][q], acc[q]); acc[q + 1] = fmaf(v.y, wt[a][c][q + 1], acc[q + 1]);
          acc[q + 2] = fmaf(v.z, wt[a][c][q + 2], acc[q + 2]); acc[q + 3] = fmaf(v.w, wt[a][c][q + 3], acc[q + 3]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < VEC; q += 4) Act<T>::st4(y + opix + q, make_float4(acc[q], acc[q + 1], acc[q + 2], acc[q + 3]));
  }
}

// ---- nearest-neighbour upsample x f (+ skip add)(+ReLU), NHWC ----
// out[b,ho,wo,c] = act(skip[b,ho,wo,c] + x[b,ho/f,wo/f,c])     (HRNet fuse_layers, pose_higher_hrnet.py:186-187,224-232)
// Thread = 4 channels of one output pixel; f is a power of two (shift).
template <typename T, typename PI = const T *, typename PO = T *>
__global__ void __launch_bounds__(256) upsample_add_kernel(PI x, PI skip, PO y,
                                                           long long total, int H, int W, int C4, int Ho, int Wo, int sh, uint32_t act) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    long long p = i / C4;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float4 v = io_ld4(x + ((((size_t)b * H + (ho >> sh)) * W + (wo >> sh)) * C4 + c4) * 4);
    if (skip) {
      const float4 s4 = io_ld4(skip + (size_t)i * 4);
      v.x += s4.x; v.y += s4.y; v.z += s4.z; v.w += s4.w;
    }
    if (act) { v.x = cpb::act_out<T>(v.x, act); v.y = cpb::act_out<T>(v.y, act); v.z = cpb::act_out<T>(v.z, act); v.w = cpb::act_out<T>(v.w, act); }
    io_st4(y + (size_t)i * 4, v);
  }
}

// ---- depthwise k x k conv (stride s, pad k/2) + bias + activation, NHWC   (mobilenetv3.py:124-127 conv2/bn2) ----
// y[b,ho,wo,c] = act(bias[c] + sum_{r,q} x[b, ho*s-p+r, wo*s-p+q, c] * w[r,q,c]).  Thread = VEC channels of one
// output pixel (VEC * sizeof(T) = 16 bytes); consecutive threads walk the channels of a pixel, so every tap is
// a coalesced row read that the neighbouring output pixels re-read from L1.  HBM-bound: 2 bytes in + out per MAC x k^2.
template <typename T, int VEC, typename PI = const T *, typename PO = T *>
__global__ void __launch_bounds__(256) dwconv_kernel(PI x, PO y, const float *__restrict__ w,
                                                     const float *__restrict__ bias, long long total, int H, int W, int C,
                                                     int Ho, int Wo, int k, int stride, int pad, uint32_t act) {
  const int CV = C / VEC;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    long long p = i / CV;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int b = (int)(p / Ho);
    const int c0 = cv * VEC;
    float acc[VEC];
#pragma unroll
    for (int q = 0; q < VEC; q += 4) {
      const float4 b4 = bias ? __ldg(reinterpret_cast<const float4 *>(bias + c0 + q)) : make_float4(0.f, 0.f, 0.f, 0.f);
      acc[q] = b4.x; acc[q + 1] = b4.y; acc[q + 2] = b4.z; acc[q + 3] = b4.w;
    }
    const int hi0 = ho * stride - pad, wi0 = wo * stride - pad;
    for (int r = 0; r < k; ++r) {
      const int hi = hi0 + r;
      if (hi < 0 || hi >= H) continue;
      for (int s = 0; s < k; ++s) {
        const int wi = wi0 + s;
        if (wi < 0 || wi >= W) continue;
        const PI xp = x + (((size_t)b * H + hi) * W + wi) * C + c0;
        const float *wp = w + (size_t)(r * k + s) * C + c0;
#pragma unroll
        for (int q = 0; q < VEC; q += 4) {
          const float4 v = io_ld4(xp + q);
          const float4 ww = __ldg(reinterpret_cast<const float4 *>(wp + q));
          acc[q] = fmaf(v.x, ww.x, acc[q]); acc[q + 1] = fmaf(v.y, ww.y, acc[q + 1]);
          acc[q + 2] = fmaf(v.z, ww.z, acc[q + 2]); acc[q + 3] = fmaf(v.w, ww.w, acc[q + 3]);
        }
      }
    }
    const PO o = y + (size_t)i * VEC;
#pragma unroll
    for (int q = 0; q < VEC; q += 4)
      io_st4(o + q, make_float4(cpb::act_out<T>(acc[q], act), cpb::act_out<T>(acc[q + 1], act), cpb::act_out<T>(acc[q + 2], act),
                                     cpb::act_out<T>(acc[q + 3], act)));
  }
}

// Register-tiled variant for the shapes MobileNetV3 uses (k in {3,5}, stride in {1,2}): a thread produces PXW
// adjacent output pixels of one row for VEC channels, so each input vector of the row segment is loaded once and
// each tap's weight vector feeds PXW pixels (the generic kernel above issues 3 loads per tap per pixel).
template <typename T, int VEC, int K, int S, int PXW, typename PI = const T *, typename PO = T *>
__global__ void __launch_bounds__(256) dwconv_tiled_kernel(PI x, PO y, const float *__restrict__ w,
                                                           const float *__restrict__ bias, long long total, int H, int W, int C,
                                                           int Ho, int Wo, uint32_t act) {
  constexpr int NIN = (PXW - 1) * S + K, PAD = K / 2;
  const int CV = C / VEC, WG = (Wo + PXW - 1) / PXW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % CV);
    long long p = i / CV;
    const int wg = (int)(p % WG); p /= WG;
    const int ho = (int)(p % Ho);
    const int b = (int)(p / Ho);
    const int c0 = cv * VEC, wo0 = wg * PXW;
    float acc[PXW][VEC];
#pragma unroll
    for (int q = 0; q < VEC; q += 4) {
      const float4 b4 = bias ? __ldg(reinterpret_cast<const float4 *>(bias + c0 + q)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int px = 0; px < PXW; ++px) { acc[px][q] = b4.x; acc[px][q + 1] = b4.y; acc[px][q + 2] = b4.z; acc[px][q + 3] = b4.w; }
    }
    const int wi0 = wo0 * S - PAD;
#pragma unroll 1
    for (int r = 0; r < K; ++r) {
      const int hi = ho * S - PAD + r;
      if (hi < 0 || hi >= H) continue;
      const PI xr = x + (((size_t)b * H + hi) * W) * C + c0;
      float in[NIN][VEC];
#pragma unroll
      for (int j = 0; j < NIN; ++j) {
        const int wi = wi0 + j;
        const bool okw = wi >= 0 && wi < W;
#pragma unroll
        for (int q = 0; q < VEC; q += 4) {
          const float4 v = okw ? io_ld4(xr + ((size_t)wi * C + q)) : make_float4(0.f, 0.f, 0.f, 0.f);
          in[j][q] = v.x; in[j][q + 1] = v.y; in[j][q + 2] = v.z; in[j][q + 3] = v.w;
        }
      }
#pragma unroll
      for (int t = 0; t < K; ++t) {
        const float *wp = w + (size_t)(r * K + t) * C + c0;
#pragma unroll
        for (int q = 0; q < VEC; q += 4) {
          const float4 ww = __ldg(reinterpret_cast<const float4 *>(wp + q));
#pragma unroll
          for (int px = 0; px < PXW; ++px) {
            acc[px][q] = fmaf(in[px * S + t][q], ww.x, acc[px][q]);
            acc[px][q + 1] = fmaf(in[px * S + t][q + 1], ww.y, acc[px][q + 1]);
            acc[px][q + 2] = fmaf(in[px * S + t][q + 2], ww.z, acc[px][q + 2]);
            acc[px][q + 3] = fmaf(in[px * S + t][q + 3], ww.w, acc[px][q + 3]);
          }
        }
      }
    }
#pragma unroll
    for (int px = 0; px < PXW; ++px) {
      if (wo0 + px >= Wo) break;
      const PO o = y + (((((size_t)b * Ho + ho) * Wo) + wo0 + px) * C + c0);
#pragma unroll
      for (int q = 0; q < VEC; q += 4)
        io_st4(o + q, make_float4(cpb::act_out<T>(acc[px][q], act), cpb::act_out<T>(acc[px][q + 1], act),
                                       cpb::act_out<T>(acc[px][q + 2], act), cpb::act_out<T>(acc[px][q + 3], act)));
    }
  }
}

// ---- global average pool (B,H,W,C) -> (B,1,1,C)   (SeModule's AdaptiveAvgPool2d(1), mobilenetv3.py:100) ----
// CTA = (image b, 64-channel chunk): 16 channel quads x 16 pixel lanes, fp32 partial sums, shared-memory tree.
template <typename T, typename PI = const T *, typename PO = T *>
__global__ void __launch_bounds__(256) avgpool_kernel(PI x, PO y, int HW, int C) {
  __shared__ float4 part[16][16];
  const int b = blockIdx.x, cq = blockIdx.y * 16 + (threadIdx.x & 15), lane = threadIdx.x >> 4;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  if (cq * 4 < C) {
    const PI xp = x + ((size_t)b * HW * C + cq * 4);
    for (int p = lane; p < HW; p += 16) {
      const float4 v = io_ld4(xp + (size_t)p * C);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  part[lane][threadIdx.x & 15] = s;
  __syncthreads();
  if (lane == 0 && cq * 4 < C) {
    for (int l = 1; l < 16; ++l) { const float4 v = part[l][threadIdx.x & 15]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    const float inv = 1.f / (float)HW;
    io_st4(y + ((size_t)b * C + cq * 4), make_float4(s.x * inv, s.y * inv, s.z * inv, s.w * inv));
  }
}

// ---- y[b,h,w,c] = x[b,h,w,c] * scale[b,c] (+ skip[b,h,w,c])   (SeModule gate + Block shortcut, mobilenetv3.py:111,146) ----
template <typename T, typename PI = const T *, typename PS = const T *, typename PO = T *>
__global__ void __launch_bounds__(256) scale_add_kernel(PI x, PS scale, PI skip, PO y, long long total, long long per_image, int C4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_image), c4 = (int)(i % C4);
    float4 v = io_ld4(x + (size_t)i * 4);
    const float4 g = io_ld4(scale + ((size_t)b * C4 + c4) * 4);
    v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
    if (skip) {
      const float4 s4 = io_ld4(skip + (size_t)i * 4);
      v.x += s4.x; v.y += s4.y; v.z += s4.z; v.w += s4.w;
    }
    io_st4(y + (size_t)i * 4, v);
  }
}

// fp32 NHWC <-> split planes (CPB200_OP_CONVERT), 4 elements per thread
__global__ void __launch_bounds__(256) convert_to_split_kernel(const float *__restrict__ x, uint16_t *__restrict__ y, long long n4, size_t plane, uint32_t fmt) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    Sp16::st4(y + i * 4, plane, fmt, __ldg(reinterpret_cast<const float4 *>(x) + i));
}
__global__ void __launch_bounds__(256) convert_from_split_kernel(const uint16_t *__restrict__ x, float *__restrict__ y, long long n4, size_t plane, uint32_t fmt) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    reinterpret_cast<float4 *>(y)[i] = Sp16::ld4(x + i * 4, plane, fmt);
}

// max-pool on split planes (pose_dla_dcn.py:196, msra_resnet.py:126): exact (the maximum is one of the inputs)
__global__ void maxpool_split_kernel(const uint16_t *__restrict__ x, uint16_t *__restrict__ y, int B, int H, int W, int C,
                                     int Ho, int Wo, int k, int stride, int pad, uint32_t fmt) {
  const int C4 = C >> 2;
  const long long total = (long long)B * Ho * Wo * C4;
  const size_t xplane = (size_t)B * H * W * C, yplane = (size_t)B * Ho * Wo * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    long long p = i / C4;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int b = (int)(p / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int r = 0; r < k; ++r) {
      const int hi = ho * stride - pad + r;
      if (hi < 0 || hi >= H) continue;
      for (int q = 0; q < k; ++q) {
        const int wi = wo * stride - pad + q;
        if (wi < 0 || wi >= W) continue;
        const float4 v = Sp16::ld4(x + (((size_t)b * H + hi) * W + wi) * C + c4 * 4, xplane, fmt);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    Sp16::st4(y + (((size_t)b * Ho + ho) * Wo + wo) * C + c4 * 4, yplane, fmt, m);
  }
}

// depthwise ConvTranspose2d(k = 2f, stride f, pad f/2) + skip add on split planes (IDAUp up_*, pose_dla_dcn.py:361-364,374-377).
// One CTA = one output row (b, ho); thread = (wo, 4 channels); every output pixel has exactly 2 x 2 contributing taps
// (k == 2f).  fp32 arithmetic, tap weights fp32 [k*k][C].
__global__ void __launch_bounds__(256) dwdeconv_add_split_kernel(const uint16_t *__restrict__ x, const uint16_t *__restrict__ skip,
                                                                 uint16_t *__restrict__ y, const float *__restrict__ w, int B, int H, int W, int C,
                                                                 int Ho, int Wo, int k, int f, int pad, uint32_t fmt) {
  const int C4 = C >> 2;
  const int b = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  const size_t xplane = (size_t)B * H * W * C, yplane = (size_t)B * Ho * Wo * C;
  const int kh0 = (ho + pad) % f;
  for (int i = threadIdx.x; i < Wo * C4; i += blockDim.x) {
    const int wo = i / C4, c4 = i - wo * C4;
    const size_t opix = (((size_t)b * Ho + ho) * Wo + wo) * C + c4 * 4;
    float4 acc = skip ? Sp16::ld4(skip + opix, yplane, fmt) : make_float4(0.f, 0.f, 0.f, 0.f);
    const int kw0 = (wo + pad) % f;
    for (int khh = kh0; khh < k; khh += f) {
      const int hn = ho + pad - khh;
      if (hn < 0) continue;
      const int hi = hn / f;
      if (hi >= H) continue;
      for (int kww = kw0; kww < k; kww += f) {
        const int wn = wo + pad - kww;
        if (wn < 0) continue;
        const int wi = wn / f;
        if (wi >= W) continue;
        const float4 v = Sp16::ld4(x + (((size_t)b * H + hi) * W + wi) * C + c4 * 4, xplane, fmt);
        const float4 ww = __ldg(reinterpret_cast<const float4 *>(w + (size_t)(khh * k + kww) * C + c4 * 4));
        acc.x = fmaf(v.x, ww.x, acc.x); acc.y = fmaf(v.y, ww.y, acc.y); acc.z = fmaf(v.z, ww.z, acc.z); acc.w = fmaf(v.w, ww.w, acc.w);
      }
    }
    Sp16::st4(y + opix, yplane, fmt, acc);
  }
}

// Fast path for the shapes IDAUp uses (k == 2f, f and C/8 powers of two, 256 % (f * C/8) == 0), mirroring
// dwdeconv_add_fast_kernel: thread = (wo, 8 channels) with 16-byte loads per plane, its four (kh, kw) tap weight vectors
// live in registers for the whole output row.  ~9 bytes of HBM traffic per output element (skip 4 + x 4/f^2 + out 4).
__global__ void __launch_bounds__(256) dwdeconv_add_split_fast_kernel(const uint16_t *__restrict__ x, const uint16_t *__restrict__ skip,
                                                                      uint16_t *__restrict__ y, const float *__restrict__ w, int B, int H, int W,
                                                                      int C, int Ho, int Wo, int k, int f, int pad, int lf, int lcv, uint32_t fmt) {
  constexpr int VEC = 8;
  const int CV = C / VEC;
  const int b = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  const int i0 = threadIdx.x;
  const int wo_first = i0 >> lcv, cv = i0 & (CV - 1);
  const int kh0 = (ho + pad) & (f - 1), kw0 = (wo_first + pad) & (f - 1);
  const size_t xplane = (size_t)B * H * W * C, yplane = (size_t)B * Ho * Wo * C;
  float wt[2][2][VEC];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float *wp = w + (size_t)((kh0 + a * f) * k + kw0 + c * f) * C + cv * VEC;
#pragma unroll
      for (int q = 0; q < VEC; q += 4) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(wp + q));
        wt[a][c][q] = v.x; wt[a][c][q + 1] = v.y; wt[a][c][q + 2] = v.z; wt[a][c][q + 3] = v.w;
      }
    }
  const uint16_t *xb = x + (size_t)b * H * W * C + cv * VEC;
  const int hn0 = ho + pad - kh0;                               // >= 0; tap a reads input row (hn0 >> lf) - a
  const int hi0 = hn0 >> lf;
  const size_t orow = ((size_t)b * Ho + ho) * Wo;
  auto ld8 = [&](const uint16_t *p, size_t plane, float (&o)[VEC]) {
    const uint4 h = __ldg(reinterpret_cast<const uint4 *>(p)), l = __ldg(reinterpret_cast<const uint4 *>(p + plane));
    const uint32_t hw_[4] = {h.x, h.y, h.z, h.w}, lw_[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 a = Sp16::up(hw_[j], fmt), c = Sp16::up(lw_[j], fmt);
      o[2 * j] = a.x + c.x; o[2 * j + 1] = a.y + c.y;
    }
  };
#pragma unroll 2                                             // two pixels' loads in flight per thread (HBM-bound kernel)
  for (int i = i0; i < Wo * CV; i += 256) {
    const int wo = i >> lcv;
    const size_t opix = (orow + wo) * C + cv * VEC;
    float acc[VEC];
    if (skip) ld8(skip + opix, yplane, acc);
    else {
#pragma unroll
      for (int q = 0; q < VEC; ++q) acc[q] = 0.f;
    }
    const int wi0 = (wo + pad - kw0) >> lf;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int hi = hi0 - a;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int wi = wi0 - c;
        if (wi < 0 || wi >= W) continue;
        float v[VEC];
        ld8(xb + ((size_t)hi * W + wi) * C, xplane, v);
#pragma unroll
        for (int q = 0; q < VEC; ++q) acc[q] = fmaf(v[q], wt[a][c][q], acc[q]);
      }
    }
    uint4 oh, ol;
    Sp16::split2(acc[0], acc[1], fmt, oh.x, ol.x); Sp16::split2(acc[2], acc[3], fmt, oh.y, ol.y);
    Sp16::split2(acc[4], acc[5], fmt, oh.z, ol.z); Sp16::split2(acc[6], acc[7], fmt, oh.w, ol.w);
    *reinterpret_cast<uint4 *>(y + opix) = oh;
    *reinterpret_cast<uint4 *>(y + opix + yplane) = ol;
  }
}


// ---- space-to-depth of the network input (CPB200_OP_S2D): NCHW fp32 (B,3,H,W) -> split planes (B,H/2,W/2,16) ----
// Thread = one output pixel: six coalesced float2 loads (channel c, row parity py: the two column parities), channel
// (py*2+px)*3 + c, channels 12..15 zero; one 32-byte store per plane.
__global__ void __launch_bounds__(256) s2d_split_kernel(const float *__restrict__ x, uint16_t *__restrict__ y, int B, int H, int W,
                                                        size_t plane, uint32_t fmt) {
  const int Ho = H >> 1, Wo = W >> 1;
  const long long total = (long long)B * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    long long p = i / Wo;
    const int ho = (int)(p % Ho), b = (int)(p / Ho);
    float v[16];
#pragma unroll
    for (int j = 12; j < 16; ++j) v[j] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int py = 0; py < 2; ++py) {
        const float2 t = __ldg(reinterpret_cast<const float2 *>(x + (((size_t)b * 3 + c) * H + 2 * ho + py) * W + 2 * wo));
        v[(py * 2 + 0) * 3 + c] = t.x; v[(py * 2 + 1) * 3 + c] = t.y;
      }
    uint32_t oh[8], ol[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) Sp16::split2(v[2 * j], v[2 * j + 1], fmt, oh[j], ol[j]);
    uint16_t *o = y + (size_t)i * 16;
    *reinterpret_cast<uint4 *>(o) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
    *reinterpret_cast<uint4 *>(o + 8) = make_uint4(oh[4], oh[5], oh[6], oh[7]);
    *reinterpret_cast<uint4 *>(o + plane) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
    *reinterpret_cast<uint4 *>(o + plane + 8) = make_uint4(ol[4], ol[5], ol[6], ol[7]);
  }
}

int run_op_split(const cpb200_op &op, cudaStream_t st) {
  const uint32_t fmt = op.act_dtype == CPB200_F16X2 ? 1u : 0u;
  switch (op.type) {
    case CPB200_OP_CONVERT: {
      const long long n = (long long)op.B * op.H * op.W * op.cin[0];
      if (n % 4) return cpb::fail(CPB200_ERR_ARG, "convert: element count must be a multiple of 4");
      const unsigned grid = (unsigned)std::min<long long>((n / 4 + 255) / 256, 132LL * 16);
      if (op.flags & CPB200_FLAG_TO_F32)
        convert_from_split_kernel<<<grid, 256, 0, st>>>(static_cast<const uint16_t *>(op.src[0]), static_cast<float *>(op.dst), n / 4, (size_t)n, fmt);
      else
        convert_to_split_kernel<<<grid, 256, 0, st>>>(static_cast<const float *>(op.src[0]), static_cast<uint16_t *>(op.dst), n / 4, (size_t)n, fmt);
      return cpb::check_launch("convert_split_kernel");
    }
    case CPB200_OP_S2D: {
      if (op.cin[0] != 3 || op.cout != 16 || (op.H & 1) || (op.W & 1) || op.Ho != op.H / 2 || op.Wo != op.W / 2)
        return cpb::fail(CPB200_ERR_ARG, "s2d: needs a (B,3,H,W) input with even H, W and a 16-channel (B,H/2,W/2) output");
      const long long total = (long long)op.B * op.Ho * op.Wo;
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 16);
      s2d_split_kernel<<<grid, 256, 0, st>>>(static_cast<const float *>(op.src[0]), static_cast<uint16_t *>(op.dst), op.B, op.H, op.W,
                                             (size_t)total * 16, fmt);
      return cpb::check_launch("s2d_split_kernel");
    }
    case CPB200_OP_MAXPOOL: {
      if (op.cin[0] % 4) return cpb::fail(CPB200_ERR_ARG, "maxpool: C %% 4 != 0");
      const long long total = (long long)op.B * op.Ho * op.Wo * (op.cin[0] / 4);
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 32);
      maxpool_split_kernel<<<grid, 256, 0, st>>>(static_cast<const uint16_t *>(op.src[0]), static_cast<uint16_t *>(op.dst),
                                                 op.B, op.H, op.W, op.cin[0], op.Ho, op.Wo, op.kh, op.stride, op.pad_h, fmt);
      return cpb::check_launch("maxpool_split_kernel");
    }
    case CPB200_OP_DWDECONV_ADD: {
      if (op.cin[0] % 4 || op.kh != 2 * op.stride) return cpb::fail(CPB200_ERR_ARG, "dwdeconv (split): needs C %% 4 == 0 and k == 2 * stride");
      {
        auto ilog2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return (1 << l) == v ? l : -1; };
        const int C = op.cin[0];
        const int lf = ilog2(op.stride), lcv = (C % 8 == 0) ? ilog2(C / 8) : -1;
        const int CVv = C / 8;
        if (lf >= 0 && lcv >= 0 && CVv <= 256 && (256 / CVv) % op.stride == 0 && getenv("CPB200_DWDECONV_GENERIC") == nullptr) {
          dwdeconv_add_split_fast_kernel<<<(unsigned)(op.B * op.Ho), 256, 0, st>>>(static_cast<const uint16_t *>(op.src[0]),
              static_cast<const uint16_t *>(op.aux), static_cast<uint16_t *>(op.dst), static_cast<const float *>(op.weight),
              op.B, op.H, op.W, C, op.Ho, op.Wo, op.kh, op.stride, op.pad_h, lf, lcv, fmt);
          return cpb::check_launch("dwdeconv_add_split_fast_kernel");
        }
      }
      dwdeconv_add_split_kernel<<<(unsigned)(op.B * op.Ho), 256, 0, st>>>(static_cast<const uint16_t *>(op.src[0]),
          static_cast<const uint16_t *>(op.aux), static_cast<uint16_t *>(op.dst), static_cast<const float *>(op.weight),
          op.B, op.H, op.W, op.cin[0], op.Ho, op.Wo, op.kh, op.stride, op.pad_h, fmt);
      return cpb::check_launch("dwdeconv_add_split_kernel");
    }
    // The element-wise MobileNetV3 / HRNet ops run their fp32 kernels straight on the planes (SpC / SpM handles):
    // no fp32 island, no CONVERT passes.  fp32 arithmetic on hi + lo, result re-split; the depthwise conv is instantiated
    // with T = bf16 only to select act_out's multiply-by-1/6 h-swish (VEC stays 4: the handles load 8 bytes per plane).
    case CPB200_OP_DWCONV: {
      constexpr int VEC = 4;
      const int C = op.cin[0];
      if (C % VEC || op.kh != op.kw || op.cout != C || (op.src_pitch[0] != 0 && op.src_pitch[0] != C)) return cpb::fail(CPB200_ERR_ARG, "dwconv (split): C %% 4 != 0, non-square kernel or sliced input");
      const SpC x{static_cast<const uint16_t *>(op.src[0]), (size_t)op.B * op.H * op.W * C, fmt};
      const SpM y{static_cast<uint16_t *>(op.dst), (size_t)op.B * op.Ho * op.Wo * C, fmt};
#define DW_TILED(KK, SS, PX)                                                                                   \
  if (op.kh == KK && op.stride == SS && op.pad_h == KK / 2) {                                                    \
    const long long tot = (long long)op.B * op.Ho * ((op.Wo + PX - 1) / PX) * (C / VEC);                         \
    const unsigned g = (unsigned)std::min<long long>((tot + 255) / 256, 132LL * 32);                            \
    dwconv_tiled_kernel<bf16, VEC, KK, SS, PX, SpC, SpM><<<g, 256, 0, st>>>(x, y, static_cast<const float *>(op.weight), \
        op.bias, tot, op.H, op.W, C, op.Ho, op.Wo, op.flags & CPB_ACT_MASK);                                    \
    return cpb::check_launch("dwconv_tiled_kernel");                                                            \
  }
      DW_TILED(3, 1, 4) DW_TILED(5, 1, 4) DW_TILED(3, 2, 2) DW_TILED(5, 2, 2)
#undef DW_TILED
      const long long total = (long long)op.B * op.Ho * op.Wo * (C / VEC);
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 32);
      dwconv_kernel<bf16, VEC, SpC, SpM><<<grid, 256, 0, st>>>(x, y, static_cast<const float *>(op.weight), op.bias, total,
          op.H, op.W, C, op.Ho, op.Wo, op.kh, op.stride, op.pad_h, op.flags & CPB_ACT_MASK);
      return cpb::check_launch("dwconv_kernel");
    }
    case CPB200_OP_AVGPOOL: {                           // split planes in, fp32 (B,1,1,C) out: the SE convs that follow run on fp32
      const int C = op.cin[0];
      if (C % 4 || op.Ho != 1 || op.Wo != 1 || (op.src_pitch[0] != 0 && op.src_pitch[0] != C)) return cpb::fail(CPB200_ERR_ARG, "avgpool (split): C %% 4 != 0, output not 1x1 or sliced input");
      const SpC x{static_cast<const uint16_t *>(op.src[0]), (size_t)op.B * op.H * op.W * C, fmt};
      avgpool_kernel<float, SpC, float *><<<dim3((unsigned)op.B, (unsigned)((C + 63) / 64)), 256, 0, st>>>(x, static_cast<float *>(op.dst), op.H * op.W, C);
      return cpb::check_launch("avgpool_kernel");
    }
    case CPB200_OP_SCALE_ADD: {                         // x, skip, y: split planes; the gate vector (B,1,1,C) is fp32
      const int C = op.cin[0];
      if (C % 4 || !op.res || (op.src_pitch[0] != 0 && op.src_pitch[0] != C)) return cpb::fail(CPB200_ERR_ARG, "scale_add (split): C %% 4 != 0, missing scale vector or sliced input");
      const size_t plane = (size_t)op.B * op.H * op.W * C;
      const long long per_image = (long long)op.H * op.W * (C / 4), total = per_image * op.B;
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 16);
      scale_add_kernel<float, SpC, const float *, SpM><<<grid, 256, 0, st>>>(SpC{static_cast<const uint16_t *>(op.src[0]), plane, fmt},
          static_cast<const float *>(op.res), SpC{static_cast<const uint16_t *>(op.aux), plane, fmt},
          SpM{static_cast<uint16_t *>(op.dst), plane, fmt}, total, per_image, C / 4);
      return cpb::check_launch("scale_add_kernel");
    }
    case CPB200_OP_UPSAMPLE_ADD: {
      const int f = op.stride, C = op.cin[0];
      int sh = 0;
      while ((1 << sh) < f) ++sh;
      if (f < 1 || (1 << sh) != f || op.Ho != op.H * f || op.Wo != op.W * f || C % 4 || (op.src_pitch[0] != 0 && op.src_pitch[0] != C))
        return cpb::fail(CPB200_ERR_ARG, "upsample_add (split): factor %d must be a power of two, C %% 4 == 0, whole-tensor input", f);
      const size_t plane_o = (size_t)op.B * op.Ho * op.Wo * C;
      const long long total = (long long)op.B * op.Ho * op.Wo * (C / 4);
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 16);
      upsample_add_kernel<float, SpC, SpM><<<grid, 256, 0, st>>>(SpC{static_cast<const uint16_t *>(op.src[0]), (size_t)op.B * op.H * op.W * C, fmt},
          SpC{static_cast<const uint16_t *>(op.aux), plane_o, fmt}, SpM{static_cast<uint16_t *>(op.dst), plane_o, fmt},
          total, op.H, op.W, C / 4, op.Ho, op.Wo, sh, op.flags & CPB_ACT_MASK);
      return cpb::check_launch("upsample_add_kernel");
    }
    default:
      return cpb::fail(CPB200_ERR_ARG, "op type %d has no split-precision kernel (the host must route it through fp32)", op.type);
  }
}

template <typename T, bool DCN>
int launch_conv(const cpb200_op &op, cudaStream_t st) {
  ConvArgs a;
  a.cin_total = 0;
  for (int i = 0; i < 4; ++i) {
    a.src[i] = op.src[i]; a.cin[i] = (i < op.nsrc) ? op.cin[i] : 0;
    a.pitch[i] = (i < op.nsrc && op.src_pitch[i] > 0) ? op.src_pitch[i] : a.cin[i];
    if (i < op.nsrc) {
      if (op.cin[i] % BK) return cpb::fail(CPB200_ERR_ARG, "conv: input channels %d not a multiple of %d", op.cin[i], BK);
      a.cin_total += op.cin[i];
    }
  }
  a.nsrc = op.nsrc; a.res = op.res; a.aux = static_cast<const float *>(op.aux); a.aux_pitch = op.aux_pitch > 0 ? op.aux_pitch : 27; a.dst = op.dst;
  a.weight = static_cast<const float *>(op.weight); a.bias = op.bias;
  a.B = op.B; a.H = op.H; a.W = op.W; a.Ho = op.Ho; a.Wo = op.Wo; a.Hd = op.Hd; a.Wd = op.Wd;
  a.cout = op.cout; a.cout_pad = (op.cout + 3) / 4 * 4;
  a.kh = op.kh; a.kw = op.kw; a.stride = op.stride; a.pad_h = op.pad_h; a.pad_w = op.pad_w;
  a.out_sy = op.out_sy; a.out_sx = op.out_sx; a.out_oy = op.out_oy; a.out_ox = op.out_ox;
  a.out_ch_off = op.out_ch_off; a.out_ch_total = op.out_ch_total; a.flags = op.flags;
  const long long M = (long long)op.B * op.Ho * op.Wo;
  if (op.cout <= 16) {
    dim3 grid((unsigned)((M + 255) / 256), (op.cout + 15) / 16);
    conv_simt_kernel<T, 256, 16, DCN><<<grid, 256, 0, st>>>(a);
  } else if (op.cout <= 32) {
    dim3 grid((unsigned)((M + 127) / 128), (op.cout + 31) / 32);
    conv_simt_kernel<T, 128, 32, DCN><<<grid, 256, 0, st>>>(a);
  } else {
    dim3 grid((unsigned)((M + 63) / 64), (op.cout + 63) / 64);
    conv_simt_kernel<T, 64, 64, DCN><<<grid, 256, 0, st>>>(a);
  }
  return cpb::check_launch("conv_simt_kernel");
}

template <typename T>
int run_op_simt(const cpb200_op &op, cudaStream_t st) {
  switch (op.type) {
    case CPB200_OP_CONV: return launch_conv<T, false>(op, st);
    case CPB200_OP_DCN:
      if (op.kh != 3 || op.kw != 3 || !op.aux) return cpb::fail(CPB200_ERR_ARG, "dcn: needs 3x3 kernel and offset/mask tensor");
      return launch_conv<T, true>(op, st);
    case CPB200_OP_STEM: {
      const int cin = op.cin[0];
      const size_t smem = (size_t)op.kh * op.kw * cin * op.cout * sizeof(float);
      if (cin > 4 || smem > 48 * 1024 || (op.kw != 7 && op.kw != 3)) return cpb::fail(CPB200_ERR_ARG, "stem: unsupported shape");
      const uint32_t act = op.flags & CPB_ACT_MASK;
      // (COUT, PX) register tiles: 16 couts x 4 pixels, 64 couts x 1 pixel
#define STEM_LAUNCH(CO, PX, ST) STEM_LAUNCH_K(CO, PX, ST, 7)
#define STEM_LAUNCH_K(CO, PX, ST, KW)                                                                            \
  {                                                                                                          \
    if (op.Wo % PX) return cpb::fail(CPB200_ERR_ARG, "stem: output width %d not a multiple of %d", op.Wo, PX); \
    const long long M = (long long)op.B * op.Ho * (op.Wo / PX);                                              \
    stem_kernel<T, CO, PX, ST, KW><<<(unsigned)((M + 127) / 128), 128, smem, st>>>(                           \
        static_cast<const float *>(op.src[0]), static_cast<T *>(op.dst), static_cast<const float *>(op.weight), \
        op.bias, op.B, cin, op.H, op.W, op.Ho, op.Wo, op.kh, op.pad_h, op.pad_w, act);                      \
  }
      if (op.kw == 3) {                               // HRNet conv1 (pose_higher_hrnet.py:243-244)
        if (op.cout == 64 && op.stride == 2) STEM_LAUNCH_K(64, 1, 2, 3)
        else if (op.cout == 16 && op.stride == 2) STEM_LAUNCH_K(16, 4, 2, 3)      // MobileNetV3 conv1 (mobilenetv3.py:165)
        else return cpb::fail(CPB200_ERR_ARG, "stem 3x3: cout %d / stride %d unsupported", op.cout, op.stride);
      } else if (op.cout == 16 && op.stride == 1) STEM_LAUNCH(16, 4, 1)
      else if (op.cout == 16 && op.stride == 2) STEM_LAUNCH(16, 4, 2)
      else if (op.cout == 32 && op.stride == 2) STEM_LAUNCH(32, 2, 2)
      else if (op.cout == 64 && op.stride == 2) STEM_LAUNCH(64, 1, 2)
      else if (op.cout == 64 && op.stride == 1) STEM_LAUNCH(64, 1, 1)
      else return cpb::fail(CPB200_ERR_ARG, "stem: cout %d / stride %d unsupported", op.cout, op.stride);
#undef STEM_LAUNCH
#undef STEM_LAUNCH_K
      return cpb::check_launch("stem_kernel");
    }
    case CPB200_OP_IM2COL_W: {
      const int cin = op.cin[0];
      if (op.cout != 32 || cin * op.kw > 32) return cpb::fail(CPB200_ERR_ARG, "im2col_w: needs kw*cin <= 32 output channels");
      const long long M = (long long)op.B * op.H * op.W;
      im2col_w_kernel<T, 32><<<(unsigned)((M + 255) / 256), 256, 0, st>>>(static_cast<const float *>(op.src[0]),
          static_cast<T *>(op.dst), op.B, cin, op.H, op.W, op.kw, op.pad_w);
      return cpb::check_launch("im2col_w_kernel");
    }
    case CPB200_OP_MAXPOOL: {
      if (op.cin[0] % 4) return cpb::fail(CPB200_ERR_ARG, "maxpool: C %% 4 != 0");
      const long long total = (long long)op.B * op.Ho * op.Wo * (op.cin[0] / 4);
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 32);
      maxpool_kernel<T><<<grid, 256, 0, st>>>(static_cast<const T *>(op.src[0]), static_cast<T *>(op.dst),
                                              op.B, op.H, op.W, op.cin[0], op.Ho, op.Wo, op.kh, op.stride, op.pad_h);
      return cpb::check_launch("maxpool_kernel");
    }
    case CPB200_OP_DWDECONV_ADD: {
      constexpr int VEC = sizeof(T) == 2 ? 8 : 4;
      if (op.cin[0] % VEC) return cpb::fail(CPB200_ERR_ARG, "dwdeconv: C %% %d != 0", VEC);
      const size_t smem = (size_t)op.kh * op.kh * op.cin[0] * sizeof(float);
      if (smem > 160 * 1024) return cpb::fail(CPB200_ERR_ARG, "dwdeconv: filter does not fit shared memory");
      if (smem > 48 * 1024 &&
          cudaFuncSetAttribute(dwdeconv_add_kernel<T, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return cpb::fail(CPB200_ERR_CUDA, "dwdeconv: cannot raise the shared-memory limit to %zu bytes", smem);
      auto ilog2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return (1 << l) == v ? l : -1; };
      {
        const int lf = ilog2(op.stride), lcv = ilog2(op.cin[0] / VEC);
        const int CVv = op.cin[0] / VEC;
        if (lf >= 0 && lcv >= 0 && op.kh == 2 * op.stride && CVv <= 256 && (256 / CVv) % op.stride == 0 && getenv("CPB200_DWDECONV_GENERIC") == nullptr) {
          dwdeconv_add_fast_kernel<T, VEC><<<(unsigned)(op.B * op.Ho), 256, 0, st>>>(static_cast<const T *>(op.src[0]),
              static_cast<const T *>(op.aux), static_cast<T *>(op.dst), static_cast<const float *>(op.weight),
              op.H, op.W, op.cin[0], op.Ho, op.Wo, op.kh, op.stride, op.pad_h, lf, lcv);
          return cpb::check_launch("dwdeconv_add_fast_kernel");
        }
      }
      dwdeconv_add_kernel<T, VEC><<<(unsigned)(op.B * op.Ho), 256, smem, st>>>(static_cast<const T *>(op.src[0]),
          static_cast<const T *>(op.aux), static_cast<T *>(op.dst), static_cast<const float *>(op.weight),
          op.H, op.W, op.cin[0], op.Ho, op.Wo, op.kh, op.stride, op.pad_h, ilog2(op.stride), ilog2(op.cin[0] / VEC));
      return cpb::check_launch("dwdeconv_add_kernel");
    }
    case CPB200_OP_DWCONV: {
      constexpr int VEC = sizeof(T) == 2 ? 8 : 4;
      const int C = op.cin[0];
      if (C % VEC || op.kh != op.kw || op.cout != C) return cpb::fail(CPB200_ERR_ARG, "dwconv: C %% %d != 0 or non-square kernel", VEC);
#define DW_TILED(KK, SS, PX)                                                                                   \
  if (op.kh == KK && op.stride == SS && op.pad_h == KK / 2) {                                                    \
    const long long tot = (long long)op.B * op.Ho * ((op.Wo + PX - 1) / PX) * (C / VEC);                         \
    const unsigned g = (unsigned)std::min<long long>((tot + 255) / 256, 132LL * 32);                            \
    dwconv_tiled_kernel<T, VEC, KK, SS, PX><<<g, 256, 0, st>>>(static_cast<const T *>(op.src[0]),                \
        static_cast<T *>(op.dst), static_cast<const float *>(op.weight), op.bias, tot, op.H, op.W, C, op.Ho,     \
        op.Wo, op.flags & CPB_ACT_MASK);                                                                        \
    return cpb::check_launch("dwconv_tiled_kernel");                                                            \
  }
      DW_TILED(3, 1, 4) DW_TILED(5, 1, 4) DW_TILED(3, 2, 2) DW_TILED(5, 2, 2)
#undef DW_TILED
      const long long total = (long long)op.B * op.Ho * op.Wo * (C / VEC);
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 32);
      dwconv_kernel<T, VEC><<<grid, 256, 0, st>>>(static_cast<const T *>(op.src[0]), static_cast<T *>(op.dst),
          static_cast<const float *>(op.weight), op.bias, total, op.H, op.W, C, op.Ho, op.Wo, op.kh, op.stride, op.pad_h,
          op.flags & CPB_ACT_MASK);
      return cpb::check_launch("dwconv_kernel");
    }
    case CPB200_OP_AVGPOOL: {
      const int C = op.cin[0];
      if (C % 4 || op.Ho != 1 || op.Wo != 1) return cpb::fail(CPB200_ERR_ARG, "avgpool: C %% 4 != 0 or output not 1x1");
      avgpool_kernel<T><<<dim3((unsigned)op.B, (unsigned)((C + 63) / 64)), 256, 0, st>>>(static_cast<const T *>(op.src[0]),
          static_cast<T *>(op.dst), op.H * op.W, C);
      return cpb::check_launch("avgpool_kernel");
    }
    case CPB200_OP_SCALE_ADD: {
      const int C = op.cin[0];
      if (C % 4 || !op.res) return cpb::fail(CPB200_ERR_ARG, "scale_add: C %% 4 != 0 or missing scale vector");
      const long long per_image = (long long)op.H * op.W * (C / 4), total = per_image * op.B;
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 16);
      scale_add_kernel<T><<<grid, 256, 0, st>>>(static_cast<const T *>(op.src[0]), static_cast<const T *>(op.res),
          static_cast<const T *>(op.aux), static_cast<T *>(op.dst), total, per_image, C / 4);
      return cpb::check_launch("scale_add_kernel");
    }
    case CPB200_OP_UPSAMPLE_ADD: {
      const int f = op.stride;
      int sh = 0;
      while ((1 << sh) < f) ++sh;
      if (f < 1 || (1 << sh) != f || op.Ho != op.H * f || op.Wo != op.W * f || op.cin[0] % 4)
        return cpb::fail(CPB200_ERR_ARG, "upsample_add: factor %d must be a power of two, C %% 4 == 0", f);
      const long long total = (long long)op.B * op.Ho * op.Wo * (op.cin[0] / 4);
      const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 16);
      upsample_add_kernel<T><<<grid, 256, 0, st>>>(static_cast<const T *>(op.src[0]), static_cast<const T *>(op.aux),
          static_cast<T *>(op.dst), total, op.H, op.W, op.cin[0] / 4, op.Ho, op.Wo, sh, op.flags & CPB_ACT_MASK);
      return cpb::check_launch("upsample_add_kernel");
    }
    default: return cpb::fail(CPB200_ERR_ARG, "unknown op type %d", op.type);
  }
}

}  // namespace

namespace cpb {
int run_op_simt_dispatch(const cpb200_op &op, cudaStream_t st) {
  if (op.act_dtype == CPB200_BF16X2 || op.act_dtype == CPB200_F16X2) return run_op_split(op, st);
  if (op.type == CPB200_OP_CONVERT) return fail(CPB200_ERR_ARG, "convert: act_dtype must name a split layout");
  if (op.act_dtype == CPB200_F32) return run_op_simt<float>(op, st);
  if (op.act_dtype == CPB200_BF16) return run_op_simt<__nv_bfloat16>(op, st);
  return fail(CPB200_ERR_ARG, "bad act_dtype %d", op.act_dtype);
}
}  // namespace cpb

// The bandwidth-bound element-wise ops of the DLA-34 program, MAXPOOL and DWDECONV_ADD, on every activation format.
// They are their own translation unit so that NVVM's full -O3 pipeline compiles them: net_simt.cu, which holds the
// other element-wise ops, is built at -O1 (centerpose_b200/build.py).  Reference semantics per op: net_simt.cu.
#include "simt_io.cuh"
#include <algorithm>

namespace {

// ---- MAXPOOL k x k / stride / pad, NHWC (exact on split planes: the maximum is one of the inputs) ----
// Two forms in one kernel, chosen by pool2_fast from the op's shape alone (the host sizes the grid with the same test):
//   2x2 / stride 2 / pad 0 on even H and W with C % 8 == 0 (every pool of DLA-34): thread = VEC channels (16 bytes, per
//     plane on split tensors) of one output pixel, the four taps loaded before the first use; grid = (row chunks, Ho, B),
//     so the only division is a 32-bit one.  A row's items read 2 * C consecutive values per output pixel: coalesced.
//   anything else: 4 channels per thread, grid-stride loop over the output, bounds-tested k x k taps.
__host__ __device__ inline bool pool2_fast(int H, int W, int C, int k, int stride, int pad) {
  return k == 2 && stride == 2 && pad == 0 && !(H & 1) && !(W & 1) && C % 8 == 0;
}
__device__ __forceinline__ float4 max4(float4 a, float4 b) {
  return make_float4(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z), fmaxf(a.w, b.w));
}
__device__ __forceinline__ Vf<4> vmax(Vf<4> a, Vf<4> b) { return {max4(a.a, b.a)}; }
__device__ __forceinline__ Vf<8> vmax(Vf<8> a, Vf<8> b) { return {max4(a.a, b.a), max4(a.b, b.b)}; }
template <typename PI> constexpr int POOL2_VEC = std::is_same<PI, const float *>::value ? 4 : 8;   // 16 bytes per plane

template <typename PI, typename PO>
__global__ void __launch_bounds__(256, 4) maxpool_kernel(PI x, PO y, int B, int H, int W, int C, int Ho, int Wo, int k,
                                                         int stride, int pad) {
  if (pool2_fast(H, W, C, k, stride, pad)) {
    constexpr int VEC = POOL2_VEC<PI>;
    const int CV = C / VEC, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= Wo * CV) return;
    const int wo = i / CV, cv = i - wo * CV, ho = blockIdx.y, b = blockIdx.z;
    const PI p = x + ((((size_t)b * H + 2 * ho) * W + 2 * wo) * C + cv * VEC);
    const size_t row = (size_t)W * C;
    const Vf<VEC> t0 = io_ldv<VEC>(p), t1 = io_ldv<VEC>(p + C), t2 = io_ldv<VEC>(p + row), t3 = io_ldv<VEC>(p + (row + C));
    io_stv(y + (((size_t)b * Ho + ho) * Wo * C + (size_t)i * VEC), vmax(vmax(t0, t1), vmax(t2, t3)));
    return;
  }
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
        const float4 v = io_ld4(x + (((size_t)b * H + hi) * W + wi) * C + c4 * 4);
        m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
      }
    }
    io_st4(y + (((size_t)b * Ho + ho) * Wo + wo) * C + c4 * 4, m);
  }
}

// ---- depthwise ConvTranspose2d(k=2f, stride f, pad f/2) + skip add, NHWC ----
// out[b,ho,wo,c] = skip[b,ho,wo,c] + sum_{kh,kw : (ho+p-kh)%f==0, (wo+p-kw)%f==0} x[b,(ho+p-kh)/f,(wo+p-kw)/f,c] * w[kh,kw,c]
// With a bias (MobileNetV2 IDAUp: k 2, stride 2, pad 0, folded BN + ReLU, mobilenetv2.py:162-183) the sum starts from
// the bias, takes the activation, and the skip is added last: out = skip + act(bias + sum ...).
// One CTA = one output row (b, ho); thread = (wo, group of VEC channels).  The k*k*C filter taps are read through the
// read-only cache, so any filter size is accepted.  No integer division in the inner loop when f and C / VEC are powers
// of two (lf = log2 f, lcv = log2(C / VEC), or -1 -> generic division).
template <int VEC, typename PI, typename PO>
__global__ void __launch_bounds__(256) dwdeconv_add_kernel(PI x, PI skip, PO y, const float *__restrict__ w,
                                                           const float *__restrict__ bias, int H, int W, int C, int Ho, int Wo,
                                                           int k, int f, int pad, int lf, int lcv, uint32_t act) {
  const int CV = C / VEC;
  const int b = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  const int kh0 = (ho + pad) % f;
  const PI xb = x + (size_t)b * H * W * C;
  const bool fast = lf >= 0 && lcv >= 0;
  for (int i = threadIdx.x; i < Wo * CV; i += blockDim.x) {
    const int wo = fast ? (i >> lcv) : (i / CV), cv = i - wo * CV;
    const size_t opix = (((size_t)b * Ho + ho) * Wo + wo) * C + cv * VEC;
    Vf<VEC> acc = bias ? ld_taps<VEC>(bias + cv * VEC) : skip ? io_ldv<VEC>(skip + opix) : Vf<VEC>{};
    const int kw0 = fast ? ((wo + pad) & (f - 1)) : ((wo + pad) % f);
    for (int khh = kh0; khh < k; khh += f) {
      const int hn = ho + pad - khh;
      const int hi = fast ? (hn >> lf) : (hn / f);
      if (hn < 0 || hi >= H) continue;
      for (int kww = kw0; kww < k; kww += f) {
        const int wn = wo + pad - kww;
        const int wi = fast ? (wn >> lf) : (wn / f);
        if (wn < 0 || wi >= W) continue;
        acc = vfma(io_ldv<VEC>(xb + ((size_t)hi * W + wi) * C + cv * VEC), ld_taps<VEC>(w + (size_t)(khh * k + kww) * C + cv * VEC), acc);
      }
    }
    if (bias) {
      acc = vact<PO>(acc, act);
      if (skip) acc = vadd(acc, io_ldv<VEC>(skip + opix));
    }
    io_stv(y + opix, acc);
  }
}

// Fast path for the shapes IDAUp uses (see run_eltwise): every item a thread visits in one output row has the same
// channel group and the same column parity class, so its four (kh, kw) tap weight vectors are loaded ONCE per CTA.
// VEC channels = 16 bytes per plane.  4 CTAs per SM: the four tap vectors of 8 channels take 32 registers on their own, and
// at 6 CTAs (40 registers) the -O3 build spills them.
template <int VEC, typename PI, typename PO>
__global__ void __launch_bounds__(256, 4) dwdeconv_add_fast_kernel(PI x, PI skip, PO y, const float *__restrict__ w, int H, int W, int C,
                                                                int Ho, int Wo, int k, int f, int pad, int lf, int lcv) {
  const int CV = C / VEC;
  const int b = blockIdx.x / Ho, ho = blockIdx.x % Ho;
  const int i0 = threadIdx.x;
  const int wo_first = i0 >> lcv, cv = i0 & (CV - 1);
  const int kh0 = (ho + pad) & (f - 1), kw0 = (wo_first + pad) & (f - 1);
  Vf<VEC> wt[2][2];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 2; ++c) wt[a][c] = ld_taps<VEC>(w + (size_t)((kh0 + a * f) * k + kw0 + c * f) * C + cv * VEC);
  const PI xb = x + (size_t)b * H * W * C + cv * VEC;
  const int hn0 = ho + pad - kh0;                               // >= 0; tap a reads input row (hn0 >> lf) - a
  const int hi0 = hn0 >> lf;
  const size_t orow = ((size_t)b * Ho + ho) * Wo;
  for (int i = i0; i < Wo * CV; i += 256) {
    const int wo = i >> lcv;
    const size_t opix = (orow + wo) * C + cv * VEC;
    Vf<VEC> acc = skip ? io_ldv<VEC>(skip + opix) : Vf<VEC>{};
    const int wi0 = (wo + pad - kw0) >> lf;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int hi = hi0 - a;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int wi = wi0 - c;
        if (wi < 0 || wi >= W) continue;
        acc = vfma(io_ldv<VEC>(xb + ((size_t)hi * W + wi) * C), wt[a][c], acc);
      }
    }
    io_stv(y + opix, acc);
  }
}

// PI / PO and T as in net_simt.cu's run_eltwise.
template <typename T, typename PI, typename PO>
int run_pool_deconv(const cpb200_op &op, uint32_t fmt, cudaStream_t st) {
  constexpr int VEC = 16 / sizeof(T);                   // channels per thread: 16 bytes, or 8 bytes per split plane
  constexpr int VEC_FAST = std::is_same<PO, SpM>::value ? 8 : VEC;   // the fast dwdeconv: 16 bytes per plane
  const int C = op.cin[0];
  if (op.src_pitch[0] != 0 && op.src_pitch[0] != C)
    return cpb::fail(CPB200_ERR_ARG, "op type %d: needs a dense input (src_pitch %d, C %d)", op.type, op.src_pitch[0], C);
  const size_t n_in = (size_t)op.B * op.H * op.W * C, n_out = (size_t)op.B * op.Ho * op.Wo * C;
  const PI x = io_handle<PI>(op.src[0], n_in, fmt), skip = io_handle<PI>(op.aux, n_out, fmt);
  const PO y = io_handle<PO>(op.dst, n_out, fmt);
  const float *w = static_cast<const float *>(op.weight);
  const uint32_t act = op.flags & CPB_ACT_MASK;
  if (op.type == CPB200_OP_MAXPOOL) {
    if (C % 4) return cpb::fail(CPB200_ERR_ARG, "maxpool: C %% 4 != 0");
    // the 2x2 form takes one thread per item of a (row chunk, ho, b) grid; grid.y / .z hold 65535 at most
    const bool fast = pool2_fast(op.H, op.W, C, op.kh, op.stride, op.pad_h);
    if (fast && (op.Ho > 65535 || op.B > 65535)) return cpb::fail(CPB200_ERR_ARG, "maxpool 2x2: Ho and B must be <= 65535");
    const long long total = (long long)op.B * op.Ho * op.Wo * (C / 4);
    const dim3 g = fast ? dim3((unsigned)((op.Wo * (C / POOL2_VEC<PI>) + 255) / 256), (unsigned)op.Ho, (unsigned)op.B)
                        : dim3((unsigned)std::min<long long>((total + 255) / 256, 132LL * 32));
    maxpool_kernel<PI, PO><<<g, 256, 0, st>>>(x, y, op.B, op.H, op.W, C, op.Ho, op.Wo, op.kh, op.stride, op.pad_h);
    return cpb::check_launch("maxpool_kernel", maxpool_kernel<PI, PO>);
  }
  if (C % VEC || op.stride < 1) return cpb::fail(CPB200_ERR_ARG, "dwdeconv: needs C %% %d == 0 and stride >= 1", VEC);
  if (act && !op.bias) return cpb::fail(CPB200_ERR_ARG, "dwdeconv: an activation needs the bias form");
  const int lf = ilog2(op.stride), CV = C / VEC_FAST, lcv = C % VEC_FAST ? -1 : ilog2(CV);
  // the fast kernel's shapes: no bias, k == 2f, f and C / VEC_FAST powers of two, and each CTA's 256 threads cover
  // whole output pixels of one column parity class
  if (!op.bias && lf >= 0 && lcv >= 0 && op.kh == 2 * op.stride && CV <= 256 && (256 / CV) % op.stride == 0) {
    dwdeconv_add_fast_kernel<VEC_FAST, PI, PO><<<(unsigned)(op.B * op.Ho), 256, 0, st>>>(x, skip, y, w, op.H, op.W, C, op.Ho,
        op.Wo, op.kh, op.stride, op.pad_h, lf, lcv);
    return cpb::check_launch("dwdeconv_add_fast_kernel", dwdeconv_add_fast_kernel<VEC_FAST, PI, PO>);
  }
  dwdeconv_add_kernel<VEC, PI, PO><<<(unsigned)(op.B * op.Ho), 256, 0, st>>>(x, skip, y, w, op.bias, op.H, op.W, C, op.Ho,
      op.Wo, op.kh, op.stride, op.pad_h, lf, ilog2(C / VEC), act);
  return cpb::check_launch("dwdeconv_add_kernel", dwdeconv_add_kernel<VEC, PI, PO>);
}

}  // namespace

namespace cpb {
int run_op_pool_deconv(const cpb200_op &op, cudaStream_t st) {
  switch (op.act_dtype) {
    case CPB200_F32: return run_pool_deconv<float, const float *, float *>(op, 0, st);
    case CPB200_BF16: return run_pool_deconv<bf16, const bf16 *, bf16 *>(op, 0, st);
    case CPB200_BF16X2: return run_pool_deconv<float, SpC, SpM>(op, 0u, st);
    case CPB200_F16X2: return run_pool_deconv<float, SpC, SpM>(op, 1u, st);
    default: return fail(CPB200_ERR_ARG, "bad act_dtype %d", op.act_dtype);
  }
}
}  // namespace cpb

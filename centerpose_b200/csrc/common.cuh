// Shared host/device helpers for the centerpose_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/centerpose_b200.h"

namespace cpb {

extern thread_local char g_err[512];
extern std::atomic<unsigned long long> g_launches;

inline int fail(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

inline int check_launch(const char *what) {
  cudaError_t e = cudaGetLastError();
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (e != cudaSuccess) return fail(CPB200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return CPB200_OK;
}

// Route log (cpb200_route_log_start / _read): network-op launch sites pass their kernel, which is recorded while the
// log is on.  Off, the cost is one relaxed atomic load per launch.
void note_launch(const void *kernel);

template <typename K>
inline int check_launch(const char *what, K *kernel) {
  note_launch(reinterpret_cast<const void *>(kernel));
  return check_launch(what);
}

#define CPB_CUDA(call)                                                                 \
  do {                                                                                 \
    cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess)                                                             \
      return cpb::fail(CPB200_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_));      \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// cv2's ApplyExifOrientation as an index mapping: pixel (oy, ox) of the oriented image is stored pixel (sy, sx) of the
// h x w image (transpose for 5..8, then flips)
__device__ __forceinline__ void exif_source(int o, int oy, int ox, int h, int w, int &sy, int &sx) {
  switch (o) {
    case 2: sy = oy; sx = w - 1 - ox; break;
    case 3: sy = h - 1 - oy; sx = w - 1 - ox; break;
    case 4: sy = h - 1 - oy; sx = ox; break;
    case 5: sy = ox; sx = oy; break;
    case 6: sy = h - 1 - ox; sx = oy; break;
    case 7: sy = h - 1 - ox; sx = w - 1 - oy; break;
    case 8: sy = ox; sx = w - 1 - oy; break;
    default: sy = oy; sx = ox; break;
  }
}

// ---- cv2.resize INTER_LINEAR on 8-bit images, one output pixel ----
// Bit-exact with OpenCV's fixed-point linear resize (resize.cpp, resizeGeneric_ with HResizeLinear / VResizeLinear and
// the SIMD vertical pass): per output coordinate d, f = float((d + 0.5) * scale - 0.5) with scale = 1 / (out / in) in
// double, i = floor(f), f -= i, a0 = rint((1 - f) * 2048), a1 = 2048 - a0.  Columns clamp the coefficient at the
// border (i < 0 or i >= in - 1: i = clamp, f = 0); rows do not: the weights stay, each of the two source rows is
// clipped to [0, in - 1] on its own (this is what makes the first and last rows of an upscale differ from a clamped
// coefficient).  Horizontal pass exact in int32, h = s[i] * a0 + s[i + 1] * a1 (< 2^19); vertical pass as the 16-bit
// SIMD code does it, t = ((h0 >> 4) * b0 >> 16) + ((h1 >> 4) * b1 >> 16), out = (t + 2) >> 2.

// source index and 11-bit weight of the left / upper tap for output coordinate d; the float steps use explicit
// round-to-nearest intrinsics so nvcc cannot contract them into FMAs (the host computes them unfused)
__device__ __forceinline__ int resize_tap(int d, double scale, int &a0) {
  float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
  const float fi = floorf(f);
  f = __fsub_rn(f, fi);
  a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  return (int)fi;
}

// the 1 / (out / in) scale of one axis
__device__ __forceinline__ double resize_scale(int out, int in) { return __ddiv_rn(1.0, __ddiv_rn((double)out, (double)in)); }

// the two source columns (x0, x1), rows (y0, y1) and weights (a0, b0) of output pixel (x, y) when an h x w image is
// resized with scales (sx, sy)
struct LinearTaps {
  int x0, x1, y0, y1, a0, b0;
};

__device__ __forceinline__ LinearTaps linear_taps(int x, int y, int h, int w, double sx, double sy) {
  LinearTaps t;
  t.x0 = resize_tap(x, sx, t.a0);
  if (t.x0 < 0) { t.x0 = 0; t.a0 = 2048; }
  if (t.x0 >= w - 1) { t.x0 = w - 1; t.a0 = 2048; }
  t.x1 = min(t.x0 + 1, w - 1);
  const int yt = resize_tap(y, sy, t.b0);
  t.y0 = min(max(yt, 0), h - 1);
  t.y1 = min(max(yt + 1, 0), h - 1);
  return t;
}

// one channel of the output pixel from its four source values s<row><col> at (y0|y1, x0|x1)
__device__ __forceinline__ unsigned char linear_mix(int s00, int s01, int s10, int s11, const LinearTaps &t) {
  const int h0 = s00 * t.a0 + s01 * (2048 - t.a0);
  const int h1 = s10 * t.a0 + s11 * (2048 - t.a0);
  const int v = (((h0 >> 4) * t.b0) >> 16) + (((h1 >> 4) * (2048 - t.b0)) >> 16);
  return (unsigned char)min(max((v + 2) >> 2, 0), 255);
}

// ---- cv2.warpAffine INTER_LINEAR on 8-bit images, constant-0 border, one output pixel ----
// Bit-exact with OpenCV's imgwarp.cpp (WarpAffineInvoker + remapBilinear): the 2x3 matrix is inverted in double
// exactly as cv2 does, source coordinates are 10-bit fixed point (AB_SCALE = 1024, round_delta = 16) reduced to 5
// fractional bits, the four bilinear weights are the integers (32-fx)(32-fy)*32 ... that sum to 2^15, and the result
// is (sum + 2^14) >> 15.

// cv2::warpAffine without WARP_INVERSE_MAP inverts the forward matrix t like this, in double on the host; the explicit
// round-to-nearest operations keep nvcc from contracting them into FMAs, so the inverse m is the host's bit for bit
__device__ __forceinline__ void warp_inverse(const double *t, double *m) {
  double D = __dsub_rn(__dmul_rn(t[0], t[4]), __dmul_rn(t[1], t[3]));
  D = D != 0 ? __ddiv_rn(1.0, D) : 0;
  m[0] = __dmul_rn(t[4], D); m[4] = __dmul_rn(t[0], D); m[1] = __dmul_rn(t[1], -D); m[3] = __dmul_rn(t[3], -D);
  m[2] = __dsub_rn(__dmul_rn(-m[0], t[2]), __dmul_rn(m[1], t[5]));
  m[5] = __dsub_rn(__dmul_rn(-m[3], t[2]), __dmul_rn(m[4], t[5]));
}

// the three channels u[] of output pixel (x, y) of the h x w HWC image `img` warped by the inverse matrix m; with
// `mirror` the source is img[:, ::-1] (source column sx is stored column w - 1 - sx)
__device__ __forceinline__ void warp_linear_u8(const unsigned char *img, int h, int w, const double *m, int x, int y,
                                               bool mirror, int u[3]) {
  // cv2 rounds m1*y, then the sum: an FMA would round once and, where the sum lands on a half-unit of 1/1024, can
  // make llrint pick the other integer (tests/post_cases.py tie_x_row, tie_y_row)
  const long long adelta = llrint(__dmul_rn(__dmul_rn(m[0], (double)x), 1024.0));
  const long long bdelta = llrint(__dmul_rn(__dmul_rn(m[3], (double)x), 1024.0));
  const long long X0 = llrint(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)y), m[2]), 1024.0)) + 16;
  const long long Y0 = llrint(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)y), m[5]), 1024.0)) + 16;
  const long long X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5;
  long long sxl = X >> 5, syl = Y >> 5;
  sxl = sxl < -32768 ? -32768 : (sxl > 32767 ? 32767 : sxl);       // saturate_cast<short>
  syl = syl < -32768 ? -32768 : (syl > 32767 ? 32767 : syl);
  const int sx = (int)sxl, sy = (int)syl, fx = (int)(X & 31), fy = (int)(Y & 31);
  const int w0 = (32 - fx) * (32 - fy) * 32, w1 = fx * (32 - fy) * 32, w2 = (32 - fx) * fy * 32, w3 = fx * fy * 32;
  const bool y0 = sy >= 0 && sy < h, y1 = sy + 1 >= 0 && sy + 1 < h, x0 = sx >= 0 && sx < w, x1 = sx + 1 >= 0 && sx + 1 < w;
  const unsigned char *p00 = img + ((long long)sy * w + (mirror ? w - 1 - sx : sx)) * 3;
  const int dx = mirror ? -3 : 3;                                    // the next source column's byte step
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v00 = (y0 && x0) ? p00[c] : 0, v01 = (y0 && x1) ? p00[dx + c] : 0;
    const int v10 = (y1 && x0) ? p00[(size_t)w * 3 + c] : 0, v11 = (y1 && x1) ? p00[(size_t)w * 3 + dx + c] : 0;
    const int s = (v00 * w0 + v01 * w1 + v10 * w2 + v11 * w3 + (1 << 14)) >> 15;
    u[c] = s < 0 ? 0 : (s > 255 ? 255 : s);
  }
}

#define CPB_ACT_MASK (CPB200_FLAG_RELU | CPB200_FLAG_HSWISH | CPB200_FLAG_HSIGMOID | CPB200_FLAG_RELU6 | CPB200_FLAG_CLIP01)
// Epilogue non-linearity selected by the op flags (at most one of RELU / HSWISH / HSIGMOID / RELU6 / CLIP01).  hswish
// and hsigmoid keep the reference's operation order x * relu6(x + 3) / 6 (mobilenetv3.py:84-93).  ReLU6 and the hard
// [0, 1] clamp take the same clamp without the + 3 and the / 6: min(max(x, 0), 6 or 1).  Their result is exact in every
// format, so the split epilogues clamp before the hi / lo re-split and a clamped 6 or 1 has lo == 0.  After the ReLU and
// identity tests the code is straight-line (selects on the flag, no further branch), as it was for hswish / hsigmoid
// alone: the tensor-core epilogues inline it for every accumulator pair.
__device__ __forceinline__ float act_fn(float v, uint32_t act) {
  if (act == CPB200_FLAG_RELU) return fmaxf(v, 0.f);
  if (act == 0u) return v;
  const bool hs = act < CPB200_FLAG_RELU6;                     // HSWISH / HSIGMOID
  const float c = fminf(fmaxf(hs ? v + 3.f : v, 0.f), act == CPB200_FLAG_CLIP01 ? 1.f : 6.f);
  const float n = act == CPB200_FLAG_HSWISH ? v * c : c;
  return hs ? n / 6.f : c;
}
// bf16-output variant: multiply by 1/6 instead of the IEEE division (differs from act_fn by <= 1 ulp of fp32,
// far below the bf16 rounding that follows).  The division costs 20+ instructions per element, enough to make the
// MobileNetV3 expand convs and depthwise convs instruction-bound.
// the multiply-by-1/6 form on its own: used wherever the result is re-split into 16-bit planes (the split tensor-core
// epilogues and the element-wise kernels on planes; tools/prof_act.py times both forms); 1 ulp of fp32 is 2^-13 of the
// planes' own precision.
__device__ __forceinline__ float act_fast(float v, uint32_t act) {
  if (act == CPB200_FLAG_RELU) return fmaxf(v, 0.f);
  if (act == 0u) return v;
  const bool hs = act < CPB200_FLAG_RELU6;
  const float c = fminf(fmaxf(hs ? v + 3.f : v, 0.f), act == CPB200_FLAG_CLIP01 ? 1.f : 6.f);
  const float r = hs ? c * (1.f / 6.f) : c;
  return act == CPB200_FLAG_HSWISH ? v * r : r;
}
template <typename T>
__device__ __forceinline__ float act_out(float v, uint32_t act) {
  if constexpr (sizeof(T) == 4) return act_fn(v, act);
  else return act_fast(v, act);
}

}  // namespace cpb

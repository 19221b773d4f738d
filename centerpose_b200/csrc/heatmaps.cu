// The heat-map views of the reference's MultiPoseDetector.debug (lib/detectors/multi_pose.py:82-94 with
// lib/utils/debugger.py gen_colormap / gen_colormap_hp / add_blend_img), byte for byte: cpb200_heatmap_views_batch.
//
// Per image and view (0: pred_hm from hm with the hm colour, 1: pred_hmhp from the C keypoint maps):
//   colormap_kernel  cm = uint8(max_c(map[c] * colour[c])) on the h x w map grid        -> workspace
//   resize1_kernel   fore = cv2.resize(cm, (h * dr, w * dr)): w * dr rows of h * dr columns (transposed for a
//                    non-square map), then 255 - fore with the 'white' theme             -> workspace
//   blend_kernel     fore resized to (W, H) unless it already is, back = uint8(clip((x * std + mean) * 255, 0, 255))
//                    from the normalized input, out = uint8(clip(back * (1 - 0.7) + fore * 0.7, 0, 255)) in float64
// Every float step is an explicit round-to-nearest intrinsic, so nvcc cannot contract it into an FMA (numpy does not).
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_heatmap_image) == 64, "cpb200_heatmap_image layout is part of the C ABI");

constexpr int kThreads = 256;

struct ViewParams {
  float colors[1 + CPB200_HEATMAP_MAX_C][3];
  float mean[3], stdv[3];
  int white;
};

// numpy's float32 -> uint8 cast on x86-64: truncate to int32 (cvttss2si, which gives 0x80000000 for NaN and for
// |v| >= 2^31) and keep the low 8 bits, so -1.5 -> 255, 300.7 -> 44, NaN -> 0
__device__ __forceinline__ unsigned char numpy_u8(float v) {
  return (v > -2147483648.f && v < 2147483648.f) ? (unsigned char)__float2int_rz(v) : (unsigned char)0;
}

// workspace of one image: [cm view 0 | cm view 1] (h * w * 3 each), then [fore view 0 | fore view 1] (H * W * 3 each)
__device__ __forceinline__ unsigned char *cm_at(unsigned char *ws, const cpb200_heatmap_image &e, int view) {
  return ws + e.ws_offset + (int64_t)view * e.h * e.w * 3;
}
__device__ __forceinline__ unsigned char *fore_at(unsigned char *ws, const cpb200_heatmap_image &e, int view) {
  return ws + e.ws_offset + (int64_t)2 * e.h * e.w * 3 + (int64_t)view * e.H * e.W * 3;
}

// grid (pixel blocks, image, view); one thread per map pixel.  numpy's max propagates NaN, fmaxf would drop it.
__global__ void __launch_bounds__(kThreads) colormap_kernel(const cpb200_heatmap_image *__restrict__ table,
                                                           const ViewParams p, unsigned char *__restrict__ ws) {
  const cpb200_heatmap_image e = table[blockIdx.y];
  const int view = blockIdx.z;
  const float *maps = view ? e.hm_hp : e.hm;
  const int C = view ? e.C : 1, n = e.h * e.w;
  const float(*col)[3] = p.colors + (view ? 1 : 0);
  unsigned char *cm = cm_at(ws, e, view);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float m[3];
    for (int c = 0; c < C; ++c) {
      const float v = maps[(size_t)c * n + i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float q = __fmul_rn(v, col[c][k]);
        if (c == 0 || isnan(q) || (!isnan(m[k]) && q > m[k])) m[k] = q;
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) cm[(size_t)i * 3 + k] = numpy_u8(m[k]);
  }
}

// grid (pixel blocks, image, view); one thread per pixel of the w * dr x h * dr intermediate
__global__ void __launch_bounds__(kThreads) resize1_kernel(const cpb200_heatmap_image *__restrict__ table, int white,
                                                          unsigned char *__restrict__ ws) {
  const cpb200_heatmap_image e = table[blockIdx.y];
  const int view = blockIdx.z;
  const int rows = e.w * e.dr, cols = e.h * e.dr;
  const unsigned char *cm = cm_at(ws, e, view);
  unsigned char *fore = fore_at(ws, e, view);
  const double sx = cpb::resize_scale(cols, e.w), sy = cpb::resize_scale(rows, e.h);
  const int total = rows * cols;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const cpb::LinearTaps t = cpb::linear_taps(i % cols, i / cols, e.h, e.w, sx, sy);
    const unsigned char *r0 = cm + (size_t)t.y0 * e.w * 3, *r1 = cm + (size_t)t.y1 * e.w * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const unsigned char v = cpb::linear_mix(r0[t.x0 * 3 + k], r0[t.x1 * 3 + k], r1[t.x0 * 3 + k], r1[t.x1 * 3 + k], t);
      fore[(size_t)i * 3 + k] = white ? (unsigned char)(255 - v) : v;
    }
  }
}

// grid (pixel blocks, image, view); one thread per output pixel
__global__ void __launch_bounds__(kThreads) blend_kernel(const cpb200_heatmap_image *__restrict__ table,
                                                        const ViewParams p, const unsigned char *__restrict__ ws,
                                                        unsigned char *__restrict__ out) {
  const cpb200_heatmap_image e = table[blockIdx.y];
  const int view = blockIdx.z;
  const int rows = e.w * e.dr, cols = e.h * e.dr, total = e.H * e.W;
  const bool resize = rows != e.H || cols != e.W;
  const unsigned char *fore = fore_at(const_cast<unsigned char *>(ws), e, view);
  unsigned char *o = out + e.out_offset + (int64_t)view * total * 3;
  const double sx = cpb::resize_scale(e.W, cols), sy = cpb::resize_scale(e.H, rows);
  const double back_w = 1.0 - 0.7;                       // 0.30000000000000004, as Python computes 1. - trans
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    cpb::LinearTaps t;
    const unsigned char *r0 = fore, *r1 = fore;
    if (resize) {
      t = cpb::linear_taps(i % e.W, i / e.W, rows, cols, sx, sy);
      r0 = fore + (size_t)t.y0 * cols * 3;
      r1 = fore + (size_t)t.y1 * cols * 3;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int f = resize ? cpb::linear_mix(r0[t.x0 * 3 + k], r0[t.x1 * 3 + k], r1[t.x0 * 3 + k], r1[t.x1 * 3 + k], t)
                           : fore[(size_t)i * 3 + k];
      float b = __fmul_rn(__fadd_rn(__fmul_rn(e.input[(size_t)k * total + i], p.stdv[k]), p.mean[k]), 255.f);
      b = b < 0.f ? 0.f : (b > 255.f ? 255.f : b);       // NaN stays NaN, as np.clip leaves it
      const double v = __dadd_rn(__dmul_rn((double)numpy_u8(b), back_w), __dmul_rn((double)f, 0.7));
      o[(size_t)i * 3 + k] = (unsigned char)(int)(v > 255.0 ? 255.0 : v);
    }
  }
}

}  // namespace

extern "C" int cpb200_heatmap_views_batch(const cpb200_heatmap_image *table, int B, const float *colors,
                                          const float *mean, const float *stdv, int white, unsigned char *out,
                                          unsigned char *workspace, void *stream) {
  if (!table || !colors || !mean || !stdv || !out || !workspace || B < 1)
    return cpb::fail(CPB200_ERR_ARG, "heatmap_views_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "heatmap_views_batch: B = %d images exceed one launch (max 65535)", B);
  ViewParams p;
  for (int c = 0; c <= CPB200_HEATMAP_MAX_C; ++c)
    for (int k = 0; k < 3; ++k) p.colors[c][k] = colors[c * 3 + k];
  for (int k = 0; k < 3; ++k) { p.mean[k] = mean[k]; p.stdv[k] = stdv[k]; }
  p.white = white ? 1 : 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // the sizes live on the device: enough blocks per view to fill the GPU for one large image, fewer as B grows
  const dim3 grid((unsigned)std::max(1, 132 * 4 / B), (unsigned)B, 2);
  colormap_kernel<<<grid, kThreads, 0, s>>>(table, p, workspace);
  if (int st = cpb::check_launch("heatmap colormap_kernel")) return st;
  resize1_kernel<<<grid, kThreads, 0, s>>>(table, p.white, workspace);
  if (int st = cpb::check_launch("heatmap resize1_kernel")) return st;
  blend_kernel<<<grid, kThreads, 0, s>>>(table, p, workspace, out);
  return cpb::check_launch("heatmap blend_kernel");
}

// Device versions of two host-side steps around the decode (SURVEY.md §8 "next" rows 2 and 3):
//   cpb200_flip_merge   flip-test averaging of the head maps  (lib/detectors/multi_pose.py:45-53 with
//                       flip_tensor / flip_lr / flip_lr_off of lib/models/utils.py:27-47) in ONE pass,
//   cpb200_soft_nms_39  the pose soft-NMS of lib/external/nms.pyx:172-275 on a device array (_batch: one CTA per image),
// and the warp / normalise part of pre_process (cpb200_pre_process, _batch: one launch for many images).
#include "common.cuh"

namespace {

struct FlipArgs {
  const float *hm, *wh, *hps, *hm_hp;
  float *o_hm, *o_wh, *o_hps, *o_hm_hp;
  int P, H, W, J, CH;               // CH = classes of hm
  signed char perm[64];             // joint j of the flipped image is averaged into joint perm[j]'s partner: src joint
};

// One thread per output element of the concatenated (hm | wh | hps | hm_hp) channel stack of image pair p.
// out = (a[2p] + flipped(a[2p+1])) / 2 where `flipped` reverses W, swaps left/right joints (hps, hm_hp) and negates
// the x component of the keypoint offsets (hps even channels).  Same fp32 operation order as the reference.
__global__ void __launch_bounds__(256) flip_merge_kernel(const FlipArgs a) {
  const int HW = a.H * a.W;
  const int c_hm = a.CH, c_wh = 2, c_hps = 2 * a.J, c_hp = a.hm_hp ? a.J : 0;
  const int C = c_hm + c_wh + c_hps + c_hp;
  const long long total = (long long)a.P * C * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % a.W);
    const int y = (int)((i / a.W) % a.H);
    int c = (int)((i / HW) % C);
    const int p = (int)(i / ((long long)HW * C));
    const float *src; float *dst; int ct, cs; float sgn = 1.f;
    if (c < c_hm) { src = a.hm; dst = a.o_hm; ct = c_hm; cs = c; }
    else if ((c -= c_hm) < c_wh) { src = a.wh; dst = a.o_wh; ct = c_wh; cs = c; }
    else if ((c -= c_wh) < c_hps) {
      src = a.hps; dst = a.o_hps; ct = c_hps;
      const int j = c >> 1, d = c & 1;
      cs = 2 * a.perm[j] + d;
      if (d == 0) sgn = -1.f;
    } else { c -= c_hps; src = a.hm_hp; dst = a.o_hm_hp; ct = c_hp; cs = a.perm[c]; }
    const float v0 = src[(((size_t)(2 * p) * ct + c) * a.H + y) * a.W + x];
    const float v1 = src[(((size_t)(2 * p + 1) * ct + cs) * a.H + y) * a.W + (a.W - 1 - x)];
    dst[(((size_t)p * ct + c) * a.H + y) * a.W + x] = (v0 + sgn * v1) / 2.f;
  }
}

// ---- soft_nms_39: one CTA, the (N,56) rows live in shared memory while the sequential outer loop runs ----
// Per outer step i: (1) first arg-max of the scores in [i,N) (block reduction), (2) swap columns 0..38 of rows i and
// maxpos, (3) every row in (i,N) decays its own score against box i IN PARALLEL — the decay of a row depends only on
// box i and the row itself, and the sequential reference decays each live row exactly once per step wherever it has
// been moved to — (4) one thread replays the reference's swap-with-last removal walk on the decayed scores.
constexpr int NMS_T = 128;
constexpr int NMS_COLS = 56, NMS_MOVE = 39;

// One CTA per image: CTA b works on the (N0, 56) rows at boxes + b * N0 * 56 and writes keep_count[b].
__global__ void __launch_bounds__(NMS_T) soft_nms_kernel(float *boxes, int N0, float sigma, float Nt, float threshold, int method,
                                                         int *keep_count) {
  boxes += (size_t)blockIdx.x * N0 * NMS_COLS;
  extern __shared__ float sb[];                       // N0 x 56, then N0 pre-decay scores
  float *s_orig = sb + N0 * NMS_COLS;
  float *s_hit = s_orig + N0;                         // 1.0 when the row overlapped box i in this step (only those are
                                                      // tested against `threshold`, nms.pyx:236-268)
  __shared__ float s_val[NMS_T / 32];
  __shared__ int s_idx[NMS_T / 32];
  __shared__ int s_n, s_maxpos;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < N0 * NMS_COLS; i += NMS_T) sb[i] = boxes[i];
  if (tid == 0) s_n = N0;
  __syncthreads();
  for (int i = 0; i < N0; ++i) {
    const int N = s_n;
    if (i >= N) break;
    // (1) first maximum of sb[pos][4], pos in [i, N)  (the reference scans with a strict '<')
    float bv = -INFINITY; int bi = 0x7fffffff;
    for (int pos = i + tid; pos < N; pos += NMS_T) {
      const float v = sb[pos * NMS_COLS + 4];
      if (v > bv) { bv = v; bi = pos; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_val[wid] = bv; s_idx[wid] = bi; }
    __syncthreads();
    if (tid == 0) {
      float v = s_val[0]; int ix = s_idx[0];
      for (int w = 1; w < NMS_T / 32; ++w)
        if (s_val[w] > v || (s_val[w] == v && s_idx[w] < ix)) { v = s_val[w]; ix = s_idx[w]; }
      // a NaN-free input always yields ix in [i,N); the reference starts from maxpos = i
      s_maxpos = (ix == 0x7fffffff) ? i : ix;
    }
    __syncthreads();
    const int maxpos = s_maxpos;
    // (2) swap columns 0..38
    if (maxpos != i && tid < NMS_MOVE) {
      const float t = sb[i * NMS_COLS + tid];
      sb[i * NMS_COLS + tid] = sb[maxpos * NMS_COLS + tid];
      sb[maxpos * NMS_COLS + tid] = t;
    }
    __syncthreads();
    // (3) parallel decay against box i   (all arithmetic in float, as the port in centerpose_b200/soft_nms.py)
    const float tx1 = sb[i * NMS_COLS], ty1 = sb[i * NMS_COLS + 1], tx2 = sb[i * NMS_COLS + 2], ty2 = sb[i * NMS_COLS + 3];
    for (int pos = i + 1 + tid; pos < N; pos += NMS_T) {
      float *r = sb + pos * NMS_COLS;
      s_orig[pos] = r[4];
      s_hit[pos] = 0.f;
      const float x1 = r[0], y1 = r[1], x2 = r[2], y2 = r[3];
      const float area = __fmul_rn(__fadd_rn(__fsub_rn(x2, x1), 1.f), __fadd_rn(__fsub_rn(y2, y1), 1.f));
      const float iw = __fadd_rn(__fsub_rn(fminf(tx2, x2), fmaxf(tx1, x1)), 1.f);
      if (iw > 0.f) {
        const float ih = __fadd_rn(__fsub_rn(fminf(ty2, y2), fmaxf(ty1, y1)), 1.f);
        if (ih > 0.f) {
          const float tarea = __fmul_rn(__fadd_rn(__fsub_rn(tx2, tx1), 1.f), __fadd_rn(__fsub_rn(ty2, ty1), 1.f));
          const float inter = __fmul_rn(iw, ih);
          const float ua = __fsub_rn(__fadd_rn(tarea, area), inter);
          const float ov = __fdiv_rn(inter, ua);
          float weight;
          if (method == 1) weight = ov > Nt ? __fsub_rn(1.f, ov) : 1.f;
          else if (method == 2) weight = (float)exp((double)__fdiv_rn(-__fmul_rn(ov, ov), sigma));
          else weight = ov > Nt ? 0.f : 1.f;
          r[4] = __fmul_rn(weight, r[4]);
          s_hit[pos] = 1.f;
        }
      }
    }
    __syncthreads();
    // (4) the reference's removal walk (swap-with-last) over the rows that overlapped box i, sequential
    if (tid == 0) {
      int n = N, pos = i + 1;
      while (pos < n) {
        if (s_hit[pos] != 0.f && sb[pos * NMS_COLS + 4] < threshold) {
          float *r = sb + pos * NMS_COLS, *l = sb + (n - 1) * NMS_COLS;
          for (int c = 0; c < 5; ++c) r[c] = l[c];
          for (int c = 5; c < NMS_MOVE; ++c) { const float t = r[c]; r[c] = l[c]; l[c] = t; }
          // the reference decays a row only when its walk reaches it: the copy left behind at the tail was never
          // visited, so it keeps the pre-decay score (the live copy at `pos` carries the decayed one)
          if (l != r) l[4] = s_orig[n - 1];
          s_hit[pos] = s_hit[n - 1];
          --n;                                         // re-examine the row that moved in (already decayed)
        } else {
          ++pos;
        }
      }
      s_n = n;
    }
    __syncthreads();
  }
  for (int i = tid; i < N0 * NMS_COLS; i += NMS_T) boxes[i] = sb[i];
  if (tid == 0 && keep_count) keep_count[blockIdx.x] = s_n;
}

int soft_nms_launch(float *boxes, int B, int N, float sigma, float Nt, float threshold, int method, int *keep_counts,
                    void *stream, const char *what) {
  if (B < 0 || N < 0 || (!boxes && B > 0 && N > 0)) return cpb::fail(CPB200_ERR_ARG, "%s: bad arguments", what);
  if (B == 0) return CPB200_OK;
  if (N == 0) {
    if (keep_counts) CPB_CUDA(cudaMemsetAsync(keep_counts, 0, (size_t)B * sizeof(int), static_cast<cudaStream_t>(stream)));
    return CPB200_OK;
  }
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "%s: B = %d images exceed one launch (max 65535)", what, B);
  const size_t smem = (size_t)N * (NMS_COLS + 2) * sizeof(float);
  if (smem > 200 * 1024) return cpb::fail(CPB200_ERR_ARG, "%s: N = %d rows do not fit shared memory (max 882)", what, N);
  if (smem > 48 * 1024) CPB_CUDA(cudaFuncSetAttribute(soft_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  soft_nms_kernel<<<B, NMS_T, smem, static_cast<cudaStream_t>(stream)>>>(boxes, N, sigma, Nt, threshold, method, keep_counts);
  return cpb::check_launch("soft_nms_kernel");
}

}  // namespace

extern "C" int cpb200_flip_merge(const float *hm, const float *wh, const float *hps, const float *hm_hp, float *o_hm, float *o_wh,
                                 float *o_hps, float *o_hm_hp, int P, int H, int W, int J, int num_classes, const int *flip_perm,
                                 void *stream) {
  if (!hm || !wh || !hps || !o_hm || !o_wh || !o_hps || (hm_hp && !o_hm_hp) || !flip_perm)
    return cpb::fail(CPB200_ERR_ARG, "flip_merge: null pointer");
  if (P <= 0 || H <= 0 || W <= 0 || J <= 0 || J > 64 || num_classes <= 0) return cpb::fail(CPB200_ERR_ARG, "flip_merge: bad shape");
  FlipArgs a;
  a.hm = hm; a.wh = wh; a.hps = hps; a.hm_hp = hm_hp; a.o_hm = o_hm; a.o_wh = o_wh; a.o_hps = o_hps; a.o_hm_hp = o_hm_hp;
  a.P = P; a.H = H; a.W = W; a.J = J; a.CH = num_classes;
  for (int j = 0; j < J; ++j) {
    if (flip_perm[j] < 0 || flip_perm[j] >= J) return cpb::fail(CPB200_ERR_ARG, "flip_merge: flip_perm[%d] out of range", j);
    a.perm[j] = (signed char)flip_perm[j];
  }
  const long long total = (long long)P * (num_classes + 2 + 2 * J + (hm_hp ? J : 0)) * H * W;
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, 132LL * 16);
  flip_merge_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return cpb::check_launch("flip_merge_kernel");
}

extern "C" int cpb200_soft_nms_39(float *boxes, int N, float sigma, float Nt, float threshold, int method, int *keep_count,
                                  void *stream) {
  return soft_nms_launch(boxes, 1, N, sigma, Nt, threshold, method, keep_count, stream, "soft_nms_39");
}

extern "C" int cpb200_soft_nms_39_batch(float *boxes, int B, int N, float sigma, float Nt, float threshold, int method,
                                        int *keep_counts, void *stream) {
  return soft_nms_launch(boxes, B, N, sigma, Nt, threshold, method, keep_counts, stream, "soft_nms_39_batch");
}

// ---- device pre_process: warpAffine (bilinear, constant-0 border) + normalise + HWC->CHW (+ mirrored copy) ----
// Replaces the cv2.warpAffine / numpy part of BaseDetector.pre_process (lib/detectors/base_detector.py:44-55).
// Bit-exact with cv2.warpAffine(flags=INTER_LINEAR) on 8-bit images (OpenCV imgwarp.cpp, WarpAffineInvoker +
// remapBilinear): the 2x3 matrix is inverted in double exactly as cv2 does, source coordinates are 10-bit fixed
// point (AB_SCALE = 1024, round_delta = 16) reduced to 5 fractional bits, the four bilinear weights are the
// integers (32-fx)(32-fy)*32 ... that sum to 2^15, result = (sum + 2^14) >> 15; then ((u/255 - mean)/std) is
// evaluated in double and rounded to float like numpy does for `(inp / 255. - mean) / std`.astype(float32).
namespace {

static_assert(sizeof(cpb200_pre_image) == 64, "cpb200_pre_image layout is part of the C ABI");

struct PreArgs {
  const unsigned char *imgs;       // packed (h, w, 3) uint8 images
  const cpb200_pre_image *table;   // B entries on the device, or NULL: `one` describes the only image
  cpb200_pre_image one;
  float *out;                      // (B or 2B, 3, OH, OW) fp32
  int OH, OW, flip;
  float mean[3], stdv[3];
};

// grid (pixel blocks, image): blockIdx.y selects the image, its forward matrix is inverted by every thread
__global__ void __launch_bounds__(256) pre_process_kernel(const PreArgs a) {
  const int b = blockIdx.y;
  long long off; int h, w; double t[6];
  if (a.table) {
    const cpb200_pre_image *p = a.table + b;
    off = p->offset; h = p->h; w = p->w;
#pragma unroll
    for (int k = 0; k < 6; ++k) t[k] = p->trans_input[k];
  } else {
    off = a.one.offset; h = a.one.h; w = a.one.w;
#pragma unroll
    for (int k = 0; k < 6; ++k) t[k] = a.one.trans_input[k];
  }
  // cv2::warpAffine without WARP_INVERSE_MAP inverts the matrix like this (imgwarp.cpp), in double on the host; the
  // explicit round-to-nearest operations keep nvcc from contracting them into FMAs, so the inverse is the host's bit for bit
  double D = __dsub_rn(__dmul_rn(t[0], t[4]), __dmul_rn(t[1], t[3]));
  D = D != 0 ? __ddiv_rn(1.0, D) : 0;
  const double m0 = __dmul_rn(t[4], D), m4 = __dmul_rn(t[0], D), m1 = __dmul_rn(t[1], -D), m3 = __dmul_rn(t[3], -D);
  const double m2 = __dsub_rn(__dmul_rn(-m0, t[2]), __dmul_rn(m1, t[5]));
  const double m5 = __dsub_rn(__dmul_rn(-m3, t[2]), __dmul_rn(m4, t[5]));
  const unsigned char *img = a.imgs + off;
  float *out = a.out + (size_t)(a.flip ? 2 * b : b) * 3 * a.OH * a.OW;
  const int total = a.OH * a.OW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int x = i % a.OW, y = i / a.OW;
    const long long adelta = llrint(m0 * (double)x * 1024.0), bdelta = llrint(m3 * (double)x * 1024.0);
    const long long X0 = llrint((m1 * (double)y + m2) * 1024.0) + 16, Y0 = llrint((m4 * (double)y + m5) * 1024.0) + 16;
    const long long X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5;
    long long sxl = X >> 5, syl = Y >> 5;
    sxl = sxl < -32768 ? -32768 : (sxl > 32767 ? 32767 : sxl);       // saturate_cast<short>
    syl = syl < -32768 ? -32768 : (syl > 32767 ? 32767 : syl);
    const int sx = (int)sxl, sy = (int)syl, fx = (int)(X & 31), fy = (int)(Y & 31);
    const int w0 = (32 - fx) * (32 - fy) * 32, w1 = fx * (32 - fy) * 32, w2 = (32 - fx) * fy * 32, w3 = fx * fy * 32;
    const bool y0 = sy >= 0 && sy < h, y1 = sy + 1 >= 0 && sy + 1 < h, x0 = sx >= 0 && sx < w, x1 = sx + 1 >= 0 && sx + 1 < w;
    const unsigned char *p00 = img + ((long long)sy * w + sx) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int v00 = (y0 && x0) ? p00[c] : 0, v01 = (y0 && x1) ? p00[3 + c] : 0;
      const int v10 = (y1 && x0) ? p00[(size_t)w * 3 + c] : 0, v11 = (y1 && x1) ? p00[(size_t)w * 3 + 3 + c] : 0;
      int u = (v00 * w0 + v01 * w1 + v10 * w2 + v11 * w3 + (1 << 14)) >> 15;
      u = u < 0 ? 0 : (u > 255 ? 255 : u);
      const float f = (float)(((double)u / 255.0 - (double)a.mean[c]) / (double)a.stdv[c]);
      out[((size_t)c * a.OH + y) * a.OW + x] = f;
      if (a.flip) out[((size_t)(3 + c) * a.OH + y) * a.OW + (a.OW - 1 - x)] = f;
    }
  }
}

int pre_process_launch(PreArgs &a, int B, const float *mean, const float *stdv, void *stream) {
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  const dim3 grid((unsigned)((a.OH * a.OW + 255) / 256), (unsigned)B);
  pre_process_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a);
  return cpb::check_launch("pre_process_kernel");
}

}  // namespace

extern "C" int cpb200_pre_process(const unsigned char *img, int h, int w, const double *trans_input, float *out, int out_h, int out_w,
                                  const float *mean, const float *stdv, int flip, void *stream) {
  if (!img || !trans_input || !out || !mean || !stdv || h <= 0 || w <= 0 || out_h <= 0 || out_w <= 0)
    return cpb::fail(CPB200_ERR_ARG, "pre_process: bad arguments");
  PreArgs a = {};
  a.imgs = img; a.table = nullptr; a.out = out; a.OH = out_h; a.OW = out_w; a.flip = flip ? 1 : 0;
  a.one.offset = 0; a.one.h = h; a.one.w = w;
  for (int i = 0; i < 6; ++i) a.one.trans_input[i] = trans_input[i];
  return pre_process_launch(a, 1, mean, stdv, stream);
}

extern "C" int cpb200_pre_process_batch(const unsigned char *imgs, const cpb200_pre_image *table, int B, float *out, int out_h,
                                        int out_w, const float *mean, const float *stdv, int flip, void *stream) {
  if (!imgs || !table || !out || !mean || !stdv || B <= 0 || out_h <= 0 || out_w <= 0)
    return cpb::fail(CPB200_ERR_ARG, "pre_process_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "pre_process_batch: B = %d images exceed one launch (max 65535)", B);
  if ((long long)out_h * out_w > (1LL << 30)) return cpb::fail(CPB200_ERR_ARG, "pre_process_batch: output too large");
  PreArgs a = {};
  a.imgs = imgs; a.table = table; a.out = out; a.OH = out_h; a.OW = out_w; a.flip = flip ? 1 : 0;
  return pre_process_launch(a, B, mean, stdv, stream);
}

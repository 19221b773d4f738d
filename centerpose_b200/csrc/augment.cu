// The training split's network input (MultiPoseDataset.__getitem__, lib/datasets/multi_pose.py, split 'train') for
// many images at once, bit for bit (cpb200_train_augment_batch).  The host draws each image's random parameters and
// builds its matrices; three kernels apply them:
//
//   train_warp_kernel   one thread per output pixel: cv2.warpAffine of img or img[:, ::-1] (cpb::warp_linear_u8, the
//                       pre-process warp), into the workspace as uint8, and color_aug's grey plane,
//                       cv2.cvtColor(inp / 255, BGR2GRAY) as cv2's SIMD path rounds it
//   train_mean_kernel   one CTA per image: gs.mean(), numpy's pairwise float32 sum over the S*S grey values in the
//                       host's summation tree, divided by S*S
//   train_color_kernel  one thread per output pixel: / 255, brightness / contrast / saturation in the image's order,
//                       lighting, (x - mean) / std, HWC -> CHW
//
// Every float32 step is written with a round-to-nearest intrinsic and the file is built with -fmad=false: numpy
// rounds each in-place operation of color_aug on its own.
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_train_image) == 240, "cpb200_train_image layout is part of the C ABI");

constexpr int kMeanThreads = 512;
constexpr int kMaxS = 768;            // the mean kernel's tree fits shared memory

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

struct Workspace {
  unsigned char *warped;            // (B, S, S, 3) uint8
  float *grey;                      // (B, S, S)
  float *means;                     // (B)
};

Workspace carve(void *ws, int B, int S) {
  const size_t plane = (size_t)S * S;
  unsigned char *p = static_cast<unsigned char *>(ws);
  Workspace w;
  w.warped = p;
  p += align256((size_t)B * plane * 3);
  w.grey = reinterpret_cast<float *>(p);
  p += align256(sizeof(float) * B * plane);
  w.means = reinterpret_cast<float *>(p);
  return w;
}

// cv2.cvtColor(float32 BGR, COLOR_BGR2GRAY): R * 0.299 + (B * 0.114 + G * 0.587) with two FMAs, as cv2's SIMD loop
// evaluates it (S * S is a multiple of 16, so no pixel takes its scalar tail)
__device__ __forceinline__ float grey_of(float b, float g, float r) {
  return __fmaf_rn(r, 0.299f, __fmaf_rn(b, 0.114f, __fmul_rn(g, 0.587f)));
}

// grid (pixel blocks, image)
__global__ void __launch_bounds__(256) train_warp_kernel(const unsigned char *imgs, const cpb200_train_image *table,
                                                         int S, Workspace ws) {
  const int b = blockIdx.y;
  const cpb200_train_image &e = table[b];
  const int h = e.h, w = e.w, mirror = e.flip, color = e.color;
  double t[6], m[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) t[k] = e.trans_input[k];
  cpb::warp_inverse(t, m);
  const unsigned char *img = imgs + e.offset;
  const size_t plane = (size_t)S * S;
  unsigned char *wo = ws.warped + (size_t)b * plane * 3;
  float *go = ws.grey + (size_t)b * plane;
  const int total = S * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int u[3];
    cpb::warp_linear_u8(img, h, w, m, i % S, i / S, mirror != 0, u);
    wo[(size_t)i * 3] = (unsigned char)u[0];
    wo[(size_t)i * 3 + 1] = (unsigned char)u[1];
    wo[(size_t)i * 3 + 2] = (unsigned char)u[2];
    if (color)
      go[i] = grey_of(__fdiv_rn((float)u[0], 255.f), __fdiv_rn((float)u[1], 255.f), __fdiv_rn((float)u[2], 255.f));
  }
}

// numpy's pairwise_sum for float32 (loops_utils.h): a leaf of n <= 128 values keeps 8 running partials r[j] over
// a[j], a[j + 8], ... and returns ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)); larger ranges split at
// n / 2 - (n / 2) % 8 and add the halves.  Every leaf here holds a multiple of 8 values (the plan's promise), so no
// leaf has a scalar tail.  Eight lanes sum one leaf: lane j keeps r[j], and the three xor shuffles add the partials
// in the tree above (float addition is commutative, so each lane's pair sum is the same number).
__global__ void __launch_bounds__(kMeanThreads) train_mean_kernel(const cpb200_train_image *table, const int32_t *plan,
                                                                  int S, Workspace ws) {
  const int b = blockIdx.x;
  if (!table[b].color) return;
  extern __shared__ float slot[];
  const int L = plan[0], D = plan[1];
  const int32_t *begin = plan + 2, *level = begin + L + 1, *node = level + D + 1;
  const float *g = ws.grey + (size_t)b * S * S;
  const int lane8 = threadIdx.x & 7;
  for (int base = 0; base < L; base += kMeanThreads / 8) {          // the trip count is uniform across the CTA
    const int leaf = base + (int)(threadIdx.x >> 3);
    float r = 0.f;
    if (leaf < L) {
      const int lo = begin[leaf], hi = begin[leaf + 1];
      r = g[lo + lane8];
      for (int i = lo + 8 + lane8; i < hi; i += 8) r = __fadd_rn(r, g[i]);
    }
    r = __fadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 1));
    r = __fadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 2));
    r = __fadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 4));
    if (leaf < L && lane8 == 0) slot[leaf] = r;
  }
  __syncthreads();
  for (int d = 0; d < D; ++d) {                                     // the nodes of one level depend on earlier ones only
    for (int k = level[d] + (int)threadIdx.x; k < level[d + 1]; k += kMeanThreads)
      slot[L + k] = __fadd_rn(slot[node[2 * k]], slot[node[2 * k + 1]]);
    __syncthreads();
  }
  if (threadIdx.x == 0) ws.means[b] = __fdiv_rn(slot[D > 0 ? L + level[D] - 1 : 0], (float)(S * S));
}

struct ColorArgs {
  const cpb200_train_image *table;
  Workspace ws;
  float *out;
  int S;
  float mean[3], stdv[3];
};

// grid (pixel blocks, image)
__global__ void __launch_bounds__(256) train_color_kernel(const ColorArgs a) {
  const int b = blockIdx.y, S = a.S;
  const cpb200_train_image &e = a.table[b];
  const int color = e.color;
  int order[3];
  float alpha[3], beta[3];
  double light[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { order[k] = e.order[k]; alpha[k] = e.alpha[k]; beta[k] = e.beta[k]; light[k] = e.light[k]; }
  const size_t plane = (size_t)S * S;
  const unsigned char *wi = a.ws.warped + (size_t)b * plane * 3;
  const float *gi = a.ws.grey + (size_t)b * plane;
  const float gm = color ? a.ws.means[b] : 0.f;
  float *out = a.out + (size_t)b * 3 * plane;
  const int total = S * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    float x[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) x[c] = __fdiv_rn((float)wi[(size_t)i * 3 + c], 255.f);
    if (color) {
      const float gs = gi[i];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        // brightness_: image *= alpha; contrast_ and saturation_ (blend_): image *= alpha, then += image2 * (1 - alpha)
        // with image2 the grey mean (a float32 scalar) or the pixel's grey value
        const float add = order[k] == 1 ? __fmul_rn(gm, beta[k]) : __fmul_rn(gs, beta[k]);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          x[c] = __fmul_rn(x[c], alpha[k]);
          if (order[k] != 0) x[c] = __fadd_rn(x[c], add);
        }
      }
      // lighting_: image += a float64 vector, so each channel is added in double and rounded back
#pragma unroll
      for (int c = 0; c < 3; ++c) x[c] = (float)__dadd_rn((double)x[c], light[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * plane + i] = __fdiv_rn(__fsub_rn(x[c], a.mean[c]), a.stdv[c]);
  }
}

}  // namespace

extern "C" size_t cpb200_train_augment_workspace_bytes(int B, int S) {
  if (B < 1 || S < 1) return 0;
  const size_t plane = (size_t)S * S;
  return align256((size_t)B * plane * 3) + align256(sizeof(float) * B * plane) + sizeof(float) * B;
}

extern "C" int cpb200_train_augment_batch(const unsigned char *imgs, const cpb200_train_image *table, int B, int S,
                                          const int32_t *plan, const float *mean, const float *stdv, float *out,
                                          void *workspace, size_t workspace_bytes, void *stream) {
  if (!imgs || !table || !plan || !mean || !stdv || !out || !workspace || B < 1 || S < 4)
    return cpb::fail(CPB200_ERR_ARG, "train_augment_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "train_augment_batch: B = %d images exceed one launch", B);
  if (S % 4 != 0 || S > kMaxS)
    return cpb::fail(CPB200_ERR_ARG, "train_augment_batch: S = %d must be a multiple of 4 and at most %d", S, kMaxS);
  if (workspace_bytes < cpb200_train_augment_workspace_bytes(B, S))
    return cpb::fail(CPB200_ERR_ARG, "train_augment_batch: workspace of %zu bytes, %zu needed", workspace_bytes,
                     cpb200_train_augment_workspace_bytes(B, S));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const Workspace ws = carve(workspace, B, S);
  const dim3 grid((unsigned)((S * S + 255) / 256), (unsigned)B);
  train_warp_kernel<<<grid, 256, 0, s>>>(imgs, table, S, ws);
  if (int st = cpb::check_launch("train_warp_kernel")) return st;
  // the tree over n values has at most n / 64 leaves (each holds at least 64 values) and one node less inside
  const size_t smem = sizeof(float) * 2 * ((size_t)S * S / 32);
  if (smem > 48 * 1024)
    CPB_CUDA(cudaFuncSetAttribute(train_mean_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  train_mean_kernel<<<(unsigned)B, kMeanThreads, smem, s>>>(table, plan, S, ws);
  if (int st = cpb::check_launch("train_mean_kernel")) return st;
  ColorArgs a = {table, ws, out, S, {}, {}};
  for (int c = 0; c < 3; ++c) { a.mean[c] = mean[c]; a.stdv[c] = stdv[c]; }
  train_color_kernel<<<grid, 256, 0, s>>>(a);
  return cpb::check_launch("train_color_kernel");
}

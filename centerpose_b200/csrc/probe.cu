// Hardware probes (diagnostics, not on the product path): empirical checks of wgmma descriptor behaviour that the
// available documentation does not settle, and TMA box throughput for the box shapes the conv kernels use.
//
// cpb200_probe_halo: can ONE (TH+2)x(TW+2) halo tile in shared memory (TMA, 128B swizzle, 128-byte pixel rows) serve all
// nine taps of a 3x3 conv through shifted wgmma descriptors?  With TW = 8 every 8-row core-matrix group of the A operand is
// one tile row, so tap (r,s) is
//   start = base + (r*(TW+2) + s)*128 B,  SBO = (TW+2)*128 B  (not a multiple of the 1024-B swizzle repeat),
// and the second warpgroup's 64 rows start 8 halo rows later.  Works iff the hardware applies the swizzle XOR to absolute
// shared-memory address bits; variant 0 leaves the descriptor's base_offset at 0 (what csrc/net_tc3.cu does), variant 1
// sets it to (start >> 7) & 7.
#include "tc_common.cuh"

namespace {

using namespace tc;

struct alignas(64) ProbeArgs {
  CUtensorMap xmap;    // (C=64, W=TW+2, H=TH+2, N=1) bf16
  CUtensorMap wmap;    // (Cin=64, Cout=64, taps=9) bf16
  float *out;          // (128, 64) fp32
  int variant;         // 0: base_offset = 0 ; 1: base_offset = (start >> 7) & 7
};

constexpr int TW = 8, TH = 16, HALO_W = TW + 2, HALO_H = TH + 2;

__global__ void __launch_bounds__(256, 1) probe_halo_kernel(const __grid_constant__ ProbeArgs a) {
  extern __shared__ __align__(1024) uint8_t raw[];
  const uint32_t base = (smem_u32(raw) + 1023u) & ~1023u;
  const uint32_t xs = base;                                   // halo tile: 180 rows x 128 B = 23040 B
  const uint32_t ws = base + 24 * 1024;                       // 9 x (64 x 128 B) = 73728 B
  __shared__ __align__(8) uint64_t bar_;
  const uint32_t bar = smem_u32(&bar_);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, HALO_W * HALO_H * 128 + 9 * 64 * 128);
    tma_load_4d(xs, &a.xmap, bar, 0, 0, 0, 0);
    for (int t = 0; t < 9; ++t) tma_load_3d(ws + t * 8192, &a.wmap, bar, 0, 0, t);
  }
  mbar_wait(bar, 0);
  const int wg = threadIdx.x >> 7, tq = threadIdx.x & 127;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  wg_fence();
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int r = t / 3, s = t % 3;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t astart = xs + (r * HALO_W + s + wg * 8 * HALO_W) * 128 + k * 32;
      uint64_t ad = desc_sbo(astart, HALO_W * 128, 1);        // SBO = one halo row of pixels
      if (a.variant == 1) ad |= (uint64_t)((astart >> 7) & 7) << 49;
      const uint64_t bd = make_desc(ws + t * 8192 + k * 32, 128, 1);
      wgmma_k16<64>(acc, ad, bd, (t > 0 || k > 0) ? 1u : 0u, 1u);
    }
  }
  wg_commit();
  wg_wait<0>();
  acc_fence(acc);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int row = wg * 64 + frag_row(tq, j), col = frag_col(tq, j);
    a.out[row * 64 + col] = acc[2 * j];
    a.out[row * 64 + col + 1] = acc[2 * j + 1];
  }
}

// ---- TMA box-throughput probe: every CTA streams boxes of one shape through an N-deep smem ring ----
struct alignas(64) TmaProbeArgs {
  CUtensorMap map;
  int tiles_w, tiles_h, nimg, total, stages, box_w, box_h, step_w, step_h;
  unsigned bytes, stage_bytes;
};

__global__ void __launch_bounds__(64, 1) probe_tma_kernel(const __grid_constant__ TmaProbeArgs a) {
  extern __shared__ __align__(1024) uint8_t raw[];
  const uint32_t base = (smem_u32(raw) + 1023u) & ~1023u;
  __shared__ __align__(8) uint64_t bars[32];
  const uint32_t full0 = smem_u32(&bars[0]), empty0 = smem_u32(&bars[16]);
  if (threadIdx.x == 0) {
    for (int s = 0; s < a.stages; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {                 // producer
    int st = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < a.total; t += gridDim.x) {
      const int tw = t % a.tiles_w, th = (t / a.tiles_w) % a.tiles_h, n = t / (a.tiles_w * a.tiles_h);
      mbar_wait(empty0 + 8 * st, ph ^ 1);
      mbar_expect_tx(full0 + 8 * st, a.bytes);
      asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                   ::"r"(base + st * a.stage_bytes), "l"(reinterpret_cast<uint64_t>(&a.map)), "r"(full0 + 8 * st),
                     "r"(0), "r"(tw * a.step_w - 1), "r"(th * a.step_h - 1), "r"(n) : "memory");
      if (++st == a.stages) { st = 0; ph ^= 1; }
    }
  } else if (threadIdx.x == 32) {         // consumer: release the slot as soon as the bytes landed
    int st = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < a.total; t += gridDim.x) {
      mbar_wait(full0 + 8 * st, ph);
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * st) : "memory");
      if (++st == a.stages) { st = 0; ph ^= 1; }
    }
  }
}

}  // namespace

// x: (1, 18, 10, 64) bf16 NHWC;  w: (9, 64, 64) bf16 [tap][cout][cin];  out: (128, 64) fp32, row = th*8 + tw
extern "C" int cpb200_probe_halo(const void *x, const void *w, float *out, int variant, void *stream) {
  void *p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
    return cpb::fail(CPB200_ERR_STATE, "probe: cuTensorMapEncodeTiled unavailable");
  EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(p);
  ProbeArgs a;
  memset(&a, 0, sizeof(a));
  {
    const cuuint64_t dims[4] = {64, HALO_W, HALO_H, 1};
    const cuuint64_t strides[3] = {128, (cuuint64_t)HALO_W * 128, (cuuint64_t)HALO_W * HALO_H * 128};
    const cuuint32_t box[4] = {64, HALO_W, HALO_H, 1};
    const cuuint32_t es[4] = {1, 1, 1, 1};
    if (enc(&a.xmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(x), dims, strides, box, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return cpb::fail(CPB200_ERR_CUDA, "probe: encode x failed");
  }
  {
    const cuuint64_t dims[3] = {64, 64, 9};
    const cuuint64_t strides[2] = {128, 64 * 128};
    const cuuint32_t box[3] = {64, 64, 1};
    const cuuint32_t es[3] = {1, 1, 1};
    if (enc(&a.wmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(w), dims, strides, box, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return cpb::fail(CPB200_ERR_CUDA, "probe: encode w failed");
  }
  a.out = out; a.variant = variant;
  const size_t smem = 24 * 1024 + 9 * 8192 + 1024;
  CPB_CUDA(cudaFuncSetAttribute(probe_halo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  probe_halo_kernel<<<1, 256, smem, static_cast<cudaStream_t>(stream)>>>(a);
  return cpb::check_launch("probe_halo_kernel");
}



// Streams (C,W,H,N) bf16 through TMA boxes {C, box_w, box_h, 1} stepping (step_w, step_h); returns after enqueue.
extern "C" int cpb200_probe_tma(const void *x, int C, int W, int H, int N, int box_w, int box_h, int step_w, int step_h,
                                int stages, void *stream) {
  void *p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
    return cpb::fail(CPB200_ERR_STATE, "probe: cuTensorMapEncodeTiled unavailable");
  EncodeTiledFn enc = reinterpret_cast<EncodeTiledFn>(p);
  TmaProbeArgs a;
  memset(&a, 0, sizeof(a));
  const CUtensorMapSwizzle sw = C == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : C == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)C, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  const cuuint32_t es[4] = {1, 1, 1, 1};
  if (enc(&a.map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(x), dims, strides, box, es,
          CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cpb::fail(CPB200_ERR_CUDA, "probe: encode failed");
  a.tiles_w = (W + step_w - 1) / step_w; a.tiles_h = (H + step_h - 1) / step_h; a.nimg = N;
  a.total = a.tiles_w * a.tiles_h * N; a.stages = stages; a.box_w = box_w; a.box_h = box_h; a.step_w = step_w; a.step_h = step_h;
  a.bytes = (unsigned)(C * 2 * box_w * box_h); a.stage_bytes = (a.bytes + 1023u) & ~1023u;
  const size_t smem = (size_t)stages * a.stage_bytes + 1024;
  if (stages > 16 || smem > 200 * 1024) return cpb::fail(CPB200_ERR_ARG, "probe: ring too large");
  CPB_CUDA(cudaFuncSetAttribute(probe_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, nsm = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  probe_tma_kernel<<<nsm, 64, smem, static_cast<cudaStream_t>(stream)>>>(a);
  return cpb::check_launch("probe_tma_kernel");
}

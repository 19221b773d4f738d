// PTX wrappers shared by the wgmma / TMA kernels (sm_90a).
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include "wgmma.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One thread of a converged warp (PTX elect.sync).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tmap_prefetch(const CUtensorMap *map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// ---- warpgroup MMA ----
// Shared-memory matrix descriptor, K-major operand in a 128B / 64B / 32B-swizzled layout (layout 1 / 2 / 3): start address,
// stride between 8-row core-matrix groups (SBO); the leading offset is unused for swizzled K-major operands.  The swizzle
// XOR is applied to absolute shared-memory address bits, so a start address may sit anywhere inside a swizzle atom (+32 B
// per K step of 16, whole 16..128-byte pixel rows for the shifted halo windows of the 3x3 / 7x7 kernels).
__device__ __forceinline__ uint64_t desc_sbo(uint32_t saddr, uint32_t sbo_bytes, uint32_t layout_type) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);                 // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                                  // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(sbo_bytes >> 4) << 32;                   // stride byte offset between 8-row groups
  d |= (uint64_t)layout_type << 62;                        // 1 = SW128, 2 = SW64, 3 = SW32
  return d;
}
// rows of `row_bytes` (= swizzle span), 8-row groups packed back to back (what a TMA box with inner extent = swizzle span writes)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t row_bytes, uint32_t layout_type) {
  return desc_sbo(saddr, 8u * row_bytes, layout_type);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Fragment order of a 64 x N accumulator: register i of thread t (0..127 of the warpgroup) holds
//   row (t / 32) * 16 + (t % 32) / 4 + 8 * ((i / 2) % 2),  column 8 * (i / 4) + 2 * (t % 4) + i % 2.
// The epilogues walk it as pairs of adjacent columns: pair j = registers (2j, 2j+1).
__device__ __forceinline__ int frag_row(int t, int j) { return (t >> 5) * 16 + ((t & 31) >> 2) + 8 * (j & 1); }
__device__ __forceinline__ int frag_col(int t, int j) { return 8 * (j >> 1) + 2 * (t & 3); }

// ------------------------------------------------------------------------------------------------------------
// Split-operand ("x2") arithmetic: every fp32 value v is carried as two 16-bit planes hi = rn16(v),
// lo = rn16(v - hi); a product a*b is evaluated on the tensor core as a_hi*b_hi + a_hi*b_lo + a_lo*b_hi with fp32
// accumulation (the dropped a_lo*b_lo term is <= 2^-16 / 2^-22 of the product for bf16 / fp16 planes).
// fmt: 0 = bf16 planes (8+8 significand bits, fp32 range), 1 = fp16 planes (11+11 bits, |v| <= 65504 — the epilogues
// saturate; weights are pre-scaled by a power of two on the host so that their lo parts stay normal numbers).
__device__ __forceinline__ void split2(float a, float b, uint32_t fmt, uint32_t &hi, uint32_t &lo) {
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
// same without the fp16 saturation, for values known to lie within +-65504 (convex combinations of stored activations)
__device__ __forceinline__ void split2_bounded(float a, float b, uint32_t fmt, uint32_t &hi, uint32_t &lo) {
  if (fmt) {
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
__device__ __forceinline__ float2 unpack2(uint32_t v, uint32_t fmt) {
  if (fmt) return __half22float2(*reinterpret_cast<const __half2 *>(&v));
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&v));
}
__device__ __forceinline__ float2 join2(uint32_t hi, uint32_t lo, uint32_t fmt) {
  const float2 h = unpack2(hi, fmt), l = unpack2(lo, fmt);
  return make_float2(h.x + l.x, h.y + l.y);
}

// 16-bit NHWC output of one pixel, channels (nb, nb + 1): f0 / f1 already carry bias and accumulator scale; adds the
// residual (same layout as the output), applies the activation, stores (P = 2: hi plane at e, lo plane `plane` later).
template <int P>
__device__ __forceinline__ void store_pair16(void *dst, const void *res, size_t e, long long plane, float f0, float f1, uint32_t act,
                                             uint32_t fmt) {
  if constexpr (P == 2) {
    uint16_t *o = static_cast<uint16_t *>(dst) + e;
    if (res) {
      const uint16_t *r = static_cast<const uint16_t *>(res) + e;
      const float2 x = join2(__ldg(reinterpret_cast<const unsigned int *>(r)), __ldg(reinterpret_cast<const unsigned int *>(r + plane)), fmt);
      f0 += x.x; f1 += x.y;
    }
    uint32_t hi, lo;
    split2(cpb::act_fast(f0, act), cpb::act_fast(f1, act), fmt, hi, lo);
    *reinterpret_cast<uint32_t *>(o) = hi;
    *reinterpret_cast<uint32_t *>(o + plane) = lo;
  } else {
    __nv_bfloat16 *o = static_cast<__nv_bfloat16 *>(dst) + e;
    if (res) {
      const float2 x = __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162 *>(static_cast<const __nv_bfloat16 *>(res) + e)));
      f0 += x.x; f1 += x.y;
    }
    *reinterpret_cast<__nv_bfloat162 *>(o) = __floats2bfloat162_rn(cpb::act_out<__nv_bfloat16>(f0, act), cpb::act_out<__nv_bfloat16>(f1, act));
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode();
int num_sms();          // SM count of the CURRENT device (cached per device)
int cur_device();

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): remember the largest value set on each device.
constexpr int MAX_DEVICES = 64;
struct SmemAttrCache { size_t v[MAX_DEVICES] = {}; };
template <typename F>
inline int ensure_smem(F *func, size_t smem, SmemAttrCache &cache) {
  const int dev = cur_device();
  if (dev < 0 || dev >= MAX_DEVICES) return cpb::fail(CPB200_ERR_STATE, "device index %d out of range", dev);
  if (smem > cache.v[dev]) {
    CPB_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cache.v[dev] = smem;
  }
  return CPB200_OK;
}

}  // namespace tc

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

// ------------------------------------------------------------------------------------------------------------
// What every wgmma kernel's consumers share: the accumulators, the K step and the epilogue.  Each kernel keeps its own
// producers and its own pixel mapping.
//
// acc holds A_hi x W_hi (P = 1: A x W); acc2 holds the split operands' small cross terms (one unused register when P = 1).
template <int R, int R2>
__device__ __forceinline__ void acc_zero(float (&acc)[R], float (&acc2)[R2]) {
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < R2; ++i) acc2[i] = 0.f;
}

// K step k (16 channels: +32 bytes in each descriptor) of an N-column product from shared-memory descriptors.  P = 2
// issues A_hi x W_hi into acc, then A_hi x W_lo and A_lo x W_hi into acc2.  The cross terms share the second array because the tensor core's fp32
// accumulator truncates (round toward zero) at every instruction, an error proportional to the accumulator's magnitude:
// the large hi x hi sum must see as few additions as possible.  Separate arrays also keep the three products of a step
// independent, so ptxas does not serialise them.  `first` = 0 overwrites the accumulators instead of adding to them.
template <int N, int P>
__device__ __forceinline__ void mma_step(float *acc, float *acc2, uint64_t a_hi, uint64_t a_lo, uint64_t w_hi, uint64_t w_lo,
                                         int k, uint32_t first, uint32_t bf) {
  if constexpr (P == 1) {
    wgmma_k16<N>(acc, a_hi + 2 * k, w_hi + 2 * k, first, 1u);
  } else {
    wgmma_k16<N>(acc, a_hi + 2 * k, w_hi + 2 * k, first, bf);
    wgmma_k16<N>(acc2, a_hi + 2 * k, w_lo + 2 * k, first, bf);
    wgmma_k16<N>(acc2, a_lo + 2 * k, w_hi + 2 * k, 1u, bf);
  }
}
// All `ksteps` (1, 2 or 4: a K slab of 16, 32 or 64 channels) K steps of one stage; `first` applies to step 0, the later
// steps accumulate.  The operand type and the step count are fixed once per stage, so the stage is straight-line code:
// with a branch between two wgmma (the fp16 / bf16 choice per instruction, or a run-time step loop), ptxas fences every
// wgmma off from the next, with a warpgroup arrive and a scoreboard wait group each.  P = 2 issues the stage's
// A_hi x W_hi products back to back into acc, then its cross terms into acc2, step by step: every accumulator element
// sees the same products in the same order as with mma_step per K step.
template <int N, int P, uint32_t BF, int KS>
__device__ __forceinline__ void mma_stage_t(float *acc, float *acc2, uint64_t a_hi, uint64_t a_lo, uint64_t w_hi,
                                            uint64_t w_lo, uint32_t first) {
#pragma unroll
  for (int k = 0; k < KS; ++k) wgmma_k16<N>(acc, a_hi + 2 * k, w_hi + 2 * k, k == 0 ? first : 1u, BF);
  if constexpr (P == 2) {
#pragma unroll
    for (int k = 0; k < KS; ++k) {
      wgmma_k16<N>(acc2, a_hi + 2 * k, w_lo + 2 * k, k == 0 ? first : 1u, BF);
      wgmma_k16<N>(acc2, a_lo + 2 * k, w_hi + 2 * k, 1u, BF);
    }
  }
}
template <int N, int P, uint32_t BF>
__device__ __forceinline__ void mma_stage_bf(float *acc, float *acc2, uint64_t a_hi, uint64_t a_lo, uint64_t w_hi, uint64_t w_lo,
                                             int ksteps, uint32_t first) {
  if (ksteps == 4) mma_stage_t<N, P, BF, 4>(acc, acc2, a_hi, a_lo, w_hi, w_lo, first);
  else if (ksteps == 2) mma_stage_t<N, P, BF, 2>(acc, acc2, a_hi, a_lo, w_hi, w_lo, first);
  else mma_stage_t<N, P, BF, 1>(acc, acc2, a_hi, a_lo, w_hi, w_lo, first);
}
template <int N, int P>
__device__ __forceinline__ void mma_stage(float *acc, float *acc2, uint64_t a_hi, uint64_t a_lo, uint64_t w_hi, uint64_t w_lo,
                                          int ksteps, uint32_t first, uint32_t bf) {
  if (P == 1 || bf) mma_stage_bf<N, P, 1u>(acc, acc2, a_hi, a_lo, w_hi, w_lo, ksteps, first);
  else mma_stage_bf<N, P, 0u>(acc, acc2, a_hi, a_lo, w_hi, w_lo, ksteps, first);
}
// the same with the A fragments in registers (wgmma_rs_k16)
template <int N, int P>
__device__ __forceinline__ void mma_step_rs(float *acc, float *acc2, const uint32_t (&a_hi)[4], const uint32_t (&a_lo)[4],
                                            uint64_t w_hi, uint64_t w_lo, uint32_t first, uint32_t bf) {
  if constexpr (P == 1) {
    wgmma_rs_k16<N>(acc, a_hi, w_hi, first, 1u);
  } else {
    wgmma_rs_k16<N>(acc, a_hi, w_hi, first, bf);
    wgmma_rs_k16<N>(acc2, a_hi, w_lo, first, bf);
    wgmma_rs_k16<N>(acc2, a_lo, w_hi, 1u, bf);
  }
}

// Output forms of an epilogue: 16-bit NHWC (P = 2: hi and lo planes), NHWC fp32, NCHW fp32.
enum : int { OUT_16, OUT_F32, OUT_NCHW };
__device__ __forceinline__ int out_form(uint32_t flags) {
  return (flags & CPB200_FLAG_OUT_NCHW_F32) ? OUT_NCHW : (flags & CPB200_FLAG_OUT_F32) ? OUT_F32 : OUT_16;
}

// Finishes channels (c, c + 1) of one output pixel from accumulator registers 2j, 2j + 1: adds acc2 (P = 2), scales by
// acc_scale and adds the bias (P = 2: fmaf(v, acc_scale, bias), the inverse of the host's power-of-two weight scale;
// P = 1: v + bias), adds the residual (16-bit form only; same layout as dst), applies the activation and stores element
// e of dst.  `plane`: elements between the hi and lo planes (16-bit form) or between two channels (NCHW).  `has1`:
// channel c + 1 exists; the fp32 forms check it, 16-bit outputs always hold whole pairs (cout % 16 == 0).
// The activation is the multiply-by-1/6 form everywhere except NCHW fp32 in the split precisions: those are the
// network's result maps at fp32 accuracy and take act_fn, the IEEE division of the fp32 CUDA-core kernels.  NHWC fp32
// keeps the fast form: plan.py uses it for the DCN offset / mask maps, which have no activation.
template <int P>
__device__ __forceinline__ void epilogue_pair(const float *acc, const float *acc2, int j, float b0, float b1, float acc_scale,
                                              uint32_t act, int form, void *dst, const void *res, size_t e, long long plane,
                                              bool has1, uint32_t fmt) {
  float f0 = acc[2 * j], f1 = acc[2 * j + 1];
  if constexpr (P == 2) {
    f0 = fmaf(f0 + acc2[2 * j], acc_scale, b0); f1 = fmaf(f1 + acc2[2 * j + 1], acc_scale, b1);
  } else {
    f0 += b0; f1 += b1;
  }
  if (form == OUT_NCHW) {
    float *o = static_cast<float *>(dst) + e;
    o[0] = P == 2 ? cpb::act_fn(f0, act) : cpb::act_fast(f0, act);
    if (has1) o[plane] = P == 2 ? cpb::act_fn(f1, act) : cpb::act_fast(f1, act);
  } else if (form == OUT_F32) {
    float *o = static_cast<float *>(dst) + e;
    o[0] = cpb::act_fast(f0, act);
    if (has1) o[1] = cpb::act_fast(f1, act);
  } else if constexpr (P == 2) {
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
    *reinterpret_cast<__nv_bfloat162 *>(o) = __floats2bfloat162_rn(cpb::act_fast(f0, act), cpb::act_fast(f1, act));
  }
}

// ------------------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode();
int num_sms();          // SM count of the CURRENT device (cached per device)
int cur_device();

// Activation formats the wgmma kernels take: bf16, or the split planes (bf16x2 / fp16x2).
bool tc_dtype(int act_dtype);
// P = 2 planes for the split precisions, fmt 1 for fp16 planes; an acc_scale of 0 is read as 1
struct Prec { int P; uint32_t fmt; float acc_scale; };
Prec prec_of(const cpb200_op &op);

// K slab: bk = 64 / 32 / 16 channels, one 128B / 64B / 32B swizzle atom, the widest that divides every input's channel
// count.  `layout` is the matching wgmma descriptor layout type.  PlanBuilder._tc_bk (plan.py) mirrors this choice when
// it packs the weights.
struct Slab { int bk; CUtensorMapSwizzle swizzle; uint32_t layout; };
Slab slab_for(const int *cin, int nsrc);
// N tile: the next power of two >= cout, 16..256; split operands hold two BN-column accumulator arrays, so BN <= 128.
int bn_for(int cout, int P);

// 4-D map {C, W, H, B * P} of an NHWC activation with `pitch` elements per pixel (a channel slice of a wider tensor
// when pitch > C); split planes: the lo plane follows the hi plane of the parent tensor, i.e. a batch of 2B images.
int encode_act_map(CUtensorMap *map, const void *src, int C, int pitch, int W, int H, int B, int P, uint32_t fmt,
                   CUtensorMapSwizzle sw, const cuuint32_t (&box)[4], const cuuint32_t (&estr)[4], const char *what);
// 3-D map {bk, rows, blocks} of weights packed slab-major (plan.py::_pack_conv_tc): block = [plane][tap][K slab],
// `rows` output channels of bk each, one box = box_rows rows of one block, a dense run.
int encode_weight_map(CUtensorMap *map, const void *w, uint32_t fmt, int bk, int rows, int box_rows, long long blocks,
                      CUtensorMapSwizzle sw, const char *what);

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

// Launches a persistent kernel: one CTA per SM of the current device, or one per tile when there are fewer tiles.
// The shared-memory attribute cache is per instantiation, i.e. per kernel.
template <auto Kernel, typename Args>
int launch(const char *name, int tiles, int threads, size_t smem, cudaStream_t st, const Args &args) {
  static SmemAttrCache cache;
  if (int rc = ensure_smem(Kernel, smem, cache)) return rc;
  const int sms = num_sms();
  Kernel<<<tiles < sms ? tiles : sms, threads, smem, st>>>(args);
  return cpb::check_launch(name, Kernel);
}

}  // namespace tc

namespace cpb {
// Kernel families of the tensor-core ops.  cpb200_prepare_ops picks one per op and stores it behind op.tc with the
// route's prepared state (op.tc == NULL: the CUDA-core kernels); cpb200_run_ops switches on it and
// cpb200_release_ops deletes it.  Whatever Plan.bind can re-bind between runs is read from the live op at every run,
// never from prepared state: dst, res and bias for every route, the DCN offset / mask tensor (aux), and src[0] for the
// stem, which reads the network input.
enum class Route { HEADS, STEM, SP, HALO, TAP };
struct Prepared {
  const Route route;
  explicit Prepared(Route r) : route(r) {}
  virtual ~Prepared() = default;
};
}  // namespace cpb

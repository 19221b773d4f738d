// Activation formats of the CUDA-core kernels (net_simt.cu, net_eltwise.cu): fp32 / bf16 NHWC accessors and the
// pointer-like handles of split planes, so one kernel source takes every format on either side.
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>
#include <type_traits>

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
// `p + n` is force-inlined: outlined (NVVM -O1), it returns the handle through the stack and stores through it become
// generic instead of global.
struct SpC {
  const uint16_t *p; size_t plane; uint32_t fmt;
  __host__ __device__ __forceinline__ SpC operator+(size_t n) const { return SpC{p + n, plane, fmt}; }
  __host__ __device__ explicit operator bool() const { return p != nullptr; }
};
struct SpM {
  uint16_t *p; size_t plane; uint32_t fmt;
  __host__ __device__ __forceinline__ SpM operator+(size_t n) const { return SpM{p + n, plane, fmt}; }
};
__device__ __forceinline__ float4 io_ld4(const float *p) { return Act<float>::ld4(p); }
__device__ __forceinline__ float4 io_ld4(const bf16 *p) { return Act<bf16>::ld4(p); }
__device__ __forceinline__ float4 io_ld4(SpC p) { return Sp16::ld4(p.p, p.plane, p.fmt); }
__device__ __forceinline__ void io_st4(float *p, float4 v) { Act<float>::st4(p, v); }
__device__ __forceinline__ void io_st4(bf16 *p, float4 v) { Act<bf16>::st4(p, v); }
__device__ __forceinline__ void io_st4(SpM p, float4 v) { Sp16::st4(p.p, p.plane, p.fmt, v); }
// N = 4 or 8 consecutive values as float4 members, not an array: NVVM's -O1 pipeline does not unroll loops, so an
// array indexed in a loop would live in local memory.  The 8-element accesses are one 16-byte access per plane.
template <int N> struct Vf;
template <> struct Vf<4> { float4 a; };
template <> struct Vf<8> { float4 a, b; };
__device__ __forceinline__ float4 bf16x4(uint32_t lo, uint32_t hi) {
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&lo));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&hi));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 sp16x4(uint32_t h0, uint32_t h1, uint32_t l0, uint32_t l1, uint32_t fmt) {
  const float2 a = Sp16::up(h0, fmt), b = Sp16::up(h1, fmt), c = Sp16::up(l0, fmt), d = Sp16::up(l1, fmt);
  return make_float4(a.x + c.x, a.y + c.y, b.x + d.x, b.y + d.y);
}
__device__ __forceinline__ Vf<8> io_ld8(const bf16 *p) {
  const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
  return {bf16x4(r.x, r.y), bf16x4(r.z, r.w)};
}
__device__ __forceinline__ Vf<8> io_ld8(SpC p) {
  const uint4 h = __ldg(reinterpret_cast<const uint4 *>(p.p)), l = __ldg(reinterpret_cast<const uint4 *>(p.p + p.plane));
  return {sp16x4(h.x, h.y, l.x, l.y, p.fmt), sp16x4(h.z, h.w, l.z, l.w, p.fmt)};
}
template <int N, typename P> __device__ __forceinline__ Vf<N> io_ldv(P p) {
  if constexpr (N == 4) return {io_ld4(p)};
  else return io_ld8(p);
}
template <typename P> __device__ __forceinline__ void io_stv(P p, Vf<4> v) { io_st4(p, v.a); }
__device__ __forceinline__ void io_stv(bf16 *p, Vf<8> v) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.a.x, v.a.y), b = __floats2bfloat162_rn(v.a.z, v.a.w);
  const __nv_bfloat162 c = __floats2bfloat162_rn(v.b.x, v.b.y), d = __floats2bfloat162_rn(v.b.z, v.b.w);
  *reinterpret_cast<uint4 *>(p) = make_uint4(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b),
                                             *reinterpret_cast<const uint32_t *>(&c), *reinterpret_cast<const uint32_t *>(&d));
}
__device__ __forceinline__ void io_stv(SpM p, Vf<8> v) {
  uint4 h, l;
  Sp16::split2(v.a.x, v.a.y, p.fmt, h.x, l.x); Sp16::split2(v.a.z, v.a.w, p.fmt, h.y, l.y);
  Sp16::split2(v.b.x, v.b.y, p.fmt, h.z, l.z); Sp16::split2(v.b.z, v.b.w, p.fmt, h.w, l.w);
  *reinterpret_cast<uint4 *>(p.p) = h;
  *reinterpret_cast<uint4 *>(p.p + p.plane) = l;
}
template <int N> __device__ __forceinline__ Vf<N> ld_taps(const float *w) {     // fp32 filter taps
  const float4 a = __ldg(reinterpret_cast<const float4 *>(w));
  if constexpr (N == 4) return {a};
  else return {a, __ldg(reinterpret_cast<const float4 *>(w + 4))};
}
__device__ __forceinline__ float4 fma4(float4 x, float4 w, float4 acc) {
  return make_float4(fmaf(x.x, w.x, acc.x), fmaf(x.y, w.y, acc.y), fmaf(x.z, w.z, acc.z), fmaf(x.w, w.w, acc.w));
}
__device__ __forceinline__ Vf<4> vfma(Vf<4> x, Vf<4> w, Vf<4> acc) { return {fma4(x.a, w.a, acc.a)}; }
__device__ __forceinline__ Vf<8> vfma(Vf<8> x, Vf<8> w, Vf<8> acc) { return {fma4(x.a, w.a, acc.a), fma4(x.b, w.b, acc.b)}; }
// The epilogue activation follows the output format: act_fn for fp32, act_fast for bf16 and split planes (common.cuh).
template <typename PO> __device__ __forceinline__ float act_io(float v, uint32_t act) {
  if constexpr (std::is_same<PO, float *>::value) return cpb::act_fn(v, act);
  else return cpb::act_fast(v, act);
}
template <typename PO> __device__ __forceinline__ float4 act4(float4 v, uint32_t act) {
  return make_float4(act_io<PO>(v.x, act), act_io<PO>(v.y, act), act_io<PO>(v.z, act), act_io<PO>(v.w, act));
}
template <typename PO> __device__ __forceinline__ Vf<4> vact(Vf<4> v, uint32_t act) { return {act4<PO>(v.a, act)}; }
template <typename PO> __device__ __forceinline__ Vf<8> vact(Vf<8> v, uint32_t act) { return {act4<PO>(v.a, act), act4<PO>(v.b, act)}; }
__device__ __forceinline__ float4 add4(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ Vf<4> vadd(Vf<4> a, Vf<4> b) { return {add4(a.a, b.a)}; }
__device__ __forceinline__ Vf<8> vadd(Vf<8> a, Vf<8> b) { return {add4(a.a, b.a), add4(a.b, b.b)}; }

inline int ilog2(int v) {                                      // log2 of a power of two, else -1
  int l = 0;
  while ((1 << l) < v) ++l;
  return (1 << l) == v ? l : -1;
}

// Activation handle of type P over the op tensor at p, n elements per plane (plain pointers ignore n and fmt).
template <typename P> P io_handle(const void *p, size_t n, uint32_t fmt) {
  void *q = const_cast<void *>(p);
  if constexpr (std::is_same<P, SpC>::value) return SpC{static_cast<const uint16_t *>(q), n, fmt};
  else if constexpr (std::is_same<P, SpM>::value) return SpM{static_cast<uint16_t *>(q), n, fmt};
  else return static_cast<P>(q);
}

}  // namespace

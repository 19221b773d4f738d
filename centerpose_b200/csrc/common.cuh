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

#define CPB_CUDA(call)                                                                 \
  do {                                                                                 \
    cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess)                                                             \
      return cpb::fail(CPB200_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_));      \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

#define CPB_ACT_MASK (CPB200_FLAG_RELU | CPB200_FLAG_HSWISH | CPB200_FLAG_HSIGMOID)
// Epilogue non-linearity selected by the op flags (at most one of RELU / HSWISH / HSIGMOID).  hswish and
// hsigmoid keep the reference's operation order x * relu6(x + 3) / 6 (mobilenetv3.py:84-93).
__device__ __forceinline__ float act_fn(float v, uint32_t act) {
  if (act == CPB200_FLAG_RELU) return fmaxf(v, 0.f);
  if (act == 0u) return v;
  const float r = fminf(fmaxf(v + 3.f, 0.f), 6.f);
  return act == CPB200_FLAG_HSWISH ? v * r / 6.f : r / 6.f;
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
  const float r = fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
  return act == CPB200_FLAG_HSWISH ? v * r : r;
}
template <typename T>
__device__ __forceinline__ float act_out(float v, uint32_t act) {
  if constexpr (sizeof(T) == 4) {
    return act_fn(v, act);
  } else {
    if (act == CPB200_FLAG_RELU) return fmaxf(v, 0.f);
    if (act == 0u) return v;
    const float r = fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f);
    return act == CPB200_FLAG_HSWISH ? v * r : r;
  }
}

}  // namespace cpb

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

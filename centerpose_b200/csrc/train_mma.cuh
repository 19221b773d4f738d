// The inner product of the training kernels (dcn_train.cu, heads_train.cu): a 64 x 128 CTA tile of 8 warps, each a
// 32 x 32 warp tile, fed BK = 16 deep slabs from shared memory.  Two precisions share every tile and accumulator layout
// (TrainPrec):
//   TRAIN_TF32X3  tensor cores, mma.sync m16n8k8 tf32 with each fp32 operand split as big + small (both tf32, rounded
//                 to nearest), summed as small*big + big*small + big*big in fp32.  tf32 keeps fp32's 8-bit exponent,
//                 so the split is scale-free: 2^k x splits to 2^k big + 2^k small over fp32's whole normal range, and
//                 every product and sum scales with it.
//   TRAIN_FP32    CUDA-core fp32 FMAs over the same shared-memory tiles, for reference-precision parity.
#pragma once
#include <stdint.h>

namespace cpb {
namespace train {

constexpr int NT = 256;                 // 8 warps: 2 along M x 4 along N, a 32 x 32 warp tile each
constexpr int BM = 64, BN = 128, BK = 16;
constexpr int AP = BK + 4;              // As[m][k] row pitch: fragment loads hit 32 distinct banks
constexpr int BP = BN + 8;              // Bs[k][n] row pitch, likewise

enum TrainPrec { TRAIN_TF32X3 = 0, TRAIN_FP32 = 1 };

__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ void split_tf32(float x, uint32_t &big, uint32_t &small) {
  big = tf32_rna(x);
  small = tf32_rna(__fsub_rn(x, __uint_as_float(big)));
}

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void zero_acc(float (&acc)[2][4][4]) {
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
}

// part += As (BM x BK) * Bs (BK x BN) for this warp's 32 x 32 tile.  Thread (gid = lane / 4, tig = lane % 4)
// holds the m16n8 accumulator fragment: part[mt][nt][0..3] at rows wm*32 + mt*16 + gid (+8 for [2], [3]) and columns
// wn*32 + nt*8 + 2*tig (+1 for [1], [3]) -- the same positions in both precisions.
template <int P>
__device__ __forceinline__ void tile_product(const float (*As)[AP], const float (*Bs)[BP], int wm, int wn, int lane,
                                             float (&part)[2][4][4]) {
  const int gid = lane >> 2, tig = lane & 3;
  if constexpr (P == TRAIN_TF32X3) {
#pragma unroll
    for (int kk = 0; kk < BK; kk += 8) {
      uint32_t ab[2][4], as[2][4], bb[4][2], bs[4][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int m = wm * 32 + mt * 16 + gid;
        split_tf32(As[m][kk + tig], ab[mt][0], as[mt][0]);
        split_tf32(As[m + 8][kk + tig], ab[mt][1], as[mt][1]);
        split_tf32(As[m][kk + tig + 4], ab[mt][2], as[mt][2]);
        split_tf32(As[m + 8][kk + tig + 4], ab[mt][3], as[mt][3]);
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int n = wn * 32 + nt * 8 + gid;
        split_tf32(Bs[kk + tig][n], bb[nt][0], bs[nt][0]);
        split_tf32(Bs[kk + tig + 4][n], bb[nt][1], bs[nt][1]);
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          mma_tf32(part[mt][nt], as[mt], bb[nt][0], bb[nt][1]);
          mma_tf32(part[mt][nt], ab[mt], bs[nt][0], bs[nt][1]);
          mma_tf32(part[mt][nt], ab[mt], bb[nt][0], bb[nt][1]);
        }
    }
  } else {
#pragma unroll 4
    for (int k = 0; k < BK; ++k) {
      float a[2][2], b[4][2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        a[mt][0] = As[wm * 32 + mt * 16 + gid][k];
        a[mt][1] = As[wm * 32 + mt * 16 + gid + 8][k];
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const float2 v = *reinterpret_cast<const float2 *>(&Bs[k][wn * 32 + nt * 8 + 2 * tig]);
        b[nt][0] = v.x;
        b[nt][1] = v.y;
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          part[mt][nt][0] = fmaf(a[mt][0], b[nt][0], part[mt][nt][0]);
          part[mt][nt][1] = fmaf(a[mt][0], b[nt][1], part[mt][nt][1]);
          part[mt][nt][2] = fmaf(a[mt][1], b[nt][0], part[mt][nt][2]);
          part[mt][nt][3] = fmaf(a[mt][1], b[nt][1], part[mt][nt][3]);
        }
    }
  }
}

// acc += As (BM x BK) * Bs (BK x BN) for this warp's 32 x 32 tile, in tile_product's fragment layout.
// The BK-deep product goes to a fresh partial that is added to acc with one rounded fp32 add.  The tensor cores'
// accumulation truncates, so chaining every MMA of a K = 4608 reduction into one accumulator drifts by some 1e-5
// relative; a partial per slab bounds the truncated chain at 6 MMAs and the long sum is rounded to nearest.  The CUDA-
// core path blocks its sum the same way.
template <int P>
__device__ __forceinline__ void tile_mma(const float (*As)[AP], const float (*Bs)[BP], int wm, int wn, int lane,
                                         float (&acc)[2][4][4]) {
  float part[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) part[mt][nt][i] = 0.f;
  tile_product<P>(As, Bs, wm, wn, lane, part);
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = __fadd_rn(acc[mt][nt][i], part[mt][nt][i]);
}

// tile_mma with the long sum compensated (Kahan): `comp` carries each add's rounding error into the next one, so a
// reduction over hundreds of slabs of same-signed products stays within a few fp32 roundings of the exact sum.
template <int P>
__device__ __forceinline__ void tile_mma_kahan(const float (*As)[AP], const float (*Bs)[BP], int wm, int wn, int lane,
                                               float (&acc)[2][4][4], float (&comp)[2][4][4]) {
  float part[2][4][4];
  zero_acc(part);
  tile_product<P>(As, Bs, wm, wn, lane, part);
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float y = __fsub_rn(part[mt][nt][i], comp[mt][nt][i]);
        const float t = __fadd_rn(acc[mt][nt][i], y);
        comp[mt][nt][i] = __fsub_rn(__fsub_rn(t, acc[mt][nt][i]), y);
        acc[mt][nt][i] = t;
      }
}

}  // namespace train
}  // namespace cpb

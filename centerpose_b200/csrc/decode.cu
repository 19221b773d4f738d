// Fused multi_pose_decode for sm_90a: 3x3 max-pool NMS + per-channel top-K + gather +
// keypoint/candidate assignment in ONE launch.
//
// Replaces (reference file:line)  lib/models/decode.py:10-16 (_nms), :87-96 (_topk_channel),
// :99-115 (_topk), :235-308 (multi_pose_decode) and lib/models/utils.py:11-25 (gathers).
//
// HBM-bound design (DESIGN.md "decode kernel"): the only full-map reads are `heat`
// (1 channel) and `hm_hp` (J channels), each read exactly once with coalesced float4 loads
// (+ a one-row halo per row strip); the 2J+6 regression channels are touched only at the
// K centre cells / J*K candidate cells (sparse 4-byte gathers straight from NCHW — the
// reference instead materialises NHWC copies of all of them, utils.py:22).
//
// Grid: one CTA per (image, heat-map channel) = B*(1+J) CTAs of 256 threads.
//   phase 1  each CTA scans its H*W map: thread = (row strip, 4-column group), rolling
//            3-row window in registers, horizontal neighbours by warp shuffle; local maxima
//            above the channel's floor go to per-warp candidate segments in shared memory
//            (ballot + popc ranking, no atomics), compacted afterwards.
//   phase 2  exact top-K SET of the candidates by adaptive bucket select (256 linear buckets over
//            the candidates' float-bit range; the boundary bucket is resolved by rank counting on
//            64-bit (value,~index) keys); only the centre channel orders its K rows (rank
//            counting) — keypoint-candidate order never reaches the output.  Degenerate inputs
//            (candidate overflow, massive ties, negative maps) take an exact but slow K-round
//            arg-max path so results stay defined everywhere.
//   phase 3  keypoint grouping for joint j is done by the joint-j CTA itself, after the centre CTA of its image
//            has published its K rows (release/acquire flag in the workspace; the centre CTA has the LOWEST block
//            index of its image, is therefore dispatched first and never waits — no deadlock, no second launch).
//            Round 1 let whichever CTA of a {centre, joint} pair finished second do the grouping; a centre CTA that
//            finished last then ran all J groupings serially (~50 of the 120 us the kernel took at B = 32).
#include "common.cuh"

namespace {

constexpr int TPB = 256;
constexpr int CAP = 4096;      // candidate capacity per channel map (32 KB of smem)
constexpr int BND = 64;        // boundary-bucket capacity resolved by rank counting
constexpr int MAXK = CPB200_DECODE_MAX_K;
constexpr unsigned FULL = 0xffffffffu;

struct DecodeParams {
  const float *heat, *wh, *kps, *reg, *hm_hp, *hp_offset;
  float *out;
  float *tk_val;   // (B, 1+J, K)
  int *tk_idx;     // (B, 1+J, K)
  int *sync;       // (B, J) pair counters, zero between launches
  int B, H, W, J, K;
  int apply_sigmoid;
  float thresh;
  const float *affine;   // optional (B,6): row-major 2x3 matrix applied to every (x,y) of image b
};

struct Smem {
  float cval[CAP];
  int cidx[CAP];
  unsigned long long bkey[BND];
  int hist[256];
  int warp_tot[8];
  float selv[MAXK];            // selected (unordered) top-K
  int seli[MAXK];
  float topv[MAXK];            // final per-channel list
  int topi[MAXK];
  float2 gxy[MAXK];
  float gs[MAXK];
  int gi[MAXK];
  float hd[MAXK];
  int hc[MAXK];
  unsigned long long red[8];
  unsigned kmin, kmax;
  int wcnt[8], wbase[8];
  int count, nsel, nbnd, digit, need, flags;
  unsigned todo_mask;
};

__device__ __forceinline__ float act(float v, bool sig) {
  return sig ? __fdividef(1.0f, 1.0f + __expf(-v)) : v;
}

__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// ---- phase 1, vector path (W % 4 == 0, 16-byte aligned map) -----------------------------
// Each thread owns a 4-column group and walks down a strip of rows with a rolling 3-row window
// (one float4 load per row, horizontal neighbours by shuffle).  Peaks above the floor are appended to
// the WARP's private candidate segment (ballot + popc ranking, no atomics, deterministic order);
// segments are compacted after the scan.
constexpr int SEG = CAP / (TPB / 32);      // 512 candidates per warp

__device__ void scan_vec(Smem &s, const float *__restrict__ map, int H, int W, bool sig, float floorv) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned lt = (1u << lane) - 1u;
  const int XG = W >> 2;
  int S = TPB / XG; if (S < 1) S = 1; if (S > H) S = H;
  const int RS = cpb::ceil_div(H, S);
  const int U = XG * S;
  const float NINF = -INFINITY;
  float *segv = s.cval + wid * SEG;
  int *segi = s.cidx + wid * SEG;
  int wcount = 0;                                            // warp-uniform
  for (int u0 = 0; u0 < U; u0 += TPB) {
    const int u = u0 + tid;
    const bool on = u < U;
    const int g = on ? (u % XG) : 0, st = on ? (u / XG) : 0;
    const int r0 = st * RS;
    const int r1 = min(H, r0 + RS);
    const int x0 = g * 4;
    const bool lpad = (g == 0), rpad = (g == XG - 1);
    const bool lsh = (lane > 0) && !lpad, rsh = (lane < 31) && !rpad;
    const float *base = map + x0;

    auto load_row = [&](int y, float4 &v, float4 &h) {
      const bool ok = on && y >= 0 && y < H;
      if (ok) {
        v = __ldg(reinterpret_cast<const float4 *>(base + (size_t)y * W));
        if (sig) { v.x = act(v.x, true); v.y = act(v.y, true); v.z = act(v.z, true); v.w = act(v.w, true); }
      } else {
        v = make_float4(NINF, NINF, NINF, NINF);
      }
      float l = __shfl_up_sync(FULL, v.w, 1);
      float r = __shfl_down_sync(FULL, v.x, 1);
      if (!lsh) l = (ok && !lpad) ? act(__ldg(base + (size_t)y * W - 1), sig) : NINF;
      if (!rsh) r = (ok && !rpad) ? act(__ldg(base + (size_t)y * W + 4), sig) : NINF;
      const float m01 = fmaxf(v.x, v.y), m23 = fmaxf(v.z, v.w);
      h.x = fmaxf(l, m01); h.y = fmaxf(m01, v.z); h.z = fmaxf(v.y, m23); h.w = fmaxf(m23, r);
    };

    float4 vcur, hprev, hcur, tmp;
    load_row(r0 - 1, tmp, hprev);
    load_row(r0, vcur, hcur);
    for (int i0 = 0; i0 < RS; i0 += 4) {
      float4 nv[4], nh[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int y = r0 + i0 + q + 1;
        load_row((y <= r1) ? y : -1, nv[q], nh[q]);            // row r1 is the strip's lower halo
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int y = r0 + i0 + q;
        const float mx = max3(hprev.x, hcur.x, nh[q].x), my = max3(hprev.y, hcur.y, nh[q].y);
        const float mz = max3(hprev.z, hcur.z, nh[q].z), mw = max3(hprev.w, hcur.w, nh[q].w);
        unsigned b = 0;
        b |= (vcur.x == mx && vcur.x > floorv) ? 1u : 0u;
        b |= (vcur.y == my && vcur.y > floorv) ? 2u : 0u;
        b |= (vcur.z == mz && vcur.z > floorv) ? 4u : 0u;
        b |= (vcur.w == mw && vcur.w > floorv) ? 8u : 0u;
        if (!(on && y < r1)) b = 0;
        unsigned m = __ballot_sync(FULL, b != 0);
        while (m) {                                            // 1 pass; a 2nd only if a float4 holds 2 peaks
          if (b) {
            const int k = __ffs(b) - 1;
            b &= b - 1;
            const float val = (k == 0) ? vcur.x : (k == 1) ? vcur.y : (k == 2) ? vcur.z : vcur.w;
            const int pos = wcount + __popc(m & lt);
            if (pos < SEG) { segv[pos] = val; segi[pos] = y * W + x0 + k; }
          }
          wcount += __popc(m);
          m = __ballot_sync(FULL, b != 0);
        }
        hprev = hcur; hcur = nh[q]; vcur = nv[q];
      }
    }
  }
  if (lane == 0) s.wcnt[wid] = wcount;
}

// ---- phase 1, W == 128 specialisation (the 512x512 configs: one warp spans a full map row) ---------------
// Same algorithm as scan_vec with everything the general path pays per row folded away at compile time: lane = column
// group, warp = row strip, no out-of-range threads, the row's left / right neighbours always come from the shuffle
// (lane 0 / 31 see -inf), row addresses advance by a constant, the logistic is a template switch.  The general path
// executes ~2.5x the instructions per row per thread.
template <bool SIG>
__device__ void scan_w128(Smem &s, const float *__restrict__ map, int H, float floorv) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned lt = (1u << lane) - 1u;
  constexpr int S = TPB / 32;                               // 8 strips
  const int RS = H / S;                                     // rows per strip (H % 8 == 0 checked by the caller)
  const int r0 = wid * RS;
  const float NINF = -INFINITY;
  float *segv = s.cval + wid * SEG;
  int *segi = s.cidx + wid * SEG;
  int wcount = 0;
  const float4 *rowp = reinterpret_cast<const float4 *>(map) + (size_t)r0 * 32 + lane;

  auto hmax = [&](const float4 &v, float4 &h) {
    float l = __shfl_up_sync(FULL, v.w, 1), r = __shfl_down_sync(FULL, v.x, 1);
    if (lane == 0) l = NINF;
    if (lane == 31) r = NINF;
    const float m01 = fmaxf(v.x, v.y), m23 = fmaxf(v.z, v.w);
    h.x = fmaxf(l, m01); h.y = fmaxf(m01, v.z); h.z = fmaxf(v.y, m23); h.w = fmaxf(m23, r);
  };
  auto ld = [&](const float4 *p) {
    float4 v = __ldg(p);
    if (SIG) { v.x = act(v.x, true); v.y = act(v.y, true); v.z = act(v.z, true); v.w = act(v.w, true); }
    return v;
  };
  const float4 ninf4 = make_float4(NINF, NINF, NINF, NINF);
  float4 vcur, hprev, hcur;
  if (r0 > 0) { const float4 t = ld(rowp - 32); hmax(t, hprev); } else hprev = ninf4;
  vcur = ld(rowp); hmax(vcur, hcur);
  int idx0 = r0 * 128 + lane * 4;                           // flat index of vcur.x
#pragma unroll 4
  for (int i = 0; i < RS; ++i) {
    float4 vn, hn;
    const bool has_next = (r0 + i + 1) < H;                 // warp-uniform
    if (has_next) { vn = ld(rowp + (size_t)(i + 1) * 32); hmax(vn, hn); } else { vn = ninf4; hn = ninf4; }
    const float mx = max3(hprev.x, hcur.x, hn.x), my = max3(hprev.y, hcur.y, hn.y);
    const float mz = max3(hprev.z, hcur.z, hn.z), mw = max3(hprev.w, hcur.w, hn.w);
    unsigned b = 0;
    b |= (vcur.x >= mx && vcur.x > floorv) ? 1u : 0u;       // v <= max always: '>=' is the equality test
    b |= (vcur.y >= my && vcur.y > floorv) ? 2u : 0u;
    b |= (vcur.z >= mz && vcur.z > floorv) ? 4u : 0u;
    b |= (vcur.w >= mw && vcur.w > floorv) ? 8u : 0u;
    unsigned m = __ballot_sync(FULL, b != 0);
    while (m) {                                             // 1 pass; a 2nd only if a float4 holds 2 peaks
      if (b) {
        const int k = __ffs(b) - 1;
        b &= b - 1;
        const float val = (k == 0) ? vcur.x : (k == 1) ? vcur.y : (k == 2) ? vcur.z : vcur.w;
        const int pos = wcount + __popc(m & lt);
        if (pos < SEG) { segv[pos] = val; segi[pos] = idx0 + k; }
      }
      wcount += __popc(m);
      m = __ballot_sync(FULL, b != 0);
    }
    hprev = hcur; hcur = hn; vcur = vn;
    idx0 += 128;
  }
  if (lane == 0) s.wcnt[wid] = wcount;
}

// Compact the per-warp segments [wid*SEG, wid*SEG + wcnt) into cval/cidx[0..n).  Returns n, or -1 when
// a segment overflowed (caller takes the exact slow path).
__device__ int compact_segments(Smem &s) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  __syncthreads();
  int base = 0, total = 0; bool over = false;
#pragma unroll
  for (int w = 0; w < TPB / 32; ++w) {
    const int c = s.wcnt[w];
    over |= c > SEG;
    if (w < wid) base += c;
    total += c;
  }
  if (over) return -1;
  const int mine = s.wcnt[wid];
  float rv[SEG / 32]; int ri[SEG / 32];
#pragma unroll
  for (int j = 0; j < SEG / 32; ++j) {
    const int e = j * 32 + lane;
    if (e < mine) { rv[j] = s.cval[wid * SEG + e]; ri[j] = s.cidx[wid * SEG + e]; }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < SEG / 32; ++j) {
    const int e = j * 32 + lane;
    if (e < mine) { s.cval[base + e] = rv[j]; s.cidx[base + e] = ri[j]; }
  }
  __syncthreads();
  return total;
}

// ---- post-NMS value of one cell straight from global memory (generic / slow paths) -------
__device__ __forceinline__ float nms_value(const float *__restrict__ map, int H, int W, int y,
                                           int x, bool sig, bool *is_peak) {
  const float v = act(__ldg(map + (size_t)y * W + x), sig);
  float m = v;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int xx = x + dx;
      if (xx < 0 || xx >= W || (dy == 0 && dx == 0)) continue;
      m = fmaxf(m, act(__ldg(map + (size_t)yy * W + xx), sig));
    }
  }
  *is_peak = (m == v);
  return (m == v) ? v : 0.0f;
}

// ---- phase 1, scalar path (any W / alignment) -------------------------------------------
__device__ void scan_scalar(Smem &s, const float *__restrict__ map, int H, int W, bool sig, float floorv) {
  const int N = H * W, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  const int iters = cpb::ceil_div(N, TPB);
  float *segv = s.cval + wid * SEG;
  int *segi = s.cidx + wid * SEG;
  int wcount = 0;
  for (int it = 0; it < iters; ++it) {
    const int cell = it * TPB + threadIdx.x;
    bool pk = false; float v = 0.f;
    if (cell < N) v = nms_value(map, H, W, cell / W, cell % W, sig, &pk);
    const bool has = pk && v > floorv;
    const unsigned m = __ballot_sync(FULL, has);
    if (has) {
      const int pos = wcount + __popc(m & lt);
      if (pos < SEG) { segv[pos] = v; segi[pos] = cell; }
    }
    wcount += __popc(m);
  }
  if (lane == 0) s.wcnt[wid] = wcount;
}

__device__ __forceinline__ unsigned long long make_key(float v, int idx) {
  unsigned u = __float_as_uint(v == 0.f ? 0.f : v);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)idx);
}
__device__ __forceinline__ float key_val(unsigned long long k) {
  unsigned u = (unsigned)(k >> 32);
  u = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
  return __uint_as_float(u);
}
__device__ __forceinline__ int key_idx(unsigned long long k) {
  return (int)(0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFull));
}

// exact, general, slow: K rounds of block-wide arg-max over the post-NMS map (degenerate inputs)
__device__ void select_slow(Smem &s, const float *__restrict__ map, int H, int W, bool sig, int K) {
  const int N = H * W, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  unsigned long long bound = ~0ull;
  for (int r = 0; r < K; ++r) {
    unsigned long long best = 0ull;
    for (int cell = tid; cell < N; cell += TPB) {
      bool pk;
      float v = nms_value(map, H, W, cell / W, cell % W, sig, &pk);
      unsigned long long k = make_key(v, cell);
      if (k < bound && k > best) best = k;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      unsigned long long other = __shfl_xor_sync(FULL, best, o);
      best = other > best ? other : best;
    }
    if (lane == 0) s.red[wid] = best;
    __syncthreads();
    best = s.red[0];
#pragma unroll
    for (int w = 1; w < TPB / 32; ++w) best = s.red[w] > best ? s.red[w] : best;
    if (tid == 0) { s.topv[r] = key_val(best); s.topi[r] = key_idx(best); }
    bound = best;
    __syncthreads();
  }
}

// ---- phase 2: exact top-K SET of the n candidates -> s.selv/s.seli[0..nsel) --------------
// Adaptive bucket select: histogram the candidates' float bits over their actual [min,max] range
// (256 linear buckets), everything above the boundary bucket is in, the boundary bucket is resolved
// by rank counting on 64-bit (value, ~index) keys, or refined with a narrower range.
// Returns false when the input is too degenerate (massive exact ties) -> caller uses select_slow.
__device__ bool select_set(Smem &s, int n, int K) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (n <= K) {
    for (int i = tid; i < n; i += TPB) { s.selv[i] = s.cval[i]; s.seli[i] = s.cidx[i]; }
    if (tid == 0) s.nsel = n;
    __syncthreads();
    return true;
  }
  // value-bit range of the candidates (all > 0, so float bits order like unsigned ints)
  unsigned lo_ = 0xFFFFFFFFu, hi_ = 0u;
  for (int i = tid; i < n; i += TPB) {
    const unsigned u = __float_as_uint(s.cval[i]);
    lo_ = min(lo_, u); hi_ = max(hi_, u);
  }
  lo_ = __reduce_min_sync(FULL, lo_); hi_ = __reduce_max_sync(FULL, hi_);
  if (tid == 0) { s.kmin = 0xFFFFFFFFu; s.kmax = 0u; s.nsel = 0; }
  __syncthreads();
  if (lane == 0) { atomicMin(&s.kmin, lo_); atomicMax(&s.kmax, hi_); }
  __syncthreads();
  unsigned lo = s.kmin, hi = s.kmax;
  int need = K;
  for (int round = 0; round < 5; ++round) {
    const unsigned range = hi - lo;
    const int shift = range ? max(0, 32 - __clz(range) - 8) : 0;
    s.hist[tid] = 0;
    if (tid == 0) s.nbnd = 0;
    __syncthreads();
    for (int i = tid; i < n; i += TPB) {
      const unsigned u = __float_as_uint(s.cval[i]);
      if (u >= lo && u <= hi) atomicAdd(&s.hist[(u - lo) >> shift], 1);
    }
    __syncthreads();
    const int h = s.hist[tid];
    int suf = h;                                  // inclusive suffix sum (buckets >= tid)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_down_sync(FULL, suf, o);
      if (lane + o < 32) suf += t;
    }
    if (lane == 0) s.warp_tot[wid] = suf;
    __syncthreads();
    for (int w = wid + 1; w < TPB / 32; ++w) suf += s.warp_tot[w];
    const int excl = suf - h;
    if (excl < need && need <= suf) { s.digit = tid; s.need = need - excl; }
    __syncthreads();
    const int tb = s.digit;
    const int need_b = s.need;                    // how many of the boundary bucket are still needed
    const int nb = s.hist[tb];
    const bool take_all = (nb == need_b);
    const bool resolve = !take_all && (nb <= BND);
    if (!take_all && !resolve && shift == 0) return false;      // > BND exact ties at the K-th value
    // everything above the boundary bucket is selected; the boundary bucket is taken whole,
    // parked for rank counting, or refined in the next round
    for (int i = tid; i < n; i += TPB) {
      const unsigned u = __float_as_uint(s.cval[i]);
      if (u < lo || u > hi) continue;
      const int b = (int)((u - lo) >> shift);
      if (b > tb || (b == tb && take_all)) {
        const int pos = atomicAdd(&s.nsel, 1);
        if (pos < MAXK) { s.selv[pos] = s.cval[i]; s.seli[pos] = s.cidx[i]; }
      } else if (b == tb && resolve) {
        const int pos = atomicAdd(&s.nbnd, 1);
        if (pos < BND) s.bkey[pos] = make_key(s.cval[i], s.cidx[i]);
      }
    }
    __syncthreads();
    if (take_all) return true;
    if (resolve) {
      const int m = s.nbnd;
      if (tid < m) {
        const unsigned long long me = s.bkey[tid];
        int rank = 0;
        for (int j = 0; j < m; ++j) rank += (s.bkey[j] > me) ? 1 : 0;
        if (rank < need_b) {
          const int pos = atomicAdd(&s.nsel, 1);
          if (pos < MAXK) { s.selv[pos] = key_val(me); s.seli[pos] = key_idx(me); }
        }
      }
      __syncthreads();
      return true;
    }
    need = need_b;
    const unsigned nlo = lo + ((unsigned)tb << shift);
    const unsigned nhi = nlo + ((1u << shift) - 1u);
    lo = nlo; hi = min(hi, nhi);
    __syncthreads();
  }
  return false;
}

// ---- phase 2b: order the selected set (centre channel) / fill placeholders ------------------
__device__ bool finalize_list(Smem &s, const float *__restrict__ map, int H, int W, bool sig, int K,
                              bool is_centre) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int N = H * W;
  const int take = min(s.nsel, K);
  if (is_centre) {
    // rows must come out sorted (score desc, index asc): rank counting over <= 128 keys
    if (tid < take) {
      const unsigned long long me = make_key(s.selv[tid], s.seli[tid]);
      int rank = 0;
      for (int j = 0; j < take; ++j) rank += (make_key(s.selv[j], s.seli[j]) > me) ? 1 : 0;
      s.topv[rank] = s.selv[tid]; s.topi[rank] = s.seli[tid];
    }
    __syncthreads();
    if (take < K) {
      // fewer than K positive peaks: the reference's topk then returns zero-valued cells; canonical
      // choice = lowest flat indices that are not selected peaks.  If a NEGATIVE peak exists the
      // zero cells no longer rank last among the rest -> exact slow path decides.
      int neg = 0;
      for (int cell = tid; cell < N; cell += TPB) {
        bool pk; const float v = nms_value(map, H, W, cell / W, cell % W, sig, &pk);
        neg |= (pk && v < 0.f) ? 1 : 0;
      }
      if (__syncthreads_or(neg)) return false;
      const int need = K - take;
      const int cand = tid;                         // 2K <= 256 candidates, one per thread
      bool free_cell = (cand < N) && (cand < 2 * K);
      if (free_cell) for (int i = 0; i < take; ++i) if (s.topi[i] == cand) { free_cell = false; break; }
      const unsigned m = __ballot_sync(FULL, free_cell);
      if (lane == 0) s.warp_tot[wid] = __popc(m);
      __syncthreads();
      int rank = __popc(m & ((1u << lane) - 1u));
      for (int w = 0; w < wid; ++w) rank += s.warp_tot[w];
      if (free_cell && rank < need) { s.topv[take + rank] = 0.0f; s.topi[take + rank] = cand; }
      __syncthreads();
    }
  } else {
    // keypoint channels: only the SET matters (order never reaches the output); entries below the
    // score threshold are interchangeable "masked" candidates (decode.py:282-285)
    for (int i = tid; i < K; i += TPB) {
      if (i < take) { s.topv[i] = s.selv[i]; s.topi[i] = s.seli[i]; }
      else { s.topv[i] = -1.0f; s.topi[i] = 0; }
    }
    __syncthreads();
  }
  return true;
}

// ---- phase 3: assign keypoint candidates of joint j to the K people of image b ----------
__device__ void group_joint(Smem &s, const DecodeParams &p, int b, int j) {
  const int tid = threadIdx.x;
  const int K = p.K, J = p.J, W = p.W, N = p.H * p.W;
  const int C1 = 1 + J;
  const float *cv = p.tk_val + ((size_t)b * C1 + (j + 1)) * K;
  const int *ci = p.tk_idx + ((size_t)b * C1 + (j + 1)) * K;
  const float *pv = p.tk_val + ((size_t)b * C1) * K;
  const int *pi = p.tk_idx + ((size_t)b * C1) * K;
  __syncthreads();
  if (tid < K) {
    const float v = __ldcg(cv + tid);
    const int idx = __ldcg(ci + tid);
    if (v > p.thresh) {                                       // decode.py:282-285
      const float fx = (float)(idx % W), fy = (float)(idx / W);
      float ox = 0.5f, oy = 0.5f;
      if (p.hp_offset) {                                      // decode.py:272-277
        ox = __ldg(p.hp_offset + ((size_t)b * 2 + 0) * N + idx);
        oy = __ldg(p.hp_offset + ((size_t)b * 2 + 1) * N + idx);
      }
      s.gxy[tid] = make_float2(__fadd_rn(fx, ox), __fadd_rn(fy, oy)); s.gs[tid] = v; s.gi[tid] = idx;
    } else {
      s.gxy[tid] = make_float2(-10000.0f, -10000.0f); s.gs[tid] = -1.0f; s.gi[tid] = 0x7fffffff;
    }
  }
  __syncthreads();
  const int pidx = tid & (MAXK - 1), half = tid >> 7;          // TPB == 2 * MAXK
  float kx = 0.f, ky = 0.f, l = 0.f, t = 0.f, r = 0.f, bt = 0.f, score = 0.f;
  float best_d = INFINITY; int best_c = 0;
  if (pidx < K) {
    const int idx = __ldcg(pi + pidx);
    score = __ldcg(pv + pidx);
    const float fx = (float)(idx % W), fy = (float)(idx / W);
    kx = __fadd_rn(__ldg(p.kps + ((size_t)b * 2 * J + 2 * j) * N + idx), fx);      // :244-247
    ky = __fadd_rn(__ldg(p.kps + ((size_t)b * 2 * J + 2 * j + 1) * N + idx), fy);
    float cx, cy;
    if (p.reg) {                                                                    // :248-255
      cx = __fadd_rn(fx, __ldg(p.reg + ((size_t)b * 2 + 0) * N + idx));
      cy = __fadd_rn(fy, __ldg(p.reg + ((size_t)b * 2 + 1) * N + idx));
    } else { cx = fx + 0.5f; cy = fy + 0.5f; }
    const float hw = __ldg(p.wh + ((size_t)b * 2 + 0) * N + idx) * 0.5f;           // :256-264
    const float hh = __ldg(p.wh + ((size_t)b * 2 + 1) * N + idx) * 0.5f;
    l = __fsub_rn(cx, hw); t = __fsub_rn(cy, hh); r = __fadd_rn(cx, hw); bt = __fadd_rn(cy, hh);
    const int hk = (K + 1) >> 1;
    const int c0 = half ? hk : 0, c1 = half ? K : hk;
    // nearest candidate on SQUARED distance (monotone in the reference's sqrt); exact ties ->
    // the reference's first-minimum over its score-sorted list = higher score, then lower index
#pragma unroll 4
    for (int c = c0; c < c1; ++c) {                                                 // :286-289
      const float2 g = s.gxy[c];
      const float dx = __fsub_rn(kx, g.x), dy = __fsub_rn(ky, g.y);
      const float d = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
      if (d < best_d) { best_d = d; best_c = c; }
      else if (d == best_d) {
        const float sc = s.gs[c], sb = s.gs[best_c];
        if (sc > sb || (sc == sb && s.gi[c] < s.gi[best_c])) best_c = c;
      }
    }
    if (half) { s.hd[pidx] = best_d; s.hc[pidx] = best_c; }
  }
  __syncthreads();
  if (half == 0 && pidx < K) {
    const float od = s.hd[pidx]; const int oc = s.hc[pidx];
    if (K > 1) {
      if (od < best_d) { best_d = od; best_c = oc; }
      else if (od == best_d) {
        const float sc = s.gs[oc], sb = s.gs[best_c];
        if (sc > sb || (sc == sb && s.gi[oc] < s.gi[best_c])) best_c = oc;
      }
    }
    const float min_dist = __fsqrt_rn(best_d);
    const float2 g = s.gxy[best_c];
    const float sx = g.x, sy = g.y, ss = s.gs[best_c];
    const bool rej = (sx < l) || (sx > r) || (sy < t) || (sy > bt) || (ss < p.thresh) ||
                     (min_dist > __fmul_rn(fmaxf(__fsub_rn(bt, t), __fsub_rn(r, l)), 0.3f));   // :300-302
    const int row = 5 + 3 * J;
    float *o = p.out + ((size_t)b * K + pidx) * row;
    float ox = rej ? kx : sx, oy = rej ? ky : sy;
    if (p.affine) {
      // fused back-projection to image pixels (lib/utils/post_process.py:8-19 + image.py:19-24,63-66):
      // [x', y'] = A(2x3) . [x, y, 1]
      const float *A = p.affine + (size_t)b * 6;
      const float a0 = __ldg(A), a1 = __ldg(A + 1), a2 = __ldg(A + 2), a3 = __ldg(A + 3), a4 = __ldg(A + 4), a5 = __ldg(A + 5);
      const float tx = fmaf(a0, ox, fmaf(a1, oy, a2)), ty = fmaf(a3, ox, fmaf(a4, oy, a5));
      ox = tx; oy = ty;
      if (j == 0) {
        const float l2 = fmaf(a0, l, fmaf(a1, t, a2)), t2 = fmaf(a3, l, fmaf(a4, t, a5));
        const float r2 = fmaf(a0, r, fmaf(a1, bt, a2)), b2 = fmaf(a3, r, fmaf(a4, bt, a5));
        l = l2; t = t2; r = r2; bt = b2;
      }
    }
    o[5 + 2 * j] = ox;
    o[5 + 2 * j + 1] = oy;
    o[5 + 2 * J + j] = ss;
    if (j == 0) { o[0] = l; o[1] = t; o[2] = r; o[3] = bt; o[4] = score; }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(TPB) decode_kernel(const DecodeParams p) {
  __shared__ Smem s;
  const int C1 = 1 + p.J;
  const int b = blockIdx.x / C1, ch = blockIdx.x % C1;
  const int tid = threadIdx.x;
  const bool is_centre = (ch == 0);
  const float *map = is_centre ? (p.heat + (size_t)b * p.H * p.W) : (p.hm_hp + ((size_t)b * p.J + (ch - 1)) * p.H * p.W);
  const bool sig = p.apply_sigmoid != 0;
  const float floorv = is_centre ? 0.0f : p.thresh;
  if (tid == 0) { s.count = 0; s.flags = 0; s.nsel = 0; s.todo_mask = 0; }
  __syncthreads();

  const bool vec_ok = ((p.W & 3) == 0) && ((reinterpret_cast<uintptr_t>(map) & 15) == 0);
  if (vec_ok && p.W == 128 && (p.H & 7) == 0) {
    if (sig) scan_w128<true>(s, map, p.H, floorv); else scan_w128<false>(s, map, p.H, floorv);
  } else if (vec_ok) scan_vec(s, map, p.H, p.W, sig, floorv);
  else scan_scalar(s, map, p.H, p.W, sig, floorv);
  const int ncand = compact_segments(s);

  bool done = false;
  if (ncand >= 0) {
    done = select_set(s, ncand, p.K);
    if (done) done = finalize_list(s, map, p.H, p.W, sig, p.K, is_centre);
  }
  if (!done) {
    __syncthreads();
    select_slow(s, map, p.H, p.W, sig, p.K);
    if (!is_centre)
      for (int i = tid; i < p.K; i += TPB)
        if (!(s.topv[i] > p.thresh)) { s.topv[i] = -1.0f; s.topi[i] = 0; }
    __syncthreads();
  }

  // publish this channel's list
  float *tv = p.tk_val + ((size_t)b * C1 + ch) * p.K;
  int *ti = p.tk_idx + ((size_t)b * C1 + ch) * p.K;
  for (int i = tid; i < p.K; i += TPB) { tv[i] = s.topv[i]; ti[i] = s.topi[i]; }
  // One word per image: bit 16 = "centre list published", low bits = joint CTAs finished.  Zero between launches
  // (the last joint CTA of the image restores it).
  int *flag = p.sync + (size_t)b * p.J;
  __syncthreads();
  if (is_centre) {
    if (tid == 0) {
      __threadfence();                                   // the K rows above are visible before the flag
      atomicAdd(flag, 1 << 16);
    }
    return;
  }
  if (tid == 0) {
    // joint CTA: its own list is in shared memory AND in the workspace (group_joint reads the workspace copy, written by
    // this CTA: visible after the barrier below); wait for the centre rows of this image
    while ((atomicAdd(flag, 0) >> 16) == 0) __nanosleep(64);
    __threadfence();
  }
  __syncthreads();
  group_joint(s, p, b, ch - 1);
  if (tid == 0) {
    const int done = atomicAdd(flag, 1) & 0xffff;
    if (done == p.J - 1) atomicExch(flag, 0);            // last joint of the image: restore the zero state
  }
}

__global__ void sigmoid_kernel(float *x, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) x[i] = 1.0f / (1.0f + expf(-x[i]));
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

extern "C" size_t cpb200_decode_workspace_bytes(int B, int J, int K) {
  if (B <= 0 || J <= 0 || K <= 0) return 0;
  const size_t n = (size_t)B * (1 + J) * K;
  return align_up(n * 4, 16) + align_up(n * 4, 16) + align_up((size_t)B * J * 4, 16);
}

static int decode_impl(const float *heat, const float *wh, const float *kps, const float *reg, const float *hm_hp,
                       const float *hp_offset, const float *affine, float *out, int B, int H, int W, int J, int K,
                       int apply_sigmoid, void *workspace, size_t workspace_bytes, void *stream) {
  if (!heat || !wh || !kps || !out) return cpb::fail(CPB200_ERR_ARG, "decode: null tensor pointer");
  if (!hm_hp)
    return cpb::fail(CPB200_ERR_ARG, "decode: hm_hp is required (the reference's decode.py:307 "
                                     "uses hm_score unconditionally)");
  if (B <= 0 || H <= 0 || W <= 0) return cpb::fail(CPB200_ERR_ARG, "decode: bad shape B=%d H=%d W=%d", B, H, W);
  if (J < 1 || J > CPB200_DECODE_MAX_J) return cpb::fail(CPB200_ERR_ARG, "decode: J=%d outside [1,%d]", J, CPB200_DECODE_MAX_J);
  if (K < 1 || K > CPB200_DECODE_MAX_K) return cpb::fail(CPB200_ERR_ARG, "decode: K=%d outside [1,%d]", K, CPB200_DECODE_MAX_K);
  if ((long long)K > (long long)H * W)
    return cpb::fail(CPB200_ERR_ARG, "decode: selected index k out of range (K=%d > H*W=%d)", K, H * W);
  if ((long long)H * W > (1ll << 30)) return cpb::fail(CPB200_ERR_ARG, "decode: map too large");
  const size_t need = cpb200_decode_workspace_bytes(B, J, K);
  if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15))
    return cpb::fail(CPB200_ERR_ARG, "decode: workspace too small or misaligned (%zu < %zu)", workspace_bytes, need);
  if ((long long)B * (1 + J) > 2147483647ll) return cpb::fail(CPB200_ERR_ARG, "decode: batch too large");

  DecodeParams p;
  p.heat = heat; p.wh = wh; p.kps = kps; p.reg = reg; p.hm_hp = hm_hp; p.hp_offset = hp_offset;
  p.out = out;
  const size_t n = (size_t)B * (1 + J) * K;
  char *ws = static_cast<char *>(workspace);
  p.tk_val = reinterpret_cast<float *>(ws);
  p.tk_idx = reinterpret_cast<int *>(ws + align_up(n * 4, 16));
  p.sync = reinterpret_cast<int *>(ws + 2 * align_up(n * 4, 16));
  p.B = B; p.H = H; p.W = W; p.J = J; p.K = K;
  p.apply_sigmoid = apply_sigmoid;
  p.affine = affine;
  p.thresh = 0.1f;                                   // decode.py:267
  decode_kernel<<<B * (1 + J), TPB, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return cpb::check_launch("decode_kernel");
}

extern "C" int cpb200_multi_pose_decode(const float *heat, const float *wh, const float *kps,
                                        const float *reg, const float *hm_hp,
                                        const float *hp_offset, float *out, int B, int H, int W,
                                        int J, int K, int apply_sigmoid, void *workspace,
                                        size_t workspace_bytes, void *stream) {
  return decode_impl(heat, wh, kps, reg, hm_hp, hp_offset, nullptr, out, B, H, W, J, K, apply_sigmoid, workspace,
                     workspace_bytes, stream);
}

extern "C" int cpb200_multi_pose_decode_affine(const float *heat, const float *wh, const float *kps,
                                               const float *reg, const float *hm_hp, const float *hp_offset,
                                               const float *affine, float *out, int B, int H, int W, int J, int K,
                                               int apply_sigmoid, void *workspace, size_t workspace_bytes,
                                               void *stream) {
  if (!affine) return cpb::fail(CPB200_ERR_ARG, "decode_affine: null affine");
  return decode_impl(heat, wh, kps, reg, hm_hp, hp_offset, affine, out, B, H, W, J, K, apply_sigmoid, workspace,
                     workspace_bytes, stream);
}

extern "C" int cpb200_sigmoid_inplace(float *x, size_t n, void *stream) {
  if (!x && n) return cpb::fail(CPB200_ERR_ARG, "sigmoid: null pointer");
  if (n == 0) return CPB200_OK;
  int blocks = (int)((n + 1023) / 1024);
  if (blocks > 132 * 16) blocks = 132 * 16;
  sigmoid_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n);
  return cpb::check_launch("sigmoid_kernel");
}

// COCO keypoint evaluation: pycocotools' COCOeval(gt, gt.loadRes(results), "keypoints") with the default Params,
// evaluate() and accumulate(), on the detection rows as tools/evaluate.py formats them (cpb200_coco_kp_eval,
// cpb200_coco_kp_oks).  Every step is float64 as numpy computes it; the file is built with -fmad=false, so no product
// is contracted into an FMA.
//
//   prep_kernel       one CTA per image: score = '{:.2f}' rounding of the row's score, a stable rank by -score
//                     (np.argsort(kind="mergesort"): NaN last, -0.0 ties 0.0), the first 20 kept with their rounded
//                     keypoints and loadRes' bbox area w * h of the rounded width and height
//   oks_kernel        one thread per (kept detection, ground truth): computeOks, its sum in np.sum's pairwise order
//   match_kernel      one thread per (image, area range, threshold): evaluateImg's greedy match
//   bitonic kernels   one sort of every kept detection by (-score, position): accumulate's stable mergesort
//   accumulate_kernel one CTA per (area range, threshold): the tp / fp scans, the backward running maximum of
//                     precision and the 101 searchsorted(side="left") of the recall thresholds
#include "common.cuh"

#include <algorithm>

namespace {

static_assert(sizeof(cpb200_coco_kp_image) == 32, "cpb200_coco_kp_image layout is part of the C ABI");
static_assert(sizeof(cpb200_coco_kp_gt) == 336, "cpb200_coco_kp_gt layout is part of the C ABI");

constexpr int J = CPB200_COCO_KP_JOINTS;
constexpr int MAXD = CPB200_COCO_KP_MAX_DETS;
constexpr int T = CPB200_COCO_KP_T, R = CPB200_COCO_KP_R, A = CPB200_COCO_KP_A, AT = A * T;
constexpr int kRowFloats = 56;
constexpr double kSpacing1 = 2.220446049250313e-16;   // np.spacing(1)
constexpr int kScanThreads = 1024;
constexpr int kSortBlock = 2 * kScanThreads;          // elements one CTA sorts in shared memory

struct Kept {                      // one kept detection as loadRes leaves it
  double x[J], y[J];
  double score, area;
};

struct Workspace {
  double *score;                   // n_rows rounded scores
  Kept *kept;                      // n_keep
  double *oks;                     // n_oks
  unsigned char *gtm;              // AT x n_gts: ground truth matched at (area range, threshold)
  unsigned char *flags;            // AT x n_keep: bit 0 dtMatches != 0, bit 1 dtIgnore
  unsigned long long *keys;        // P sort keys
  unsigned *order;                 // P positions in `kept`
  int *tp;                         // AT x n_keep cumulative true positives
  double *pr;                      // AT x n_keep precision, then its backward running maximum
  int64_t P;
};

size_t align256(size_t n) { return (n + 255) / 256 * 256; }

int64_t sort_size(int n_keep) {
  int64_t p = kSortBlock;
  while (p < n_keep) p <<= 1;
  return p;
}

Workspace carve(void *base, int64_t n_rows, int n_gts, int n_keep, int64_t n_oks, size_t *total) {
  Workspace w;
  char *p = static_cast<char *>(base);
  size_t at = 0;
  auto take = [&](size_t bytes) { char *q = p ? p + at : nullptr; at += align256(std::max<size_t>(bytes, 1)); return q; };
  w.P = sort_size(n_keep);
  w.score = reinterpret_cast<double *>(take(sizeof(double) * n_rows));
  w.kept = reinterpret_cast<Kept *>(take(sizeof(Kept) * n_keep));
  w.oks = reinterpret_cast<double *>(take(sizeof(double) * n_oks));
  w.gtm = reinterpret_cast<unsigned char *>(take((size_t)AT * n_gts));
  w.flags = reinterpret_cast<unsigned char *>(take((size_t)AT * n_keep));
  w.keys = reinterpret_cast<unsigned long long *>(take(sizeof(unsigned long long) * w.P));
  w.order = reinterpret_cast<unsigned *>(take(sizeof(unsigned) * w.P));
  w.tp = reinterpret_cast<int *>(take(sizeof(int) * AT * (size_t)n_keep));
  w.pr = reinterpret_cast<double *>(take(sizeof(double) * AT * (size_t)n_keep));
  if (total) *total = at;
  return w;
}

// float('{:.2f}'.format(v)): v * 100 rounded to the nearest integer, ties to even, decided on the exact product
// (p + e, its rounding error e from an FMA), then divided by 100 (the nearest double to k / 100 is what float() of
// the decimal string gives).  Exact for |v| < 2^53 / 100; NaN and infinities pass through.
__device__ __forceinline__ double round2(double v) {
  const double p = __dmul_rn(v, 100.0);
  const double e = __fma_rn(v, 100.0, -p);
  double k = rint(p);
  const double d = __dsub_rn(p, k);
  if (d == 0.5 && e > 0.0) k = __dadd_rn(k, 1.0);
  else if (d == -0.5 && e < 0.0) k = __dsub_rn(k, 1.0);
  return __ddiv_rn(k, 100.0);
}

// np.argsort(-score, kind="mergesort") order on the negated score: NaN after every number, -0.0 == 0.0
__device__ __forceinline__ bool key_less(double a, double b) { return isnan(b) ? !isnan(a) : a < b; }

// np.max((0, v), axis=0): NaN propagates
__device__ __forceinline__ double max0(double v) { return isnan(v) ? v : (v > 0.0 ? v : 0.0); }

// ---- 1. detection prep ----
__global__ void __launch_bounds__(256) prep_kernel(const cpb200_coco_kp_image *__restrict__ images,
                                                   const float *__restrict__ rows, Workspace w) {
  const cpb200_coco_kp_image im = images[blockIdx.x];
  double *score = w.score + im.det_begin;
  for (int i = threadIdx.x; i < im.det_count; i += blockDim.x)
    score[i] = round2((double)rows[(im.det_begin + i) * kRowFloats + 4]);
  __syncthreads();
  for (int i = threadIdx.x; i < im.det_count; i += blockDim.x) {
    const double ki = -score[i];
    int rank = 0;
    for (int j = 0; j < im.det_count && rank < MAXD; ++j) {
      const double kj = -score[j];
      rank += key_less(kj, ki) || (!key_less(ki, kj) && j < i);
    }
    if (rank >= MAXD) continue;
    const float *r = rows + (im.det_begin + i) * kRowFloats;
    Kept &k = w.kept[im.keep_begin + rank];
    for (int j = 0; j < J; ++j) {
      k.x[j] = round2((double)r[5 + 2 * j]);
      k.y[j] = round2((double)r[6 + 2 * j]);
    }
    k.score = score[i];
    // loadRes takes its bbox branch (the results carry a bbox): area = w * h of the formatted [x, y, w, h]
    k.area = __dmul_rn(round2(__dsub_rn((double)r[2], (double)r[0])), round2(__dsub_rn((double)r[3], (double)r[1])));
  }
}

// ---- 2. OKS ----
// np.sum of n <= 17 terms: sequential below 8, else eight running partials combined pairwise, then the rest in order
__device__ __forceinline__ double numpy_sum(const double *a, int n) {
  if (n < 8) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s = __dadd_rn(s, a[i]);
    return s;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  int i = 8;
  for (; i + 8 <= n; i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                       __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) s = __dadd_rn(s, a[i]);
  return s;
}

__global__ void __launch_bounds__(128) oks_kernel(const cpb200_coco_kp_image *__restrict__ images,
                                                  const cpb200_coco_kp_gt *__restrict__ gts,
                                                  const cpb200_coco_kp_params p, const Kept *__restrict__ kept,
                                                  double *__restrict__ oks) {
  const cpb200_coco_kp_image im = images[blockIdx.x];
  const int D = min(im.det_count, MAXD), G = im.gt_count;
  for (int q = threadIdx.x; q < D * G; q += blockDim.x) {
    const Kept &d = kept[im.keep_begin + q / G];
    const cpb200_coco_kp_gt &g = gts[im.gt_begin + q % G];
    const bool any = g.visible != 0;
    const double x0 = __dsub_rn(g.bbox[0], g.bbox[2]), x1 = __dadd_rn(g.bbox[0], __dmul_rn(g.bbox[2], 2.0));
    const double y0 = __dsub_rn(g.bbox[1], g.bbox[3]), y1 = __dadd_rn(g.bbox[1], __dmul_rn(g.bbox[3], 2.0));
    const double den = __dadd_rn(g.area, kSpacing1);
    double t[J];
    int n = 0;
    for (int j = 0; j < J; ++j) {
      double dx, dy;
      if (any) {
        if (!((g.visible >> j) & 1)) continue;
        dx = __dsub_rn(d.x[j], g.x[j]);
        dy = __dsub_rn(d.y[j], g.y[j]);
      } else {                     // no visible joint: the distance to the box three times the ground truth's
        dx = __dadd_rn(max0(__dsub_rn(x0, d.x[j])), max0(__dsub_rn(d.x[j], x1)));
        dy = __dadd_rn(max0(__dsub_rn(y0, d.y[j])), max0(__dsub_rn(d.y[j], y1)));
      }
      const double e = __ddiv_rn(__ddiv_rn(__ddiv_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), p.vars[j]), den), 2.0);
      t[n++] = exp(-e);
    }
    oks[im.oks_offset + q] = __ddiv_rn(numpy_sum(t, n), (double)n);
  }
}

// ---- 3. evaluateImg's match ----
__device__ __forceinline__ int gt_ignored(const cpb200_coco_kp_gt &g, double lo, double hi) {
  return g.ignore || g.area < lo || g.area > hi;
}

__global__ void __launch_bounds__(128) match_kernel(const cpb200_coco_kp_image *__restrict__ images, int n_images,
                                                    const cpb200_coco_kp_gt *__restrict__ gts, int n_gts, int n_keep,
                                                    const cpb200_coco_kp_params p, Workspace w) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)n_images * AT) return;
  const cpb200_coco_kp_image im = images[tid / AT];
  const int at = (int)(tid % AT), a = at / T, t = at % T;
  const double lo = p.area_rng[a][0], hi = p.area_rng[a][1];
  const double thr = fmin(p.iou_thrs[t], 1.0 - 1e-10);
  const int D = min(im.det_count, MAXD), G = im.gt_count;
  const cpb200_coco_kp_gt *g = gts + im.gt_begin;
  unsigned char *gtm = w.gtm + (size_t)at * n_gts + im.gt_begin;
  unsigned char *flags = w.flags + (size_t)at * n_keep + im.keep_begin;
  const double *oks = w.oks + im.oks_offset;
  for (int k = 0; k < G; ++k) gtm[k] = 0;
  for (int d = 0; d < D; ++d) {
    double iou = thr;
    int m = -1;
    // the ground truths stable-sorted by _ignore: the kept ones in file order, then the ignored ones
    for (int pass = 0; pass < 2; ++pass) {
      bool stop = false;
      for (int k = 0; k < G; ++k) {
        const int ig = gt_ignored(g[k], lo, hi);
        if (ig != pass) continue;
        if (gtm[k] && !g[k].iscrowd) continue;
        if (m > -1 && !gt_ignored(g[m], lo, hi) && ig) { stop = true; break; }
        const double v = oks[d * G + k];
        if (v < iou) continue;
        iou = v;
        m = k;
      }
      if (stop) break;
    }
    bool matched = false;
    int ignore = 0;
    if (m != -1) {
      ignore = gt_ignored(g[m], lo, hi);
      matched = g[m].id != 0;
      gtm[m] = 1;
    }
    const double area = w.kept[im.keep_begin + d].area;
    if (!matched && (area < lo || area > hi)) ignore = 1;
    flags[d] = (unsigned char)((matched ? 1 : 0) | (ignore ? 2 : 0));
  }
}

// ---- 4. the stable sort of every kept detection by -score ----
__device__ __forceinline__ unsigned long long score_key(double s) {
  double k = -s;
  if (isnan(k)) return ~0ull;
  if (k == 0.0) k = 0.0;
  const unsigned long long b = (unsigned long long)__double_as_longlong(k);
  return (b >> 63) ? ~b : (b | (1ull << 63));
}

__global__ void sort_init_kernel(const Kept *__restrict__ kept, int n_keep, Workspace w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w.P) return;
  w.keys[i] = i < n_keep ? score_key(kept[i].score) : ~0ull;     // padding after everything, NaN included
  w.order[i] = i < n_keep ? (unsigned)i : 0xffffffffu;
}

__device__ __forceinline__ bool pair_greater(unsigned long long ka, unsigned oa, unsigned long long kb, unsigned ob) {
  return ka > kb || (ka == kb && oa > ob);
}

// one compare-exchange step of stride j in bitonic sequences of length k, across the whole array
__global__ void bitonic_global_kernel(Workspace w, int64_t k, int64_t j) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t l = i ^ j;
  if (i >= w.P || l <= i) return;
  const bool up = (i & k) == 0;
  const unsigned long long ki = w.keys[i], kl = w.keys[l];
  const unsigned oi = w.order[i], ol = w.order[l];
  if (pair_greater(ki, oi, kl, ol) == up) {
    w.keys[i] = kl; w.keys[l] = ki;
    w.order[i] = ol; w.order[l] = oi;
  }
}

// the steps of stride < kSortBlock in shared memory: every k from 2 to k_hi when k_lo == 2, else k_lo alone
__global__ void __launch_bounds__(kScanThreads) bitonic_local_kernel(Workspace w, int64_t k_lo, int64_t k_hi) {
  __shared__ unsigned long long sk[kSortBlock];
  __shared__ unsigned so[kSortBlock];
  const int64_t base = (int64_t)blockIdx.x * kSortBlock;
  for (int i = threadIdx.x; i < kSortBlock; i += blockDim.x) { sk[i] = w.keys[base + i]; so[i] = w.order[base + i]; }
  __syncthreads();
  for (int64_t k = k_lo; k <= k_hi; k <<= 1) {
    for (int j = (int)(k >= kSortBlock ? kSortBlock >> 1 : k >> 1); j > 0; j >>= 1) {
      const int t = threadIdx.x;
      const int i = 2 * t - (t & (j - 1));                   // the lower index of this thread's pair
      const int l = i + j;
      const bool up = ((base + i) & k) == 0;
      if (pair_greater(sk[i], so[i], sk[l], so[l]) == up) {
        const unsigned long long kk = sk[i]; sk[i] = sk[l]; sk[l] = kk;
        const unsigned oo = so[i]; so[i] = so[l]; so[l] = oo;
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < kSortBlock; i += blockDim.x) { w.keys[base + i] = sk[i]; w.order[base + i] = so[i]; }
}

// ---- 5. accumulate ----
// inclusive block scan (sum) of one value per thread; `sh` holds 32 entries
__device__ __forceinline__ unsigned long long block_sum_scan(unsigned long long v, unsigned long long *sh,
                                                             unsigned long long &total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  if (lane == 31) sh[warp] = v;
  __syncthreads();
  if (warp == 0) {
    unsigned long long s = sh[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long n = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += n;
    }
    sh[lane] = s;
  }
  __syncthreads();
  if (warp > 0) v += sh[warp - 1];
  total = sh[31];
  __syncthreads();
  return v;
}

// inclusive block scan (max) of one value per thread
__device__ __forceinline__ double block_max_scan(double v, double *sh, double &total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = fmax(v, n);
  }
  if (lane == 31) sh[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double s = sh[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double n = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s = fmax(s, n);
    }
    sh[lane] = s;
  }
  __syncthreads();
  if (warp > 0) v = fmax(v, sh[warp - 1]);
  total = sh[31];
  __syncthreads();
  return v;
}

__global__ void __launch_bounds__(kScanThreads) accumulate_kernel(const cpb200_coco_kp_image *__restrict__ images,
                                                                  int n_images, const cpb200_coco_kp_gt *__restrict__ gts,
                                                                  int n_keep, const cpb200_coco_kp_params p,
                                                                  Workspace w, double *__restrict__ precision,
                                                                  double *__restrict__ recall,
                                                                  double *__restrict__ scores) {
  __shared__ unsigned long long shu[32];
  __shared__ double shd[32];
  const int at = blockIdx.x, a = at / T, t = at % T;
  const double lo = p.area_rng[a][0], hi = p.area_rng[a][1];
  unsigned long long cnt = 0, npig_u;
  for (int n = threadIdx.x; n < n_images; n += blockDim.x)      // the evaluated images' ground truths only
    for (int k = 0; k < images[n].gt_count; ++k) cnt += !gt_ignored(gts[images[n].gt_begin + k], lo, hi);
  block_sum_scan(cnt, shu, npig_u);
  const int64_t npig = (int64_t)npig_u;
  if (npig == 0) {                 // accumulate skips this range: its entries stay -1
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
      precision[(t * R + r) * A + a] = -1.0;
      scores[(t * R + r) * A + a] = -1.0;
    }
    if (threadIdx.x == 0) recall[t * A + a] = -1.0;
    return;
  }
  const unsigned char *flags = w.flags + (size_t)at * n_keep;
  int *tp = w.tp + (size_t)at * n_keep;
  double *pr = w.pr + (size_t)at * n_keep;
  // cumulative tp and fp counts in score order (tp in the low, fp in the high 32 bits), and the precision
  unsigned long long carry = 0;
  for (int base = 0; base < n_keep; base += kScanThreads) {
    const int i = base + threadIdx.x;
    unsigned long long v = 0;
    if (i < n_keep) {
      const unsigned f = flags[w.order[i]];
      if (!(f & 2)) v = (f & 1) ? 1ull : (1ull << 32);
    }
    unsigned long long total;
    v = block_sum_scan(v, shu, total) + carry;
    carry += total;
    if (i < n_keep) {
      const double tpi = (double)(v & 0xffffffffull), fpi = (double)(v >> 32);
      tp[i] = (int)(v & 0xffffffffull);
      pr[i] = __ddiv_rn(tpi, __dadd_rn(__dadd_rn(fpi, tpi), kSpacing1));
    }
  }
  __syncthreads();
  // the backward running maximum of precision: a prefix maximum over the reversed positions, last chunk first
  double later = -1.0;
  for (int end = n_keep; end > 0; end -= kScanThreads) {
    const int i = end - 1 - threadIdx.x;
    double v = i >= 0 ? pr[i] : -1.0;
    double total;
    v = fmax(block_max_scan(v, shd, total), later);
    later = fmax(later, total);
    if (i >= 0) pr[i] = v;
  }
  __syncthreads();
  const double np = (double)npig;
  if (threadIdx.x == 0) recall[t * A + a] = n_keep ? __ddiv_rn((double)tp[n_keep - 1], np) : 0.0;
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    const double thr = p.rec_thrs[r];
    int lo_i = 0, hi_i = n_keep;                 // first position whose recall tp / npig is >= thr
    while (lo_i < hi_i) {
      const int mid = (lo_i + hi_i) >> 1;
      if (__ddiv_rn((double)tp[mid], np) < thr) lo_i = mid + 1;
      else hi_i = mid;
    }
    const bool in = lo_i < n_keep;               // past the end: accumulate's try / except leaves 0
    precision[(t * R + r) * A + a] = in ? pr[lo_i] : 0.0;
    scores[(t * R + r) * A + a] = in ? w.kept[w.order[lo_i]].score : 0.0;
  }
}

int check_args(const cpb200_coco_kp_image *images, int n_images, const float *rows, int64_t n_rows,
               const cpb200_coco_kp_gt *gts, int n_gts, int n_keep, int64_t n_oks, const cpb200_coco_kp_params *params,
               void *workspace, const char *what) {
  if (!images || n_images < 1 || n_rows < 0 || n_gts < 0 || n_keep < 0 || n_oks < 0 || !params || !workspace ||
      (n_rows > 0 && !rows) || (n_gts > 0 && !gts))
    return cpb::fail(CPB200_ERR_ARG, "%s: bad arguments", what);
  if (n_keep > n_rows || (int64_t)n_keep > (int64_t)MAXD * n_images)
    return cpb::fail(CPB200_ERR_ARG, "%s: %d kept detections for %d images and %lld rows", what, n_keep, n_images,
                     (long long)n_rows);
  return CPB200_OK;
}

int prep_and_oks(const cpb200_coco_kp_image *images, int n_images, const float *rows, const cpb200_coco_kp_gt *gts,
                 const cpb200_coco_kp_params &p, const Workspace &w, double *oks, cudaStream_t s) {
  prep_kernel<<<n_images, 256, 0, s>>>(images, rows, w);
  if (int st = cpb::check_launch("coco_kp prep_kernel")) return st;
  oks_kernel<<<n_images, 128, 0, s>>>(images, gts, p, w.kept, oks);
  return cpb::check_launch("coco_kp oks_kernel");
}

}  // namespace

extern "C" size_t cpb200_coco_kp_eval_workspace_bytes(int n_images, int64_t n_rows, int n_gts, int n_keep,
                                                      int64_t n_oks) {
  (void)n_images;
  size_t total = 0;
  carve(nullptr, std::max<int64_t>(n_rows, 0), std::max(n_gts, 0), std::max(n_keep, 0), std::max<int64_t>(n_oks, 0),
        &total);
  return total;
}

extern "C" int cpb200_coco_kp_oks(const cpb200_coco_kp_image *images, int n_images, const float *rows, int64_t n_rows,
                                  const cpb200_coco_kp_gt *gts, int n_gts, int n_keep, int64_t n_oks,
                                  const cpb200_coco_kp_params *params, double *oks, void *workspace, void *stream) {
  if (int st = check_args(images, n_images, rows, n_rows, gts, n_gts, n_keep, n_oks, params, workspace, "coco_kp_oks"))
    return st;
  if (!oks && n_oks > 0) return cpb::fail(CPB200_ERR_ARG, "coco_kp_oks: no output");
  const Workspace w = carve(workspace, n_rows, n_gts, n_keep, n_oks, nullptr);
  return prep_and_oks(images, n_images, rows, gts, *params, w, oks, static_cast<cudaStream_t>(stream));
}

extern "C" int cpb200_coco_kp_eval(const cpb200_coco_kp_image *images, int n_images, const float *rows, int64_t n_rows,
                                   const cpb200_coco_kp_gt *gts, int n_gts, int n_keep, int64_t n_oks,
                                   const cpb200_coco_kp_params *params, double *precision, double *recall,
                                   double *scores, void *workspace, void *stream) {
  if (int st = check_args(images, n_images, rows, n_rows, gts, n_gts, n_keep, n_oks, params, workspace, "coco_kp_eval"))
    return st;
  if (!precision || !recall || !scores) return cpb::fail(CPB200_ERR_ARG, "coco_kp_eval: no output");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const cpb200_coco_kp_params p = *params;
  const Workspace w = carve(workspace, n_rows, n_gts, n_keep, n_oks, nullptr);
  if (int st = prep_and_oks(images, n_images, rows, gts, p, w, w.oks, s)) return st;
  const int64_t threads = (int64_t)n_images * AT;
  match_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(images, n_images, gts, n_gts, n_keep, p, w);
  if (int st = cpb::check_launch("coco_kp match_kernel")) return st;
  sort_init_kernel<<<(unsigned)((w.P + 255) / 256), 256, 0, s>>>(w.kept, n_keep, w);
  if (int st = cpb::check_launch("coco_kp sort_init_kernel")) return st;
  const unsigned blocks = (unsigned)(w.P / kSortBlock);
  bitonic_local_kernel<<<blocks, kScanThreads, 0, s>>>(w, 2, kSortBlock);
  if (int st = cpb::check_launch("coco_kp bitonic_local_kernel")) return st;
  for (int64_t k = 2 * kSortBlock; k <= w.P; k <<= 1) {
    for (int64_t j = k >> 1; j >= kSortBlock; j >>= 1) {
      bitonic_global_kernel<<<(unsigned)((w.P + 255) / 256), 256, 0, s>>>(w, k, j);
      if (int st = cpb::check_launch("coco_kp bitonic_global_kernel")) return st;
    }
    bitonic_local_kernel<<<blocks, kScanThreads, 0, s>>>(w, k, k);
    if (int st = cpb::check_launch("coco_kp bitonic_local_kernel")) return st;
  }
  accumulate_kernel<<<AT, kScanThreads, 0, s>>>(images, n_images, gts, n_keep, p, w, precision, recall, scores);
  return cpb::check_launch("coco_kp accumulate_kernel");
}

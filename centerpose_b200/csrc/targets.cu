// Multi-pose training targets and MultiPoseLoss for the reference's validation pass (cpb200_multi_pose_targets_batch,
// cpb200_multi_pose_loss_batch, cpb200_gaussian_radius).
//
// The targets are what MultiPoseDataset.__getitem__ returns, bit for bit: for the val split (no augmentation: rot 0,
// no flip, one matrix) and for the train split's augmented draws (cpb200_multi_pose_targets_train_batch).  The file is built with -fmad=false so that no product is contracted into an FMA; the one FMA the
// reference's np.dot performs is written out with __fma_rn.
//
//   targets_kernel  one CTA per (image, object slot): the slot's annotation (the k-th non-crowd one in file order),
//                   its box, radius, centre and joints into the sparse targets, then the CTA stamps the object's
//                   Gaussians into hm and hm_hp with atomic maxima (every draw is a max, so the order is free)
//   focal_kernel    one CTA per (image, heat-map channel): _neg_loss's positive / negative sums and positive count
//   loss_kernel     one warp per image: the regression losses and the weighted total, from the focal partials
//
// The trainer's MultiPoseLoss (cpb200_multi_pose_loss_train_batch / _backward) normalises once over the batch:
//   train_loss_kernel        one CTA: focal_kernel's partials of every image combined, the regression losses with
//                            batch-wide mask counts, the stats, the loss and the normalisers the backward reads
//   loss_grad_dense_kernel   d loss / d logit of hm and hm_hp, the regression gradients zero-filled
//   loss_grad_sparse_kernel  one CTA per (regression term, image): the gathered entries' gradients, as counts of c
#include <algorithm>

#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_val_image) == 64, "cpb200_val_image layout is part of the C ABI");
static_assert(sizeof(cpb200_train_image) == 240, "cpb200_train_image layout is part of the C ABI");
static_assert(sizeof(cpb200_coco_kp_gt) == 336, "cpb200_coco_kp_gt layout is part of the C ABI");

constexpr int J = CPB200_COCO_KP_JOINTS;
constexpr int M = CPB200_MAX_OBJS;
constexpr int kStampThreads = 256;

// gaussian_radius((h, w), min_overlap=0.7) of lib/utils/image.py in double, left to right as Python evaluates it
// (the file has no FMA contraction): (1 - 0.7) is 0.30000000000000004, 4 * 0.7 is 2.8, -2 * 0.7 is -1.4
__device__ __host__ inline double gaussian_radius(int height, int width) {
  const double mo = 0.7, omo = 1.0 - 0.7, hw = (double)(height + width), wh = (double)width * (double)height;
  const double c1 = wh * omo / (1.0 + mo);
  const double r1 = (hw + sqrt(hw * hw - 4.0 * c1)) / 2.0;
  const double b2 = 2.0 * hw, c2 = omo * (double)width * (double)height;
  const double r2 = (b2 + sqrt(b2 * b2 - 16.0 * c2)) / 2.0;
  const double a3 = 4.0 * mo, b3 = -2.0 * mo * hw, c3 = (mo - 1.0) * (double)width * (double)height;
  const double r3 = (b3 + sqrt(b3 * b3 - 4.0 * a3 * c3)) / 2.0;
  return fmin(r1, fmin(r2, r3));
}

__device__ inline int radius_of(int height, int width) {
  const double r = gaussian_radius(height, width);
  return r > 0 ? (int)r : 0;                      // max(0, int(r)): int() truncates toward zero
}

// affine_transform(pt, t): np.dot(t, float32([x, y, 1])) in float64, rounded to float32 where it is stored
__device__ inline float affine_x(const double *t, float x, float y) {
  return (float)__dadd_rn(__fma_rn(t[0], (double)x, __dmul_rn(t[1], (double)y)), t[2]);
}

// float32(gaussian2D((2r+1, 2r+1), sigma=(2r+1)/6)[r + dy, r + dx]); the reference's eps * max cut never fires
__device__ inline float gauss(int dx, int dy, double sigma) {
  const double e = -(double)(dx * dx + dy * dy) / (2.0 * sigma * sigma);
  return (float)exp(e);
}

struct Stamp {
  int x, y, r;
  int map;                           // -1: hm, else the hm_hp channel
};

// What the targets kernel reads of one image.  The val split's entry is the case without flip or rotation whose
// joints go through the box matrix.
struct ImageView {
  int gt_begin, gt_count, flip, rot;
  float width;                       // the image width, for the flip
  const double *t, *t_rot;           // trans_output (boxes) and trans_output_rot (joints)
};

__device__ inline ImageView view(const cpb200_val_image &e) {
  return ImageView{e.gt_begin, e.gt_count, 0, 0, 0.f, e.trans_output, e.trans_output};
}

__device__ inline ImageView view(const cpb200_train_image &e) {
  return ImageView{e.gt_begin, e.gt_count, e.flip, e.rot, (float)e.w, e.trans_output, e.trans_output_rot};
}

// the dataset's flip_idx pairs (1, 2), (3, 4), ..., (15, 16): after a flip joint j holds the annotation's joint
__device__ inline int flip_partner(int j) { return j == 0 ? 0 : (j & 1 ? j + 1 : j - 1); }

template <typename Image>
struct TargetArgs {
  const Image *images;
  const cpb200_coco_kp_gt *gts;
  cpb200_multi_pose_targets out;
  int R;
};

template <typename Image>
__global__ void __launch_bounds__(kStampThreads) targets_kernel(const TargetArgs<Image> a) {
  const int k = blockIdx.x, b = blockIdx.y, R = a.R;
  const Image e = a.images[b];
  const ImageView im = view(e);
  __shared__ int s_ann, s_n;
  __shared__ Stamp s_st[1 + J];
  // rot != 0: hm = hm * 0 + 0.9999 after every object, so no object stamps it and slot 0's CTA fills it
  if (im.rot && k == 0)
    for (int i = threadIdx.x; i < R * R; i += blockDim.x) a.out.hm[(size_t)b * R * R + i] = 0.9999f;
  // the k-th annotation with iscrowd != 1, in file order (warp 0 counts with ballots)
  if (threadIdx.x < 32) {
    int seen = 0, found = -1;
    for (int base = 0; base < im.gt_count && found < 0; base += 32) {
      const int i = base + (int)threadIdx.x;
      const bool keep = i < im.gt_count && a.gts[im.gt_begin + i].iscrowd != 1;
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      const int n = __popc(m);
      if (seen + n > k) {
        unsigned mm = m;
        for (int q = 0; q < k - seen; ++q) mm &= mm - 1;     // drop the set bits below the one wanted
        found = base + __ffs(mm) - 1;
      }
      seen += n;
    }
    if (threadIdx.x == 0) { s_ann = found; s_n = 0; }
  }
  __syncthreads();
  if (s_ann < 0) return;
  if (threadIdx.x == 0) {
    const cpb200_coco_kp_gt &g = a.gts[im.gt_begin + s_ann];
    const double *t = im.t;
    const float hi = (float)(R - 1);
    // float32([x, y, x + w, y + h]); flipped: bbox[[0, 2]] = width - bbox[[2, 0]] - 1 in float32; corners through
    // trans_output, clipped to [0, R - 1]
    float bb[4] = {(float)g.bbox[0], (float)g.bbox[1], (float)(g.bbox[0] + g.bbox[2]), (float)(g.bbox[1] + g.bbox[3])};
    if (im.flip) {
      const float x0 = bb[0];
      bb[0] = __fsub_rn(__fsub_rn(im.width, bb[2]), 1.f);
      bb[2] = __fsub_rn(__fsub_rn(im.width, x0), 1.f);
    }
    for (int c = 0; c < 4; c += 2) {
      const float x = bb[c], y = bb[c + 1];
      bb[c] = affine_x(t, x, y);
      bb[c + 1] = affine_x(t + 3, x, y);
    }
    for (int c = 0; c < 4; ++c) bb[c] = fminf(fmaxf(bb[c], 0.f), hi);
    const float h = __fsub_rn(bb[3], bb[1]), w = __fsub_rn(bb[2], bb[0]);
    // with rot != 0 every object is drawn, a degenerate box too (its radius is 0)
    if ((h > 0 && w > 0) || im.rot) {
      const int r = radius_of((int)ceilf(h), (int)ceilf(w));
      const float cx = __fdiv_rn(__fadd_rn(bb[0], bb[2]), 2.f), cy = __fdiv_rn(__fadd_rn(bb[1], bb[3]), 2.f);
      const int ix = (int)cx, iy = (int)cy;
      const size_t o = (size_t)b * M + k;
      a.out.wh[2 * o] = w;
      a.out.wh[2 * o + 1] = h;
      a.out.ind[o] = (int64_t)iy * R + ix;
      a.out.reg[2 * o] = __fsub_rn(cx, (float)ix);
      a.out.reg[2 * o + 1] = __fsub_rn(cy, (float)iy);
      // num_kpts == 0: reg_mask 0, and hm[ct] = 0.9999, which this object's own stamp (1.0 at ct) always overwrites;
      // rot != 0 zeroes reg_mask and hps_mask afterwards
      a.out.reg_mask[o] = g.visible != 0 && !im.rot;
      int n = 0;
      if (!im.rot) s_st[n++] = Stamp{ix, iy, r, -1};
      const double *tr = im.t_rot;
      for (int j = 0; j < J; ++j) {
        // flipped: pts[:, 0] = width - pts[:, 0] - 1 in float32, then the flip_idx rows (v included) swap
        const int src = im.flip ? flip_partner(j) : j;
        if (!((g.visible >> src) & 1)) continue;
        float x = (float)g.x[src];
        const float y = (float)g.y[src];
        if (im.flip) x = __fsub_rn(__fsub_rn(im.width, x), 1.f);
        const float px = affine_x(tr, x, y), py = affine_x(tr + 3, x, y);
        if (!(px >= 0 && px < (float)R && py >= 0 && py < (float)R)) continue;
        const int qx = (int)px, qy = (int)py;
        const size_t p = o * J + j;
        a.out.hps[2 * p] = __fsub_rn(px, (float)ix);
        a.out.hps[2 * p + 1] = __fsub_rn(py, (float)iy);
        a.out.hps_mask[2 * p] = a.out.hps_mask[2 * p + 1] = !im.rot;
        a.out.hp_offset[2 * p] = __fsub_rn(px, (float)qx);
        a.out.hp_offset[2 * p + 1] = __fsub_rn(py, (float)qy);
        a.out.hp_ind[p] = (int64_t)qy * R + qx;
        a.out.hp_mask[p] = 1;
        s_st[n++] = Stamp{qx, qy, r, j};
      }
      s_n = n;
    }
  }
  __syncthreads();
  // draw_umich_gaussian: the window [x - min(x, r), x + min(R - x, r + 1)) x [same in y]; values are >= 0, so their
  // float bit patterns order as ints and atomicMax on them is np.maximum
  for (int s = 0; s < s_n; ++s) {
    const Stamp st = s_st[s];
    const int x0 = st.x - min(st.x, st.r), x1 = st.x + min(R - st.x, st.r + 1);
    const int y0 = st.y - min(st.y, st.r), y1 = st.y + min(R - st.y, st.r + 1);
    const int W = x1 - x0, n = W * (y1 - y0);
    const double sigma = (double)(2 * st.r + 1) / 6.0;
    float *map = st.map < 0 ? a.out.hm + (size_t)b * R * R : a.out.hm_hp + ((size_t)b * J + st.map) * R * R;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int x = x0 + i % W, y = y0 + i / W;
      atomicMax(reinterpret_cast<int *>(map + (size_t)y * R + x), __float_as_int(gauss(x - st.x, y - st.y, sigma)));
    }
  }
}

__global__ void radius_kernel(const int *hw, int n, int *radius) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) radius[i] = radius_of(hw[2 * i], hw[2 * i + 1]);
}

// ---- MultiPoseLoss ----

// _sigmoid then _neg_loss's two terms for one element, in float32 and in the order torch evaluates them; both terms are
// taken and multiplied by their indicator, so a non-finite logit poisons both sums as it does in the reference
struct Focal { double pos, neg, npos; };

__device__ inline void focal_term(float logit, float gt, Focal &f) {
  float p = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-logit)));
  p = p != p ? p : fminf(fmaxf(p, 1e-4f), 0.9999f);          // torch.clamp keeps NaN
  const float pi = gt == 1.f ? 1.f : 0.f, ni = gt < 1.f ? 1.f : 0.f;
  const float q = __fsub_rn(1.f, p), w = __fsub_rn(1.f, gt), w2 = __fmul_rn(w, w);
  f.pos += (double)__fmul_rn(__fmul_rn(logf(p), __fmul_rn(q, q)), pi);
  f.neg += (double)__fmul_rn(__fmul_rn(__fmul_rn(logf(q), __fmul_rn(p, p)), __fmul_rn(w2, w2)), ni);
  f.npos += (double)pi;
}

__device__ inline double block_sum(double v, double *red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0;
  if (threadIdx.x == 0)
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  return s;
}

// grid (1 + J, B): channel 0 is hm, 1..J the hm_hp channels; partial[(b * (1 + J) + c) * 3 + {pos, neg, npos}]
__global__ void __launch_bounds__(256) focal_kernel(const float *hm, const float *hm_hp, const float *t_hm,
                                                    const float *t_hm_hp, int R, double *partial) {
  const int c = blockIdx.x, b = blockIdx.y, n = R * R;
  const float *x = c == 0 ? hm + (size_t)b * n : hm_hp + ((size_t)b * J + c - 1) * n;
  const float *g = c == 0 ? t_hm + (size_t)b * n : t_hm_hp + ((size_t)b * J + c - 1) * n;
  Focal f = {0, 0, 0};
  for (int i = threadIdx.x; i < n; i += blockDim.x) focal_term(x[i], g[i], f);
  __shared__ double red[8];
  double *out = partial + ((size_t)b * (1 + J) + c) * 3;
  const double pos = block_sum(f.pos, red), neg = block_sum(f.neg, red), npos = block_sum(f.npos, red);
  if (threadIdx.x == 0) { out[0] = pos; out[1] = neg; out[2] = npos; }
}

// _neg_loss's sums over `images` images (partials (1 + J) channels apart) x `channels` channels, image by image and
// channel by channel; p points at the first image's first channel
__device__ inline Focal focal_sum(const double *p, int images, int channels) {
  Focal f = {0, 0, 0};
  for (int b = 0; b < images; ++b)
    for (int c = 0; c < channels; ++c) {
      const double *q = p + 3 * ((size_t)b * (1 + J) + c);
      f.pos += q[0]; f.neg += q[1]; f.npos += q[2];
    }
  return f;
}

__device__ inline float focal_value(const Focal &f) {
  return (float)(f.npos == 0 ? -f.neg : -(f.pos + f.neg) / f.npos);
}

// sum |pred * m - t * m| and sum(m) (RegL1Loss, RegWeightedL1Loss) over `images` images of `n` entries of `dim`
// values, pred gathered at ind: this thread's share, entries first, first + step, ... in float64
struct L1Sum { double s, cnt; };

template <typename MaskT>
__device__ inline L1Sum l1_part(const float *map, int R, const int64_t *ind, const MaskT *mask, bool per_value,
                                const float *t, int n, int dim, int images, int first, int step) {
  L1Sum a = {0, 0};
  const size_t plane = (size_t)R * R;
  for (int i = first; i < images * n * dim; i += step) {
    const int b = i / (n * dim), c = i % dim;
    const float m = per_value ? (float)mask[i] : (float)mask[i / dim];
    const float pr = map[((size_t)b * dim + c) * plane + ind[i / dim]];
    a.s += (double)fabsf(__fsub_rn(__fmul_rn(pr, m), __fmul_rn(t[i], m)));
    a.cnt += m;
  }
  return a;
}

__device__ inline L1Sum warp_l1_sum(L1Sum a) {
  for (int o = 16; o > 0; o >>= 1) {
    a.s += __shfl_xor_sync(0xffffffffu, a.s, o);
    a.cnt += __shfl_xor_sync(0xffffffffu, a.cnt, o);
  }
  return a;
}

// the mask count + 1e-4 in float32 as torch adds it
__device__ inline float l1_den(const L1Sum &a) { return __fadd_rn((float)a.cnt, 1e-4f); }
__device__ inline float l1_value(const L1Sum &a) { return (float)(a.s / (double)l1_den(a)); }

// one image's loss, summed by its warp
template <typename MaskT>
__device__ inline float l1_loss(const float *map, int R, const int64_t *ind, const MaskT *mask, bool per_value,
                                const float *t, int n, int dim) {
  return l1_value(warp_l1_sum(l1_part(map, R, ind, mask, per_value, t, n, dim, 1, threadIdx.x & 31, 32)));
}

// loss = HM_WEIGHT * hm + WH_WEIGHT * wh + OFF_WEIGHT * off + HP_WEIGHT * hp + HM_HP_WEIGHT * hm_hp
//        + OFF_WEIGHT * hp_offset, in float32, left to right; o receives the seven stats in CPB200_LOSS_STATS order
__device__ inline void write_stats(const cpb200_multi_pose_loss_cfg &c, float hm_loss, float wh_loss, float off_loss,
                                   float hp_loss, float hm_hp_loss, float hp_offset_loss, float *o) {
  float loss = __fmul_rn(c.hm_weight, hm_loss);
  loss = __fadd_rn(loss, __fmul_rn(c.wh_weight, wh_loss));
  loss = __fadd_rn(loss, __fmul_rn(c.off_weight, off_loss));
  loss = __fadd_rn(loss, __fmul_rn(c.hp_weight, hp_loss));
  loss = __fadd_rn(loss, __fmul_rn(c.hm_hp_weight, hm_hp_loss));
  loss = __fadd_rn(loss, __fmul_rn(c.off_weight, hp_offset_loss));
  o[0] = loss; o[1] = hm_loss; o[2] = hp_loss; o[3] = hm_hp_loss; o[4] = hp_offset_loss; o[5] = wh_loss;
  o[6] = off_loss;
}

// which of MultiPoseLoss's terms the LOSS gates keep
struct Gates {
  bool wh, off, hp_offset, hm_hp;
};

__host__ __device__ inline Gates gates(const cpb200_multi_pose_loss_cfg &c) {
  return Gates{c.wh_weight > 0, c.reg_offset && c.off_weight > 0, c.reg_hp_offset && c.off_weight > 0,
               c.hm_hp && c.hm_hp_weight > 0};
}

struct LossArgs {
  cpb200_multi_pose_heads heads;
  cpb200_multi_pose_targets t;
  int B, R;
  cpb200_multi_pose_loss_cfg cfg;
  const double *partial;
  float *stats;
};

__global__ void loss_kernel(const LossArgs a) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= a.B) return;
  const int R = a.R;
  const size_t plane = (size_t)R * R;
  const cpb200_multi_pose_loss_cfg &c = a.cfg;
  const double *p = a.partial + (size_t)b * (1 + J) * 3;
  const int64_t *ind = a.t.ind + (size_t)b * M;
  const unsigned char *reg_mask = a.t.reg_mask + (size_t)b * M;
  const Gates g = gates(c);
  const float hm_loss = focal_value(focal_sum(p, 1, 1));
  const float hp_loss = l1_loss(a.heads.hps + (size_t)b * 2 * J * plane, R, ind, a.t.hps_mask + (size_t)b * M * 2 * J,
                                true, a.t.hps + (size_t)b * M * 2 * J, M, 2 * J);
  float wh_loss = 0, off_loss = 0, hp_offset_loss = 0, hm_hp_loss = 0;
  if (g.wh)
    wh_loss = l1_loss(a.heads.wh + (size_t)b * 2 * plane, R, ind, reg_mask, false, a.t.wh + (size_t)b * M * 2, M, 2);
  if (g.off)
    off_loss = l1_loss(a.heads.reg + (size_t)b * 2 * plane, R, ind, reg_mask, false, a.t.reg + (size_t)b * M * 2, M, 2);
  if (g.hp_offset)
    hp_offset_loss = l1_loss(a.heads.hp_offset + (size_t)b * 2 * plane, R, a.t.hp_ind + (size_t)b * M * J,
                             a.t.hp_mask + (size_t)b * M * J, false, a.t.hp_offset + (size_t)b * M * J * 2, M * J, 2);
  if (g.hm_hp) hm_hp_loss = focal_value(focal_sum(p + 3, 1, J));
  float o[CPB200_LOSS_STATS];
  write_stats(c, hm_loss, wh_loss, off_loss, hp_loss, hm_hp_loss, hp_offset_loss, o);
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < CPB200_LOSS_STATS; ++i) a.stats[(size_t)b * CPB200_LOSS_STATS + i] = o[i];
}

// ---- MultiPoseLoss over the whole batch, and its gradient (the trainer's loss) ----

// what the forward leaves in the workspace after the focal partials for the backward
enum Norm { kNposHm, kNposHmHp, kDenHps, kDenWh, kDenReg, kDenHpOffset, kNorms };
constexpr int kTrainThreads = 1024;

struct TrainLossArgs {
  cpb200_multi_pose_heads heads;
  cpb200_multi_pose_targets t;
  int B, R;
  cpb200_multi_pose_loss_cfg cfg;
  const double *partial;
  float *stats, *loss, *norm;
};

// one regression term over the batch, summed by the whole CTA: per-thread shares, warp sums, then the warps in order
template <typename MaskT>
__device__ inline L1Sum block_l1(const float *map, int R, const int64_t *ind, const MaskT *mask, bool per_value,
                                 const float *t, int n, int dim, int images, L1Sum *red) {
  L1Sum a = warp_l1_sum(l1_part(map, R, ind, mask, per_value, t, n, dim, images, threadIdx.x, blockDim.x));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  L1Sum s = {0, 0};
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { s.s += red[w].s; s.cnt += red[w].cnt; }
  return s;
}

// one CTA: _neg_loss normalised once over the batch (the partials of every image and channel, in a fixed order) and
// the regression losses with batch-wide mask counts
__global__ void __launch_bounds__(kTrainThreads) train_loss_kernel(const TrainLossArgs a) {
  __shared__ L1Sum red[kTrainThreads / 32];
  const cpb200_multi_pose_loss_cfg &c = a.cfg;
  const Gates g = gates(c);
  const int B = a.B, R = a.R;
  const L1Sum hp = block_l1(a.heads.hps, R, a.t.ind, a.t.hps_mask, true, a.t.hps, M, 2 * J, B, red);
  L1Sum wh = {0, 0}, off = {0, 0}, hp_offset = {0, 0};
  if (g.wh) wh = block_l1(a.heads.wh, R, a.t.ind, a.t.reg_mask, false, a.t.wh, M, 2, B, red);
  if (g.off) off = block_l1(a.heads.reg, R, a.t.ind, a.t.reg_mask, false, a.t.reg, M, 2, B, red);
  if (g.hp_offset)
    hp_offset = block_l1(a.heads.hp_offset, R, a.t.hp_ind, a.t.hp_mask, false, a.t.hp_offset, M * J, 2, B, red);
  if (threadIdx.x != 0) return;
  const Focal fh = focal_sum(a.partial, B, 1);
  const Focal fp = g.hm_hp ? focal_sum(a.partial + 3, B, J) : Focal{0, 0, 0};
  float o[CPB200_LOSS_STATS];
  write_stats(c, focal_value(fh), g.wh ? l1_value(wh) : 0.f, g.off ? l1_value(off) : 0.f, l1_value(hp),
              g.hm_hp ? focal_value(fp) : 0.f, g.hp_offset ? l1_value(hp_offset) : 0.f, o);
  for (int i = 0; i < CPB200_LOSS_STATS; ++i) a.stats[i] = o[i];
  *a.loss = o[0];
  a.norm[kNposHm] = (float)fh.npos;                 // pos_inds.sum() in float32: exact below 2^24
  a.norm[kNposHmHp] = (float)fp.npos;
  a.norm[kDenHps] = l1_den(hp);
  a.norm[kDenWh] = l1_den(wh);
  a.norm[kDenReg] = l1_den(off);
  a.norm[kDenHpOffset] = l1_den(hp_offset);
}

// d loss / d logit of one hm or hm_hp element, in the order torch's autograd evaluates _sigmoid and _neg_loss's
// backward: g is the gradient of each summed term (-(grad_loss * weight) / num_pos, or -(grad_loss * weight) with no
// positive, when the positive term is not in the graph at all)
__device__ inline float focal_grad(float x, float gt, float g, bool pos_term) {
  const float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
  const float p = s != s ? s : fminf(fmaxf(s, 1e-4f), 0.9999f);
  const float pi = gt == 1.f ? 1.f : 0.f, ni = gt < 1.f ? 1.f : 0.f;
  const float q = __fsub_rn(1.f, p), w = __fsub_rn(1.f, gt), w2 = __fmul_rn(w, w);
  // log(1 - p) * p^2 * (1 - gt)^4 * neg_inds: mul's backward scales by the indicator first, then by the weight
  const float h = __fmul_rn(__fmul_rn(g, ni), __fmul_rn(w2, w2));
  float d = __fadd_rn(-__fdiv_rn(__fmul_rn(h, __fmul_rn(p, p)), q), __fmul_rn(__fmul_rn(h, logf(q)), __fmul_rn(2.f, p)));
  if (pos_term) {
    // log(p) * (1 - p)^2 * pos_inds
    const float gp = __fmul_rn(g, pi);
    const float pos = __fadd_rn(__fdiv_rn(__fmul_rn(gp, __fmul_rn(q, q)), p),
                                -__fmul_rn(__fmul_rn(gp, logf(p)), __fmul_rn(2.f, q)));
    d = __fadd_rn(pos, d);
  }
  // clamp passes the gradient where the logistic lies within its bounds, bounds included; then the logistic's own
  const float ds = s >= 1e-4f && s <= 0.9999f ? d : 0.f;
  return __fmul_rn(__fmul_rn(ds, __fsub_rn(1.f, s)), s);
}

struct DenseArgs {
  const float *x[2], *gt[2];       // hm, hm_hp logits and targets
  float *grad[2];                  // their gradients (grad[1] NULL: hm_hp is not in the loss)
  float *zero[4];                  // the regression gradients, zero-filled for the sparse kernel (NULL: skipped)
  size_t n[2], n_zero[4];
  float weight[2];
  const float *grad_loss, *norm;
};

// grid-stride over blockIdx.y's map: 0 hm, 1 hm_hp, 2.. the four regression maps
__global__ void __launch_bounds__(256) loss_grad_dense_kernel(const DenseArgs a) {
  const int m = blockIdx.y;
  const size_t step = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= 2) {
    float *z = a.zero[m - 2];
    if (z)
      for (; i < a.n_zero[m - 2]; i += step) z[i] = 0.f;
    return;
  }
  if (!a.grad[m]) return;
  const float npos = a.norm[m == 0 ? kNposHm : kNposHmHp];
  const float G = -__fmul_rn(*a.grad_loss, a.weight[m]);
  const float g = npos == 0.f ? G : __fdiv_rn(G, npos);
  const float *x = a.x[m], *gt = a.gt[m];
  float *out = a.grad[m];
  for (; i < a.n[m]; i += step) out[i] = focal_grad(x[i], gt[i], g, npos != 0.f);
}

struct SparseTerm {
  const float *map, *t;            // head map (B, dim, R, R) and target (B, n, dim)
  const int64_t *ind;              // (B, n)
  const void *mask;                // (B, n) or (B, n, dim) per mask_kind
  float *grad;                     // (B, dim, R, R), zero-filled; NULL: the term is not in the loss
  float weight;
  int n, dim, mask_kind, den;      // mask_kind 0: uint8 per slot, 1: uint8 per value, 2: int64 per slot
};

struct SparseArgs {
  SparseTerm term[4];
  int R;
  const float *grad_loss, *norm;
};

constexpr int kSparseEntries = M * J * 2;          // the largest term: hp_offset's M * J slots of 2 values

// grid (4 terms, B): every entry adds sign(pred * m - t * m) * m * c into (channel, ind) of its map, with
// c = grad_loss * weight / (sum(m) + 1e-4).  Each pixel's contributions are whole multiples of c, so the entry with
// the smallest slot among those that reach a pixel counts them and writes count * c: one rounding, no atomics, the
// same bits on every run.  Entries with m == 0 add 0 and leave the zero fill in place.
__global__ void __launch_bounds__(256) loss_grad_sparse_kernel(const SparseArgs a) {
  const SparseTerm tm = a.term[blockIdx.x];
  if (!tm.grad) return;
  const int b = blockIdx.y, n = tm.n, dim = tm.dim, R = a.R;
  const size_t plane = (size_t)R * R;
  __shared__ int64_t s_ind[M * J];
  __shared__ int s_q[kSparseEntries];              // sign * m of every entry
  for (int k = threadIdx.x; k < n; k += blockDim.x) s_ind[k] = tm.ind[(size_t)b * n + k];
  __syncthreads();
  for (int e = threadIdx.x; e < n * dim; e += blockDim.x) {
    const int k = e / dim, c = e % dim;
    const size_t i = (size_t)b * n * dim + e;
    const int m = tm.mask_kind == 0   ? ((const unsigned char *)tm.mask)[(size_t)b * n + k]
                  : tm.mask_kind == 1 ? ((const unsigned char *)tm.mask)[i]
                                      : (int)((const int64_t *)tm.mask)[(size_t)b * n + k];
    const float fm = (float)m;
    const float pr = tm.map[((size_t)b * dim + c) * plane + s_ind[k]];
    const float d = __fsub_rn(__fmul_rn(pr, fm), __fmul_rn(tm.t[i], fm));
    s_q[e] = m == 0 ? 0 : (d > 0.f ? m : d < 0.f ? -m : 0);     // torch's sign: 0 for 0 and NaN
  }
  __syncthreads();
  const float cst = __fdiv_rn(__fmul_rn(*a.grad_loss, tm.weight), a.norm[tm.den]);
  for (int e = threadIdx.x; e < n * dim; e += blockDim.x) {
    const int k = e / dim, c = e % dim;
    if (s_q[e] == 0) continue;
    const int64_t px = s_ind[k];
    bool first = true;
    for (int j = 0; j < k && first; ++j) first = !(s_ind[j] == px && s_q[j * dim + c] != 0);
    if (!first) continue;
    int count = 0;
    for (int j = k; j < n; ++j) count += s_ind[j] == px ? s_q[j * dim + c] : 0;
    // + 0 turns a -0 into the +0 that adding to torch's zero-filled gradient leaves
    tm.grad[((size_t)b * dim + c) * plane + px] = __fadd_rn(__fmul_rn((float)count, cst), 0.f);
  }
}

bool targets_complete(const cpb200_multi_pose_targets &t) {
  return t.hm && t.hm_hp && t.wh && t.reg && t.ind && t.reg_mask && t.hps && t.hps_mask && t.hp_offset && t.hp_ind &&
         t.hp_mask;
}

template <typename Image>
int targets_launch(const Image *images, int B, const cpb200_coco_kp_gt *gts, int R, cpb200_multi_pose_targets out,
                   void *stream, const char *what) {
  if (!images || B < 1 || !gts || R < 1 || !targets_complete(out)) return cpb::fail(CPB200_ERR_ARG, "%s: bad arguments", what);
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "%s: B = %d images exceed one launch", what, B);
  if ((long long)R * R * J >= (1LL << 31)) return cpb::fail(CPB200_ERR_ARG, "%s: R = %d too large", what, R);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t plane = (size_t)R * R, bm = (size_t)B * M;
  // the reference's np.zeros: every slot and pixel no object writes stays 0
  CPB_CUDA(cudaMemsetAsync(out.hm, 0, sizeof(float) * B * plane, s));
  CPB_CUDA(cudaMemsetAsync(out.hm_hp, 0, sizeof(float) * B * J * plane, s));
  CPB_CUDA(cudaMemsetAsync(out.wh, 0, sizeof(float) * bm * 2, s));
  CPB_CUDA(cudaMemsetAsync(out.reg, 0, sizeof(float) * bm * 2, s));
  CPB_CUDA(cudaMemsetAsync(out.ind, 0, sizeof(int64_t) * bm, s));
  CPB_CUDA(cudaMemsetAsync(out.reg_mask, 0, bm, s));
  CPB_CUDA(cudaMemsetAsync(out.hps, 0, sizeof(float) * bm * 2 * J, s));
  CPB_CUDA(cudaMemsetAsync(out.hps_mask, 0, bm * 2 * J, s));
  CPB_CUDA(cudaMemsetAsync(out.hp_offset, 0, sizeof(float) * bm * J * 2, s));
  CPB_CUDA(cudaMemsetAsync(out.hp_ind, 0, sizeof(int64_t) * bm * J, s));
  CPB_CUDA(cudaMemsetAsync(out.hp_mask, 0, sizeof(int64_t) * bm * J, s));
  TargetArgs<Image> a = {images, gts, out, R};
  targets_kernel<Image><<<dim3(M, (unsigned)B), kStampThreads, 0, s>>>(a);
  return cpb::check_launch("targets_kernel");
}

}  // namespace

extern "C" int cpb200_multi_pose_targets_batch(const cpb200_val_image *images, int B, const cpb200_coco_kp_gt *gts,
                                               int R, cpb200_multi_pose_targets out, void *stream) {
  return targets_launch(images, B, gts, R, out, stream, "multi_pose_targets_batch");
}

extern "C" int cpb200_multi_pose_targets_train_batch(const cpb200_train_image *images, int B,
                                                     const cpb200_coco_kp_gt *gts, int R,
                                                     cpb200_multi_pose_targets out, void *stream) {
  return targets_launch(images, B, gts, R, out, stream, "multi_pose_targets_train_batch");
}

extern "C" size_t cpb200_multi_pose_loss_workspace_bytes(int B) {
  return sizeof(double) * 3 * (1 + J) * (size_t)(B > 0 ? B : 0);
}

extern "C" int cpb200_multi_pose_loss_batch(cpb200_multi_pose_heads heads, cpb200_multi_pose_targets targets, int B,
                                            int R, const cpb200_multi_pose_loss_cfg *cfg, float *stats,
                                            void *workspace, void *stream) {
  if (!heads.hm || !heads.wh || !heads.hps || !heads.reg || !heads.hm_hp || !heads.hp_offset ||
      !targets_complete(targets) || B < 1 || R < 1 || !cfg || !stats || !workspace)
    return cpb::fail(CPB200_ERR_ARG, "multi_pose_loss_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "multi_pose_loss_batch: B = %d images exceed one launch", B);
  if ((long long)R * R * 2 * J >= (1LL << 31)) return cpb::fail(CPB200_ERR_ARG, "multi_pose_loss_batch: R = %d too large", R);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  double *partial = static_cast<double *>(workspace);
  focal_kernel<<<dim3(1 + J, (unsigned)B), 256, 0, s>>>(heads.hm, heads.hm_hp, targets.hm, targets.hm_hp, R, partial);
  if (int st = cpb::check_launch("focal_kernel")) return st;
  LossArgs a = {heads, targets, B, R, *cfg, partial, stats};
  loss_kernel<<<(unsigned)((B + 3) / 4), 128, 0, s>>>(a);
  return cpb::check_launch("loss_kernel");
}

extern "C" int cpb200_gaussian_radius(const int *hw, int n, int *radius, void *stream) {
  if (!hw || !radius || n < 0) return cpb::fail(CPB200_ERR_ARG, "gaussian_radius: bad arguments");
  if (n == 0) return CPB200_OK;
  radius_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(hw, n, radius);
  return cpb::check_launch("radius_kernel");
}

namespace {

// the targets and heads the gated loss reads, and the size limits of one launch
int train_loss_check(const cpb200_multi_pose_heads &h, const cpb200_multi_pose_targets &t, int B, int R,
                     const cpb200_multi_pose_loss_cfg *cfg, const char *what) {
  if (!cfg || B < 1 || R < 1) return cpb::fail(CPB200_ERR_ARG, "%s: bad arguments", what);
  const Gates g = gates(*cfg);
  if (!h.hm || !h.hps || (g.wh && !h.wh) || (g.off && !h.reg) || (g.hm_hp && !h.hm_hp) ||
      (g.hp_offset && !h.hp_offset))
    return cpb::fail(CPB200_ERR_ARG, "%s: a head map the loss reads is NULL", what);
  if (!t.hm || !t.wh || !t.ind || !t.reg_mask || !t.hps || !t.hps_mask || (cfg->reg_offset && !t.reg) ||
      (cfg->hm_hp && !t.hm_hp) || (cfg->reg_hp_offset && (!t.hp_offset || !t.hp_ind || !t.hp_mask)))
    return cpb::fail(CPB200_ERR_ARG, "%s: a target the LOSS settings keep is NULL", what);
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "%s: B = %d images exceed one launch", what, B);
  if ((long long)B * M * J * 2 >= (1LL << 31) || (long long)R * R * 2 * J >= (1LL << 31))
    return cpb::fail(CPB200_ERR_ARG, "%s: B = %d, R = %d too large", what, B, R);
  return CPB200_OK;
}

size_t partial_doubles(int B) { return (size_t)3 * (1 + J) * (size_t)B; }

}  // namespace

extern "C" size_t cpb200_multi_pose_loss_train_workspace_bytes(int B) {
  return B > 0 ? sizeof(double) * partial_doubles(B) + sizeof(float) * kNorms : 0;
}

extern "C" int cpb200_multi_pose_loss_train_batch(cpb200_multi_pose_heads heads, cpb200_multi_pose_targets targets,
                                                  int B, int R, const cpb200_multi_pose_loss_cfg *cfg, float *stats,
                                                  float *loss, void *workspace, void *stream) {
  if (int st = train_loss_check(heads, targets, B, R, cfg, "multi_pose_loss_train_batch")) return st;
  if (!stats || !loss || !workspace) return cpb::fail(CPB200_ERR_ARG, "multi_pose_loss_train_batch: bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  double *partial = static_cast<double *>(workspace);
  // hm_hp's channels only where the loss reads them
  focal_kernel<<<dim3(gates(*cfg).hm_hp ? 1 + J : 1, (unsigned)B), 256, 0, s>>>(heads.hm, heads.hm_hp, targets.hm,
                                                                               targets.hm_hp, R, partial);
  if (int st = cpb::check_launch("focal_kernel")) return st;
  TrainLossArgs a = {heads, targets, B, R, *cfg, partial, stats, loss,
                     reinterpret_cast<float *>(partial + partial_doubles(B))};
  train_loss_kernel<<<1, kTrainThreads, 0, s>>>(a);
  return cpb::check_launch("train_loss_kernel");
}

extern "C" int cpb200_multi_pose_loss_train_backward(cpb200_multi_pose_heads heads, cpb200_multi_pose_targets targets,
                                                     int B, int R, const cpb200_multi_pose_loss_cfg *cfg,
                                                     const float *grad_loss, const void *workspace,
                                                     cpb200_multi_pose_heads grads, void *stream) {
  const char *what = "multi_pose_loss_train_backward";
  if (int st = train_loss_check(heads, targets, B, R, cfg, what)) return st;
  const Gates g = gates(*cfg);
  if (!grad_loss || !workspace || !grads.hm || !grads.hps || (g.wh && !grads.wh) || (g.off && !grads.reg) ||
      (g.hm_hp && !grads.hm_hp) || (g.hp_offset && !grads.hp_offset))
    return cpb::fail(CPB200_ERR_ARG, "%s: bad arguments", what);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const float *norm = reinterpret_cast<const float *>(static_cast<const double *>(workspace) + partial_doubles(B));
  const size_t plane = (size_t)R * R;
  // the heads the gates leave out get no gradient: their pointers are dropped
  float *g_wh = g.wh ? const_cast<float *>(grads.wh) : nullptr;
  float *g_reg = g.off ? const_cast<float *>(grads.reg) : nullptr;
  float *g_hp_offset = g.hp_offset ? const_cast<float *>(grads.hp_offset) : nullptr;
  float *g_hps = const_cast<float *>(grads.hps);
  DenseArgs d = {{heads.hm, heads.hm_hp}, {targets.hm, targets.hm_hp},
                 {const_cast<float *>(grads.hm), g.hm_hp ? const_cast<float *>(grads.hm_hp) : nullptr},
                 {g_wh, g_hps, g_reg, g_hp_offset},
                 {B * plane, (size_t)B * J * plane}, {B * 2 * plane, B * 2 * J * plane, B * 2 * plane, B * 2 * plane},
                 {cfg->hm_weight, cfg->hm_hp_weight}, grad_loss, norm};
  const size_t most = (size_t)B * 2 * J * plane;
  const unsigned blocks = (unsigned)std::min<size_t>((most + 255) / 256, 132 * 16);
  loss_grad_dense_kernel<<<dim3(blocks, 6), 256, 0, s>>>(d);
  if (int st = cpb::check_launch("loss_grad_dense_kernel")) return st;
  SparseArgs sp = {{{heads.hps, targets.hps, targets.ind, targets.hps_mask, g_hps, cfg->hp_weight, M, 2 * J, 1, kDenHps},
                    {heads.wh, targets.wh, targets.ind, targets.reg_mask, g_wh, cfg->wh_weight, M, 2, 0, kDenWh},
                    {heads.reg, targets.reg, targets.ind, targets.reg_mask, g_reg, cfg->off_weight, M, 2, 0, kDenReg},
                    {heads.hp_offset, targets.hp_offset, targets.hp_ind, targets.hp_mask, g_hp_offset,
                     cfg->off_weight, M * J, 2, 2, kDenHpOffset}},
                   R, grad_loss, norm};
  loss_grad_sparse_kernel<<<dim3(4, (unsigned)B), 256, 0, s>>>(sp);
  return cpb::check_launch("loss_grad_sparse_kernel");
}

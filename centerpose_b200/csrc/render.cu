// cpb200_render_poses_batch: MultiPoseDetector.show_results' drawing (the reference's Debugger.add_coco_bbox and
// add_coco_hp for every row above VIS_THRESH) on the device, byte for byte as cv2 4.13 draws it.  One kernel, one CTA
// per image:
//   1. every limb polygon of the image is scan-converted as cv2.fillConvexPoly (LINE_8, shift 0) does, one thread per
//      limb, into its span rows in the workspace (geometry only, so all persons at once);
//   2. the persons are then drawn in order, each step a block-wide loop with a barrier after it: the thickness-2 box
//      (three-pixel bands with plus-shaped corner caps), the filled label box, the label text through its per-pixel
//      tables, the radius-2 joint discs;
//   3. each limb in order marks the pixels its polygon covers (its edges' 8-connected lines and its spans) with its
//      rank r among the person's n limbs, unless an earlier limb marked them.  A pixel first covered by limb r sees
//      addWeighted(img, 0.8, canvas, 0.2, 0) with canvas = 255 for limbs r..n-1, and with canvas = img (which leaves
//      it unchanged) before, so one pass over the person's limb box applies fold[n - r] and clears the marks.
// The host side (centerpose_b200/render.py) builds the tables and the polygons (cv2.ellipse2Poly); the kernel trusts
// them.  cv2's rules are pinned by tests/render_model.py.
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_render_image) == 40, "cpb200_render_image layout is part of the C ABI");
static_assert(sizeof(cpb200_render_person) == 224, "cpb200_render_person layout is part of the C ABI");
static_assert(sizeof(cpb200_render_limb) == 24, "cpb200_render_limb layout is part of the C ABI");
static_assert(sizeof(cpb200_render_text_px) == 8, "cpb200_render_text_px layout is part of the C ABI");

constexpr int kThreads = 512;
constexpr int kXYShift = 16;
constexpr unsigned char kUnmarked = 0xFF;

// addWeighted(v, 0.8, c, 0.2, 0) on uint8: float32 products and sum, rounded half to even, saturated
__device__ __forceinline__ unsigned char blend(unsigned char v, unsigned char c) {
  const float r = __fadd_rn(__fadd_rn(__fmul_rn((float)v, 0.8f), __fmul_rn((float)c, 0.2f)), 0.f);
  return (unsigned char)min(max(__float2int_rn(r), 0), 255);
}

// cv2's clipLine: the int64 end points moved onto the image's border with double arithmetic truncated to int64
__device__ bool clip_line(long long w, long long h, long long &x1, long long &y1, long long &x2, long long &y2) {
  const long long right = w - 1, bottom = h - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    long long a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += (long long)__ddiv_rn(__dmul_rn((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += (long long)__ddiv_rn(__dmul_rn((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += (long long)__ddiv_rn(__dmul_rn((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += (long long)__ddiv_rn(__dmul_rn((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// cv2.line(..., 1, LINE_8) between integer points: clipped, then walked left to right; marks its pixels with `rank`
__device__ void mark_line(unsigned char *mark, int w, int h, long long x1, long long y1, long long x2, long long y2,
                          unsigned char rank) {
  if (x1 < 0 || x1 >= w || x2 < 0 || x2 >= w || y1 < 0 || y1 >= h || y2 < 0 || y2 >= h)
    if (!clip_line(w, h, x1, y1, x2, y2)) return;
  int dx = (int)(x2 - x1), dy = (int)(y2 - y1), sx = 1, sy = 1;
  int x = (int)x1, y = (int)y1;
  if (dx < 0) {
    dx = -dx;
    dy = -dy;
    x = (int)x2;
    y = (int)y2;
  }
  if (dy < 0) {
    dy = -dy;
    sy = -1;
  }
  const bool vert = dy > dx;
  if (vert) {
    const int t = dx;
    dx = dy;
    dy = t;
    const int s = sx;
    sx = sy;
    sy = s;
  }
  int err = dx - (dy + dy);
  const int plus = dx + dx, minus = -(dy + dy);
  // per pixel the walk steps (mx, my), plus (px, py) when the error carries
  const int mx = vert ? 0 : sx, my = vert ? sx : 0, px = vert ? sy : 0, py = vert ? 0 : sy;
  for (int i = 0; i <= dx; ++i) {
    unsigned char *m = mark + (size_t)y * w + x;
    if (*m == kUnmarked) *m = rank;
    const bool carry = err < 0;
    err += minus + (carry ? plus : 0);
    x += mx + (carry ? px : 0);
    y += my + (carry ? py : 0);
  }
}

// The span part of cv2.fillConvexPoly (LINE_8, shift 0): per row of [row0, row1] the filled [lo, hi], lo > hi when
// the row has none.  The rows above the image are stepped over in one jump per edge change (cv2 walks them one by one
// and draws nothing).
__device__ void scan_spans(const int32_t *v, int n, int w, int h, int row0, int row1, int2 *rows) {
  for (int r = row0; r <= row1; ++r) rows[r - row0] = make_int2(1, 0);
  if (n < 3 || row1 < row0) return;
  int imin = 0;
  long long ymin = v[1], ymax = v[1], xmin = v[0], xmax = v[0];
  for (int i = 0; i < n; ++i) {
    const long long x = v[2 * i], y = v[2 * i + 1];
    if (y < ymin) {
      ymin = y;
      imin = i;
    }
    ymax = max(ymax, y);
    xmax = max(xmax, x);
    xmin = min(xmin, x);
  }
  if (xmax < 0 || ymax < 0 || xmin >= w || ymin >= h) return;
  ymax = min(ymax, (long long)h - 1);
  struct Edge {
    int idx, di;
    long long x, dx, ye;
  } e[2] = {{imin, 1, -(1ll << kXYShift), 0, ymin}, {imin, n - 1, -(1ll << kXYShift), 0, ymin}};
  int edges = n;
  long long y = ymin;
  const long long half = 1ll << (kXYShift - 1);
  while (true) {
    for (int i = 0; i < 2; ++i) {
      if (y >= e[i].ye) {
        int idx0 = e[i].idx, idx = idx0 + e[i].di;
        if (idx >= n) idx -= n;
        for (; edges-- > 0;) {
          const long long ty = v[2 * idx + 1];
          if (ty > y) {
            const long long xs = (long long)v[2 * idx0] << kXYShift, xe = (long long)v[2 * idx] << kXYShift;
            e[i].ye = ty;
            e[i].dx = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y));
            e[i].x = xs;
            e[i].idx = idx;
            break;
          }
          idx0 = idx;
          idx += e[i].di;
          if (idx >= n) idx -= n;
        }
      }
    }
    if (edges < 0) break;
    if (y >= 0) {
      const int l = e[0].x > e[1].x ? 1 : 0;
      long long x1 = (e[l].x + half) >> kXYShift, x2 = (e[1 - l].x + half) >> kXYShift;
      if (x2 >= 0 && x1 < w) {
        x1 = max(x1, 0ll);
        x2 = min(x2, (long long)w - 1);
        if (x1 <= x2 && y >= row0 && y <= row1) rows[y - row0] = make_int2((int)x1, (int)x2);
      }
      e[0].x += e[0].dx;
      e[1].x += e[1].dx;
      ++y;
    } else {
      // no edge changes before min(ye) and nothing is drawn before row 0
      const long long t = min(min(e[0].ye, e[1].ye), 0ll);
      e[0].x += e[0].dx * (t - y);
      e[1].x += e[1].dx * (t - y);
      y = t;
    }
    if (y > ymax) break;
  }
}

// fill the clipped rectangle [x0, x1] x [y0, y1] of a (h, w) BGR image with `c`, block-wide
__device__ void fill_rect(unsigned char *img, int w, int h, long long x0, long long y0, long long x1, long long y1,
                          uchar4 c) {
  x0 = max(x0, 0ll);
  y0 = max(y0, 0ll);
  x1 = min(x1, (long long)w - 1);
  y1 = min(y1, (long long)h - 1);
  if (x0 > x1 || y0 > y1) return;
  const int rw = (int)(x1 - x0 + 1), n = rw * (int)(y1 - y0 + 1);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    unsigned char *p = img + ((size_t)(y0 + i / rw) * w + (x0 + i % rw)) * 3;
    p[0] = c.x;
    p[1] = c.y;
    p[2] = c.z;
  }
}

__global__ void __launch_bounds__(kThreads) render_poses_kernel(unsigned char *pixels,
                                                               const cpb200_render_image *images,
                                                               const cpb200_render_person *persons,
                                                               const cpb200_render_limb *limbs, const int32_t *verts,
                                                               const cpb200_render_text_px *text_px,
                                                               const unsigned char *luts, unsigned char *ws) {
  __shared__ unsigned char fold[CPB200_RENDER_MAX_LIMBS + 1][256];   // fold[m][v]: v after m blends with white
  const cpb200_render_image im = images[blockIdx.x];
  unsigned char *img = pixels + im.offset;
  unsigned char *mark = ws + im.ws_offset;
  const int h = im.h, w = im.w;
  for (int v = threadIdx.x; v < 256; v += blockDim.x) {
    unsigned char u = (unsigned char)v;
    fold[0][v] = u;
    for (int m = 1; m <= CPB200_RENDER_MAX_LIMBS; ++m) fold[m][v] = u = blend(u, 255);
  }
  for (size_t p = threadIdx.x; p < (size_t)h * w; p += blockDim.x) mark[p] = kUnmarked;
  for (int l = im.limb_begin + threadIdx.x; l < im.limb_begin + im.limb_count; l += blockDim.x) {
    const cpb200_render_limb L = limbs[l];
    scan_spans(verts + 2 * L.vert_begin, L.vert_count, w, h, L.row0, L.row1,
               reinterpret_cast<int2 *>(ws + L.rows_offset));
  }
  __syncthreads();
  const uchar4 white = make_uchar4(255, 255, 255, 0);
  for (int q = im.person_begin; q < im.person_begin + im.person_count; ++q) {
    const cpb200_render_person &P = persons[q];
    const uchar4 c = make_uchar4(P.color[0], P.color[1], P.color[2], 0);
    // cv2.rectangle(box, c, 2): a band three pixels wide along each side that has length, a plus at each corner
    const long long x1 = P.box[0], y1 = P.box[1], x2 = P.box[2], y2 = P.box[3];
    const long long lx = min(x1, x2), hx = max(x1, x2), ly = min(y1, y2), hy = max(y1, y2);
    if (x1 != x2) {
      fill_rect(img, w, h, lx, y1 - 1, hx, y1 + 1, c);
      fill_rect(img, w, h, lx, y2 - 1, hx, y2 + 1, c);
    }
    if (y1 != y2) {
      fill_rect(img, w, h, x1 - 1, ly, x1 + 1, hy, c);
      fill_rect(img, w, h, x2 - 1, ly, x2 + 1, hy, c);
    }
    for (int k = 0; k < 4; ++k) {
      const long long cx = (k & 1) ? x2 : x1, cy = (k & 2) ? y2 : y1;
      fill_rect(img, w, h, cx - 1, cy, cx + 1, cy, c);
      fill_rect(img, w, h, cx, cy - 1, cx, cy + 1, c);
    }
    __syncthreads();
    fill_rect(img, w, h, min(P.label[0], P.label[2]), min(P.label[1], P.label[3]), max(P.label[0], P.label[2]),
              max(P.label[1], P.label[3]), c);
    __syncthreads();
    for (int i = threadIdx.x; i < P.text_count; i += blockDim.x) {
      const cpb200_render_text_px t = text_px[P.text_begin + i];
      unsigned char *p = img + ((size_t)(P.text_y + t.dy) * w + (P.text_x + t.dx)) * 3;
      const unsigned char *lut = luts + t.lut;
      p[0] = lut[p[0]];
      p[1] = lut[p[1]];
      p[2] = lut[p[2]];
    }
    __syncthreads();
    // cv2.circle(joint, 2, white, -1): rows -2..2 with half-widths 0, 1, 2, 1, 0 (13 pixels)
    for (int i = threadIdx.x; i < CPB200_RENDER_JOINTS * 13; i += blockDim.x) {
      const int j = i / 13, k = i % 13;
      if (!((P.joints >> j) & 1)) continue;
      const int dy = k < 1 ? -2 : k < 4 ? -1 : k < 9 ? 0 : k < 12 ? 1 : 2;
      const int dx = k < 1 ? 0 : k < 4 ? k - 2 : k < 9 ? k - 6 : k < 12 ? k - 10 : 0;
      const long long x = (long long)P.joint_x[j] + dx, y = (long long)P.joint_y[j] + dy;
      if (x < 0 || x >= w || y < 0 || y >= h) continue;
      unsigned char *p = img + ((size_t)y * w + x) * 3;
      p[0] = white.x;
      p[1] = white.y;
      p[2] = white.z;
    }
    __syncthreads();
    if (P.limb_count == 0) continue;
    for (int r = 0; r < P.limb_count; ++r) {
      const cpb200_render_limb L = limbs[P.limb_begin + r];
      const int32_t *v = verts + 2 * L.vert_begin;
      for (int i = threadIdx.x; i < L.vert_count; i += blockDim.x) {
        const int a = i == 0 ? L.vert_count - 1 : i - 1;
        mark_line(mark, w, h, v[2 * a], v[2 * a + 1], v[2 * i], v[2 * i + 1], (unsigned char)r);
      }
      const int2 *rows = reinterpret_cast<const int2 *>(ws + L.rows_offset);
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
      for (int y = L.row0 + warp; y <= L.row1; y += kThreads / 32) {
        const int2 s = rows[y - L.row0];
        for (int x = s.x + lane; x <= s.y; x += 32) {
          unsigned char *m = mark + (size_t)y * w + x;
          if (*m == kUnmarked) *m = (unsigned char)r;
        }
      }
      __syncthreads();
    }
    const int bx0 = P.fold_box[0], by0 = P.fold_box[1], bw = P.fold_box[2] - bx0 + 1, bh = P.fold_box[3] - by0 + 1;
    if (bw > 0 && bh > 0) {
      for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
        const size_t o = (size_t)(by0 + i / bw) * w + (bx0 + i % bw);
        const int r = mark[o];
        if (r == kUnmarked) continue;
        mark[o] = kUnmarked;
        const unsigned char *f = fold[P.limb_count - r];
        unsigned char *p = img + o * 3;
        p[0] = f[p[0]];
        p[1] = f[p[1]];
        p[2] = f[p[2]];
      }
    }
    __syncthreads();
  }
}

}  // namespace

extern "C" int cpb200_render_poses_batch(unsigned char *pixels, const cpb200_render_image *images, int B,
                                         const cpb200_render_person *persons, const cpb200_render_limb *limbs,
                                         const int32_t *verts, const cpb200_render_text_px *text_px,
                                         const unsigned char *luts, void *workspace, void *stream) {
  if (!pixels || !images || !persons || !limbs || !verts || !text_px || !luts || !workspace || B < 1)
    return cpb::fail(CPB200_ERR_ARG, "render_poses_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "render_poses_batch: B = %d images exceed one launch (max 65535)", B);
  render_poses_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      pixels, images, persons, limbs, verts, text_px, luts, static_cast<unsigned char *>(workspace));
  return cpb::check_launch("render_poses_kernel");
}

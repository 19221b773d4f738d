// The drawing plan of run_video on the device: what centerpose_b200/render.py's build() makes on the host (the
// persons, limbs and limb polygons of cpb200_render_poses_batch), made from detection rows already on the device.
// One CTA per image:
//   1. the rows whose score is above VIS_THRESH become the image's persons, in row order (a serial scan of the flags);
//   2. per person (one thread each) the int32 box, the label box, the joints and, per limb, render.limb_polygon's
//      float64 geometry and cv2.ellipse2Poly's polygon, counted first: the vertex and span-row totals are scanned in
//      person order, so every run lays the tables out the same way;
//   3. the same threads write the polygons and the limbs at their offsets.
// The label text is not drawn from here: each person's key (label, border cut) goes back to the host, whose cache of
// cv2.putText tables fills text_begin / text_count.  cv2's polygon rules are pinned by tests/render_model.py.
#include <climits>

#include "common.cuh"
#include "../../include/centerpose_b200_video.h"

namespace {

static_assert(sizeof(cpb200_render_label) == 24, "cpb200_render_label layout is part of the C ABI");
static_assert(sizeof(cpb200_render_key) == 24, "cpb200_render_key layout is part of the C ABI");

constexpr int kThreads = 256;
constexpr int kMaxRows = 2048;               // rows per image (16 bytes of shared memory each)
constexpr int kEdges = 18;
__constant__ int kEdgeA[kEdges] = {0, 0, 1, 2, 3, 4, 5, 5, 7, 6, 8, 5, 6, 11, 11, 13, 12, 14};
__constant__ int kEdgeB[kEdges] = {1, 2, 3, 4, 5, 6, 6, 7, 9, 8, 10, 11, 12, 12, 13, 15, 14, 16};

// cv2's sine table for integer degrees 0..450: sin(i degrees) to seven decimals, as float
__constant__ float kSin[451] = {
    0.0f, 0.0174524002f, 0.0348994993f, 0.0523359999f, 0.0697565004f, 0.0871556997f, 0.104528502f, 0.121869303f,
    0.139173105f, 0.156434506f, 0.173648193f, 0.190808997f, 0.2079117f, 0.224951103f, 0.241921902f, 0.258819014f,
    0.275637388f, 0.29237169f, 0.309017003f, 0.325568199f, 0.342020094f, 0.35836789f, 0.374606609f, 0.390731096f,
    0.406736612f, 0.4226183f, 0.438371092f, 0.453990489f, 0.469471604f, 0.484809607f, 0.5f, 0.515038073f,
    0.529919326f, 0.544638991f, 0.559192896f, 0.573576391f, 0.587785304f, 0.601814985f, 0.615661502f, 0.629320383f,
    0.642787576f, 0.656059027f, 0.669130623f, 0.681998372f, 0.694658399f, 0.707106829f, 0.719339788f, 0.7313537f,
    0.74314481f, 0.754709601f, 0.766044378f, 0.777145982f, 0.788010776f, 0.798635483f, 0.809017003f, 0.819151998f,
    0.829037607f, 0.838670611f, 0.848048091f, 0.857167304f, 0.866025388f, 0.874619722f, 0.882947624f, 0.891006529f,
    0.898793995f, 0.906307817f, 0.913545489f, 0.920504928f, 0.927183926f, 0.933580399f, 0.939692616f, 0.945518613f,
    0.95105648f, 0.956304789f, 0.96126169f, 0.965925813f, 0.970295727f, 0.974370122f, 0.978147626f, 0.981627226f,
    0.984807789f, 0.987688303f, 0.990268111f, 0.992546201f, 0.994521916f, 0.99619472f, 0.997564077f, 0.99862951f,
    0.999390781f, 0.99984771f, 1.0f, 0.99984771f, 0.999390781f, 0.99862951f, 0.997564077f, 0.99619472f,
    0.994521916f, 0.992546201f, 0.990268111f, 0.987688303f, 0.984807789f, 0.981627226f, 0.978147626f, 0.974370122f,
    0.970295727f, 0.965925813f, 0.96126169f, 0.956304789f, 0.95105648f, 0.945518613f, 0.939692616f, 0.933580399f,
    0.927183926f, 0.920504928f, 0.913545489f, 0.906307817f, 0.898793995f, 0.891006529f, 0.882947624f, 0.874619722f,
    0.866025388f, 0.857167304f, 0.848048091f, 0.838670611f, 0.829037607f, 0.819151998f, 0.809017003f, 0.798635483f,
    0.788010776f, 0.777145982f, 0.766044378f, 0.754709601f, 0.74314481f, 0.7313537f, 0.719339788f, 0.707106829f,
    0.694658399f, 0.681998372f, 0.669130623f, 0.656059027f, 0.642787576f, 0.629320383f, 0.615661502f, 0.601814985f,
    0.587785304f, 0.573576391f, 0.559192896f, 0.544638991f, 0.529919326f, 0.515038073f, 0.5f, 0.484809607f,
    0.469471604f, 0.453990489f, 0.438371092f, 0.4226183f, 0.406736612f, 0.390731096f, 0.374606609f, 0.35836789f,
    0.342020094f, 0.325568199f, 0.309017003f, 0.29237169f, 0.275637388f, 0.258819014f, 0.241921902f, 0.224951103f,
    0.2079117f, 0.190808997f, 0.173648193f, 0.156434506f, 0.139173105f, 0.121869303f, 0.104528502f, 0.0871556997f,
    0.0697565004f, 0.0523359999f, 0.0348994993f, 0.0174524002f, 0.0f, -0.0174524002f, -0.0348994993f, -0.0523359999f,
    -0.0697565004f, -0.0871556997f, -0.104528502f, -0.121869303f, -0.139173105f, -0.156434506f, -0.173648193f, -0.190808997f,
    -0.2079117f, -0.224951103f, -0.241921902f, -0.258819014f, -0.275637388f, -0.29237169f, -0.309017003f, -0.325568199f,
    -0.342020094f, -0.35836789f, -0.374606609f, -0.390731096f, -0.406736612f, -0.4226183f, -0.438371092f, -0.453990489f,
    -0.469471604f, -0.484809607f, -0.5f, -0.515038073f, -0.529919326f, -0.544638991f, -0.559192896f, -0.573576391f,
    -0.587785304f, -0.601814985f, -0.615661502f, -0.629320383f, -0.642787576f, -0.656059027f, -0.669130623f, -0.681998372f,
    -0.694658399f, -0.707106829f, -0.719339788f, -0.7313537f, -0.74314481f, -0.754709601f, -0.766044378f, -0.777145982f,
    -0.788010776f, -0.798635483f, -0.809017003f, -0.819151998f, -0.829037607f, -0.838670611f, -0.848048091f, -0.857167304f,
    -0.866025388f, -0.874619722f, -0.882947624f, -0.891006529f, -0.898793995f, -0.906307817f, -0.913545489f, -0.920504928f,
    -0.927183926f, -0.933580399f, -0.939692616f, -0.945518613f, -0.95105648f, -0.956304789f, -0.96126169f, -0.965925813f,
    -0.970295727f, -0.974370122f, -0.978147626f, -0.981627226f, -0.984807789f, -0.987688303f, -0.990268111f, -0.992546201f,
    -0.994521916f, -0.99619472f, -0.997564077f, -0.99862951f, -0.999390781f, -0.99984771f, -1.0f, -0.99984771f,
    -0.999390781f, -0.99862951f, -0.997564077f, -0.99619472f, -0.994521916f, -0.992546201f, -0.990268111f, -0.987688303f,
    -0.984807789f, -0.981627226f, -0.978147626f, -0.974370122f, -0.970295727f, -0.965925813f, -0.96126169f, -0.956304789f,
    -0.95105648f, -0.945518613f, -0.939692616f, -0.933580399f, -0.927183926f, -0.920504928f, -0.913545489f, -0.906307817f,
    -0.898793995f, -0.891006529f, -0.882947624f, -0.874619722f, -0.866025388f, -0.857167304f, -0.848048091f, -0.838670611f,
    -0.829037607f, -0.819151998f, -0.809017003f, -0.798635483f, -0.788010776f, -0.777145982f, -0.766044378f, -0.754709601f,
    -0.74314481f, -0.7313537f, -0.719339788f, -0.707106829f, -0.694658399f, -0.681998372f, -0.669130623f, -0.656059027f,
    -0.642787576f, -0.629320383f, -0.615661502f, -0.601814985f, -0.587785304f, -0.573576391f, -0.559192896f, -0.544638991f,
    -0.529919326f, -0.515038073f, -0.5f, -0.484809607f, -0.469471604f, -0.453990489f, -0.438371092f, -0.4226183f,
    -0.406736612f, -0.390731096f, -0.374606609f, -0.35836789f, -0.342020094f, -0.325568199f, -0.309017003f, -0.29237169f,
    -0.275637388f, -0.258819014f, -0.241921902f, -0.224951103f, -0.2079117f, -0.190808997f, -0.173648193f, -0.156434506f,
    -0.139173105f, -0.121869303f, -0.104528502f, -0.0871556997f, -0.0697565004f, -0.0523359999f, -0.0348994993f, -0.0174524002f,
    -0.0f, 0.0174524002f, 0.0348994993f, 0.0523359999f, 0.0697565004f, 0.0871556997f, 0.104528502f, 0.121869303f,
    0.139173105f, 0.156434506f, 0.173648193f, 0.190808997f, 0.2079117f, 0.224951103f, 0.241921902f, 0.258819014f,
    0.275637388f, 0.29237169f, 0.309017003f, 0.325568199f, 0.342020094f, 0.35836789f, 0.374606609f, 0.390731096f,
    0.406736612f, 0.4226183f, 0.438371092f, 0.453990489f, 0.469471604f, 0.484809607f, 0.5f, 0.515038073f,
    0.529919326f, 0.544638991f, 0.559192896f, 0.573576391f, 0.587785304f, 0.601814985f, 0.615661502f, 0.629320383f,
    0.642787576f, 0.656059027f, 0.669130623f, 0.681998372f, 0.694658399f, 0.707106829f, 0.719339788f, 0.7313537f,
    0.74314481f, 0.754709601f, 0.766044378f, 0.777145982f, 0.788010776f, 0.798635483f, 0.809017003f, 0.819151998f,
    0.829037607f, 0.838670611f, 0.848048091f, 0.857167304f, 0.866025388f, 0.874619722f, 0.882947624f, 0.891006529f,
    0.898793995f, 0.906307817f, 0.913545489f, 0.920504928f, 0.927183926f, 0.933580399f, 0.939692616f, 0.945518613f,
    0.95105648f, 0.956304789f, 0.96126169f, 0.965925813f, 0.970295727f, 0.974370122f, 0.978147626f, 0.981627226f,
    0.984807789f, 0.987688303f, 0.990268111f, 0.992546201f, 0.994521916f, 0.99619472f, 0.997564077f, 0.99862951f,
    0.999390781f, 0.99984771f, 1.0f,
};

// float32 to int32 as numpy on x86 converts (cvttss2si): out of range and NaN give INT32_MIN
__device__ __forceinline__ int trunc_i32(float f) {
  return (f != f || f >= 2147483648.f || f < -2147483648.f) ? INT_MIN : (int)f;
}

__device__ __forceinline__ int wrap_sub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }

// cv2.ellipse2Poly(center, (half_len, 2), angle, 0, 360, 1): 361 points of the double ellipse, each rounded half to
// even, consecutive duplicates dropped (a single point becomes the centre twice).  Writes them when `out` is set;
// returns their number and their bounds.
__device__ int ellipse_points(int cx, int cy, int half_len, int angle, int2 *out, long long &xmin, long long &xmax,
                              long long &ymin, long long &ymax) {
  while (angle < 0) angle += 360;
  while (angle > 360) angle -= 360;
  const double alpha = (double)kSin[450 - angle], beta = (double)kSin[angle];
  int px = INT_MIN, py = INT_MIN, n = 0;
  xmin = ymin = LLONG_MAX;
  xmax = ymax = LLONG_MIN;
  for (int i = 0; i <= 360; ++i) {
    const double x = __dmul_rn((double)half_len, (double)kSin[450 - i]);
    const double y = __dmul_rn(2.0, (double)kSin[i]);
    const double fx = __dsub_rn(__dadd_rn((double)cx, __dmul_rn(x, alpha)), __dmul_rn(y, beta));
    const double fy = __dadd_rn(__dadd_rn((double)cy, __dmul_rn(x, beta)), __dmul_rn(y, alpha));
    const int qx = __double2int_rn(fx), qy = __double2int_rn(fy);
    if (n == 0 || qx != px || qy != py) {
      if (out) out[n] = make_int2(qx, qy);
      ++n;
      px = qx;
      py = qy;
      xmin = min(xmin, (long long)qx);
      xmax = max(xmax, (long long)qx);
      ymin = min(ymin, (long long)qy);
      ymax = max(ymax, (long long)qy);
    }
  }
  if (n == 1) {
    if (out) out[0] = out[1] = make_int2(cx, cy);
    n = 2;
    xmin = xmax = cx;
    ymin = ymax = cy;
  }
  return n;
}

__global__ void ellipse_poly_kernel(const int4 *params, int n, int2 *verts, int32_t *counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int4 p = params[i];
  long long a, b, c, d;
  counts[i] = ellipse_points(p.x, p.y, p.z, p.w, verts + (size_t)i * CPB200_ELLIPSE_MAX_POINTS, a, b, c, d);
}

// render.limb_polygon's geometry of the limb between joints (xa, ya) and (xb, yb): numpy's int32 differences and
// squares (wrapping), the float64 mean through int(), sqrt, degrees(atan2(dy, dx)) through int().  False when the
// squared length wraps negative (numpy's NaN length, which int() refuses).
__device__ bool limb_geometry(int xa, int ya, int xb, int yb, int &cx, int &cy, int &half_len, int &angle) {
  const int dy = wrap_sub(ya, yb), dx = wrap_sub(xa, xb);
  cy = (int)(((double)ya + (double)yb) / 2.0);
  cx = (int)(((double)xa + (double)xb) / 2.0);
  const int s = (int)((unsigned)dy * (unsigned)dy + (unsigned)dx * (unsigned)dx);
  if (s < 0) return false;
  half_len = (int)(sqrt((double)s) / 2.0);
  // the angles that are whole degrees come out exact in Python; atan2 rounds differently there, so they are set
  if (dy == 0) angle = dx < 0 ? 180 : 0;
  else if (dx == 0) angle = dy > 0 ? 90 : -90;
  else if (dy == dx || dy == -dx) angle = dx > 0 ? (dy > 0 ? 45 : -45) : (dy > 0 ? 135 : -135);
  else angle = (int)__dmul_rn(atan2((double)dy, (double)dx), 180.0 / 3.141592653589793);
  return true;
}

// "{:.1f}".format(score) for a finite score >= 0: k with the text "p{k / 10}.{k % 10}", k = round(10 * score) on the
// exact value (never a tie: (2k + 1) / 20 is not a binary fraction)
__device__ long long label_index(double d) {
  long long k = (long long)floor(__dmul_rn(d, 10.0));
  if (fma(d, 10.0, -(double)k) < 0) --k;
  else if (fma(d, 10.0, -(double)(k + 1)) >= 0) ++k;
  if (fma(d, 10.0, -((double)k + 0.5)) > 0) ++k;
  return k;
}

struct Plan {
  const float *row;
  int h, w;
  // where the person's polygons go (pass 3) or nullptr (pass 2, counting)
  int2 *verts;
  int vert_base;                 // index of verts[0] in the whole vertex array
  long long rows_base;           // workspace byte of the person's first span row
};

// One person: fills P (text fields 0) and, when plan.verts is set, its limbs; returns its vertex and span-row byte
// totals, or a status > 0.
__device__ int plan_person(const Plan &plan, const cpb200_render_label *labels, int n_labels, int color,
                           cpb200_render_person &P, cpb200_render_key &key, cpb200_render_limb *limbs,
                           int limb_base, int &n_verts, long long &n_rows) {
  const float *row = plan.row;
  const int h = plan.h, w = plan.w;
  const double score = (double)row[4];
  n_verts = 0;
  n_rows = 0;
  if (!isfinite(score)) return 2;
  const long long k = label_index(score);
  if (k < 0 || k >= n_labels) return 2;
  const cpb200_render_label L = labels[k];
  for (int i = 0; i < 4; ++i) P.box[i] = trunc_i32(row[i]);
  P.label[0] = P.box[0];
  P.label[1] = wrap_sub(wrap_sub(P.box[1], L.th), 2);
  P.label[2] = (int)((unsigned)P.box[0] + (unsigned)L.tw);
  P.label[3] = wrap_sub(P.box[1], 2);
  P.text_x = P.box[0];
  P.text_y = wrap_sub(P.box[1], 2);
  P.text_begin = P.text_count = 0;
  P.color[0] = color & 255;
  P.color[1] = (color >> 8) & 255;
  P.color[2] = (color >> 16) & 255;
  P.color[3] = 0;
  const long long ox = P.text_x, oy = P.text_y;
  const long long ax = max(-ox, (long long)L.x0), bx = min(w - 1 - ox, (long long)L.x1);
  const long long ay = max(-oy, (long long)L.y0), by = min(h - 1 - oy, (long long)L.y1);
  key.label = (int)k;
  key.valid = ax <= bx && ay <= by;
  key.ax = key.valid ? (int)ax : 0;
  key.bx = key.valid ? (int)bx : 0;
  key.ay = key.valid ? (int)ay : 0;
  key.by = key.valid ? (int)by : 0;
  int joints = 0;
  for (int j = 0; j < CPB200_RENDER_JOINTS; ++j) {
    P.joint_x[j] = trunc_i32(row[5 + 2 * j]);
    P.joint_y[j] = trunc_i32(row[6 + 2 * j]);
    if (row[39 + j] > 0.f) joints |= 1 << j;
  }
  P.joints = joints;
  P.pad[0] = P.pad[1] = 0;
  P.limb_begin = limb_base;
  long long fx0 = w, fy0 = h, fx1 = -1, fy1 = -1;
  int count = 0;
  for (int e = 0; e < kEdges; ++e) {
    const int a = kEdgeA[e], b = kEdgeB[e];
    if (!(((joints >> a) & 1) && ((joints >> b) & 1))) continue;
    int cx, cy, half_len, angle;
    if (!limb_geometry(P.joint_x[a], P.joint_y[a], P.joint_x[b], P.joint_y[b], cx, cy, half_len, angle)) return 3;
    long long xmin, xmax, ymin, ymax;
    int2 *out = plan.verts ? plan.verts + n_verts : nullptr;
    const int nv = ellipse_points(cx, cy, half_len, angle, out, xmin, xmax, ymin, ymax);
    const long long row0 = max(ymin, 0ll), row1 = min(ymax, (long long)h - 1);
    if (plan.verts) {
      cpb200_render_limb &Lb = limbs[limb_base + count];
      Lb.vert_begin = plan.vert_base + n_verts;
      Lb.vert_count = nv;
      Lb.row0 = (int)row0;
      Lb.row1 = (int)row1;
      Lb.rows_offset = plan.rows_base + n_rows;
    }
    n_verts += nv;
    n_rows += max(row1 - row0 + 1, 0ll) * 8;
    fx0 = min(fx0, xmin - 2);
    fx1 = max(fx1, xmax + 2);
    fy0 = min(fy0, ymin - 2);
    fy1 = max(fy1, ymax + 2);
    ++count;
  }
  P.limb_count = count;
  P.fold_box[0] = (int)max(fx0, 0ll);
  P.fold_box[1] = (int)max(fy0, 0ll);
  P.fold_box[2] = (int)min(fx1, (long long)w - 1);
  P.fold_box[3] = (int)min(fy1, (long long)h - 1);
  if (plan.verts)
    for (int e = count; e < kEdges; ++e) {
      cpb200_render_limb &Lb = limbs[limb_base + e];
      Lb.vert_begin = 0;
      Lb.vert_count = 0;
      Lb.row0 = 0;
      Lb.row1 = -1;
      Lb.rows_offset = 0;
    }
  return 0;
}

__global__ void __launch_bounds__(kThreads) render_plan_kernel(
    const float *rows, int N, int h, int w, double vis_thresh, int color, const cpb200_render_label *labels,
    int n_labels, long long verts_per_image, long long rows_per_image, long long ws_marks,
    cpb200_render_image *images, cpb200_render_person *persons, cpb200_render_limb *limbs, int2 *verts,
    cpb200_render_key *keys, int32_t *counts) {
  __shared__ int pidx[kMaxRows];               // person index of row r, -1 when not drawn
  __shared__ int vert_at[kMaxRows];            // per person: first vertex, then (after the scan) its offset
  __shared__ long long rows_at[kMaxRows];
  __shared__ int n_persons, status;
  __shared__ long long total_rows;
  __shared__ int total_verts;
  const int b = blockIdx.x;
  const float *img_rows = rows + (size_t)b * N * 56;
  for (int r = threadIdx.x; r < N; r += blockDim.x) pidx[r] = (double)img_rows[(size_t)r * 56 + 4] > vis_thresh;
  if (threadIdx.x == 0) status = 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    int p = 0;
    for (int r = 0; r < N; ++r) pidx[r] = pidx[r] ? p++ : -1;
    n_persons = p;
  }
  __syncthreads();
  const int pb = b * N;                        // the image's first person slot
  const Plan counting{nullptr, h, w, nullptr, 0, 0};
  for (int r = threadIdx.x; r < N; r += blockDim.x) {
    const int p = pidx[r];
    if (p < 0) continue;
    Plan plan = counting;
    plan.row = img_rows + (size_t)r * 56;
    int nv;
    long long nr;
    const int st = plan_person(plan, labels, n_labels, color, persons[pb + p], keys[pb + p], limbs,
                               (pb + p) * kEdges, nv, nr);
    if (st) atomicMax(&status, st);
    vert_at[p] = nv;
    rows_at[p] = nr;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int v = 0;
    long long s = 0;
    for (int p = 0; p < n_persons; ++p) {
      const int nv = vert_at[p];
      const long long nr = rows_at[p];
      vert_at[p] = v;
      rows_at[p] = s;
      v += nv;
      s += nr;
    }
    total_verts = v;
    total_rows = s;
    if (status == 0 && (v > verts_per_image || s > rows_per_image)) status = 1;
  }
  __syncthreads();
  if (status == 0)
    for (int r = threadIdx.x; r < N; r += blockDim.x) {
      const int p = pidx[r];
      if (p < 0) continue;
      const long long vb = (long long)b * verts_per_image + vert_at[p];
      const Plan plan{img_rows + (size_t)r * 56, h, w, verts + vb, (int)vb,
                      (long long)gridDim.x * ws_marks + b * rows_per_image + rows_at[p]};
      int nv;
      long long nr;
      plan_person(plan, labels, n_labels, color, persons[pb + p], keys[pb + p], limbs, (pb + p) * kEdges, nv, nr);
    }
  if (threadIdx.x == 0) {
    cpb200_render_image &I = images[b];
    I.offset = (long long)b * h * w * 3;
    I.ws_offset = b * ws_marks;
    I.h = h;
    I.w = w;
    I.person_begin = pb;
    I.person_count = status == 0 ? n_persons : 0;
    I.limb_begin = pb * kEdges;
    I.limb_count = status == 0 ? n_persons * kEdges : 0;
    counts[4 * b] = n_persons;
    counts[4 * b + 1] = total_verts;
    counts[4 * b + 2] = (int)min(total_rows, (long long)INT_MAX);
    counts[4 * b + 3] = status;
  }
}

}  // namespace

extern "C" int cpb200_ellipse_poly_batch(const int32_t *params, int n, int32_t *verts, int32_t *counts, void *stream) {
  if (!params || !verts || !counts || n < 1) return cpb::fail(CPB200_ERR_ARG, "ellipse_poly_batch: bad arguments");
  ellipse_poly_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const int4 *>(params), n, reinterpret_cast<int2 *>(verts), counts);
  return cpb::check_launch("ellipse_poly_kernel");
}

extern "C" int cpb200_render_plan_batch(const float *rows, int B, int N, int h, int w, double vis_thresh, int color,
                                        const cpb200_render_label *labels, int n_labels, int64_t verts_per_image,
                                        int64_t rows_per_image, cpb200_render_image *images,
                                        cpb200_render_person *persons, cpb200_render_limb *limbs, int32_t *verts,
                                        cpb200_render_key *keys, int32_t *counts, void *stream) {
  if (!rows || !labels || !images || !persons || !limbs || !verts || !keys || !counts || B < 1 || N < 0 || h < 1 ||
      w < 1 || n_labels < 1 || verts_per_image < 0 || rows_per_image < 0 || !(vis_thresh >= 0))
    return cpb::fail(CPB200_ERR_ARG, "render_plan_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "render_plan_batch: B = %d images exceed one launch (max 65535)", B);
  if (N > kMaxRows) return cpb::fail(CPB200_ERR_ARG, "render_plan_batch: N = %d rows per image (max %d)", N, kMaxRows);
  if ((long long)B * N * kEdges > INT_MAX || (long long)B * verts_per_image > INT_MAX)
    return cpb::fail(CPB200_ERR_ARG, "render_plan_batch: the limb or vertex tables exceed int32 indices");
  const long long ws_marks = ((long long)h * w + 7) / 8 * 8;
  render_plan_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      rows, N, h, w, vis_thresh, color, labels, n_labels, verts_per_image, rows_per_image, ws_marks, images, persons,
      limbs, reinterpret_cast<int2 *>(verts), keys, counts);
  return cpb::check_launch("render_plan_kernel");
}

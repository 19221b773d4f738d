/*
 * centerpose_b200 — C ABI of the video path's drawing plan, with the conventions of centerpose_b200.h (DEVICE
 * pointers, the caller's stream, 0 = ok and the text through cpb200_last_error()).  The entry points are exported by
 * the same library; this header takes the drawing tables of cpb200_render_poses_batch from centerpose_b200.h.
 */
#ifndef CENTERPOSE_B200_VIDEO_H_
#define CENTERPOSE_B200_VIDEO_H_

#include "centerpose_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* cv2.ellipse2Poly(center, (half_len, 2), angle, 0, 360, 1) makes at most this many points */
#define CPB200_ELLIPSE_MAX_POINTS 361

/* The polygon of n limbs (csrc/render_plan.cu): params holds n (cx, cy, half_len, angle) int32 quadruples, and
 * limb i's points go to verts[i * 2 * CPB200_ELLIPSE_MAX_POINTS ...] as (x, y) int32 pairs, their number to counts[i];
 * point for point cv2.ellipse2Poly(center, (half_len, 2), angle, 0, 360, 1) (cv2's sine table, its rounding half to
 * even, consecutive duplicates removed).  half_len >= 0.  1 <= n. */
int cpb200_ellipse_poly_batch(const int32_t *params, int n, int32_t *verts, int32_t *counts, void *stream);

/* The metrics of one label string (24 bytes): getTextSize(txt, SIMPLEX, 0.5, 2)'s width and height, and the box
 * (x0, x1, y0, y1) around the origin that holds every pixel putText(txt, SIMPLEX, 0.5, 1, LINE_AA) can touch. */
typedef struct cpb200_render_label {
  int32_t tw, th;
  int32_t x0, x1, y0, y1;
} cpb200_render_label;

/* One drawn person's label text key (24 bytes): label index k (the text is "p{k / 10}.{k % 10}", score formatted as
 * "{:.1f}"), and how the (h, w) image border cuts the text's box, [ax, bx] x [ay, by] around its origin; valid = 0 when
 * no pixel of the text lies in the image (the person then has no text pixels). */
typedef struct cpb200_render_key {
  int32_t label, ax, bx, ay, by, valid;
} cpb200_render_key;

/* The tables cpb200_render_poses_batch draws from, built on the device from B images' detection rows, what
 * centerpose_b200/render.py's build() makes on the host: rows (B, N, 56) float32; the images are (h, w), image b's
 * pixels at byte b * h * w * 3.  Per image the rows whose score, as a double, is above vis_thresh (>= 0), in row order,
 * become persons b * N + 0, 1, ...: the int32 box (float32 to int32 as x86 converts: out of range and NaN give
 * INT32_MIN), the label box from labels[k], the joints scoring above 0, and for every limb of the skeleton whose two
 * joints score above 0 the ellipse2Poly polygon of render.limb_polygon's float64 geometry.  Person p's limbs are in
 * limbs[p * 18 ...]; the unused slots of a drawn person are empty limbs (vert_count 0).  color is B | G << 8 | R << 16.
 * Image b's vertices go to verts[2 * b * verts_per_image ...] and its limbs' span rows to workspace byte
 * B * ws_image + b * rows_per_image, where ws_image = (h * w + 7) / 8 * 8 (the marks of image b are at b * ws_image),
 * so the render workspace is B * (ws_image + rows_per_image) bytes.  text_begin and text_count are left 0: keys[p]
 * says which text the caller's cache holds for person p.  counts[4 * b ...] = (persons, vertices, span-row bytes,
 * status); status 0 ok, 1 vertices or span rows past their share (the tables are then incomplete: call again with
 * more), 2 a label index outside labels or a score that is not finite, 3 a limb whose squared length wraps int32 (the
 * reference's numpy arithmetic gives NaN there).  1 <= B <= 65535, 0 <= N <= 2048. */
int cpb200_render_plan_batch(const float *rows, int B, int N, int h, int w, double vis_thresh, int color,
                             const cpb200_render_label *labels, int n_labels, int64_t verts_per_image,
                             int64_t rows_per_image, cpb200_render_image *images, cpb200_render_person *persons,
                             cpb200_render_limb *limbs, int32_t *verts, cpb200_render_key *keys, int32_t *counts,
                             void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CENTERPOSE_B200_VIDEO_H_ */

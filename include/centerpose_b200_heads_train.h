/*
 * centerpose_b200 — C ABI of the keypoint heads for training, with the conventions of centerpose_b200.h (DEVICE
 * pointers, the caller's stream and workspace, 0 = ok and the text through cpb200_last_error()).  The entry points
 * are exported by the same library; this header takes the heads struct from centerpose_b200.h.
 */
#ifndef CENTERPOSE_B200_HEADS_TRAIN_H_
#define CENTERPOSE_B200_HEADS_TRAIN_H_

#include "centerpose_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- The keypoint heads for training: KeypointHead (lib/models/heads/keypoint.py) forward and backward ----
 * Six heads in HEADS order (hm, wh, hps, reg, hm_hp, hp_offset) with 1, 2, 34, 2, 17, 2 outputs, each
 * Conv2d(C, hc, 3, padding 1) -> ReLU -> Conv2d(hc, c_h, 1).  NCHW fp32: x (B,C,H,W); the weights concatenated in
 * HEADS order, w0 (6*hc,C,3,3), b0 (6*hc), w2 (58,hc), b2 (58); each head's map (B,c_h,H,W) in the heads struct.
 * The hc x H x W hidden maps never reach HBM: the forward keeps each tile in shared memory and the backward
 * recomputes it, so the ReLU mask is the forward's.  precision: CPB200_DCN_TF32X3 (tensor cores, each fp32 operand
 * split into two tf32 parts) or CPB200_DCN_FP32 (CUDA cores), as for the DCN.  Every shape is taken.  Every output and
 * gradient is a sum in a fixed order, so the same bits on every run.  Nothing is allocated and nothing waits on the
 * host. */

/* Workspace of cpb200_heads_train_backward; 0 for a bad shape.  The backward runs over chunks of
 * max(1, min(B, floor(256 MiB / (6*hc*H*W*4)))) images; the workspace holds one chunk's d_hidden (6*hc*H*W floats per
 * image), its per-tile partials of dW2, db0 and db2 (64*hc + 58 floats per image and 128-pixel tile) and the weight
 * gradient's split-K partials (6*hc*C*9 floats per split, the splits of a full or of the last chunk, whichever has more,
 * at most 16 MiB unless one split is larger). */
size_t cpb200_heads_train_workspace_bytes(int B, int C, int H, int W, int hc);

/* The six head maps out.hm .. out.hp_offset = w2 . relu(conv3x3(x, w0) + b0) + b2, head by head. */
int cpb200_heads_train_forward(const float *x, const float *w0, const float *b0, const float *w2, const float *b2,
                               cpb200_multi_pose_heads out, int B, int C, int H, int W, int hc, int precision,
                               void *stream);

/* The gradients for the six maps' grad_output (same shapes as the maps).  A NULL member of grad_output: that head gets
 * no gradient, and its rows of grad_w0, grad_b0, grad_w2 and grad_b2 are set to 0.  grad_x (B,C,H,W) may be NULL:
 * the data pass is then skipped.  grad_w0, grad_b0, grad_w2 and grad_b2 are in the layout of the weights. */
int cpb200_heads_train_backward(const float *x, const float *w0, const float *b0, const float *w2,
                                cpb200_multi_pose_heads grad_output, float *grad_x, float *grad_w0, float *grad_b0,
                                float *grad_w2, float *grad_b2, int B, int C, int H, int W, int hc, int precision,
                                void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CENTERPOSE_B200_HEADS_TRAIN_H_ */

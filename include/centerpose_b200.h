/*
 * centerpose_b200 — C ABI of the H100-native (sm_90a) centerpose inference hot path.
 *
 * The reference (tensorboy/centerpose) has no FFI for this path: its seams are Python
 * callables (SURVEY.md §8b).  Every entry point below names the reference interface it
 * replaces; INTEGRATION.md shows the ctypes binding a maintainer adds on the reference side.
 *
 * Conventions (mirroring the reference's only native seam, the `_ext` DCNv2 module,
 * lib/models/backbones/DCNv2/src/dcn_v2.h:9-39 / src/cuda/dcn_v2_cuda.cu:42-172):
 *   - all tensor arguments are DEVICE pointers, fp32 unless said otherwise, contiguous;
 *   - work is enqueued on the caller's `stream` (a cudaStream_t passed as void*), no
 *     internal synchronisation, no allocation: scratch comes from caller-owned workspaces
 *     whose size is returned by the matching *_workspace_bytes() query;
 *   - return value 0 = ok; non-zero = error, text via cpb200_last_error() (thread-local);
 *     the Python shim raises RuntimeError, matching AT_ERROR/AT_ASSERTM -> RuntimeError.
 *   - no torch types anywhere in the signatures.
 */
#ifndef CENTERPOSE_B200_H_
#define CENTERPOSE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CPB200_OK 0
#define CPB200_ERR_ARG 1      /* bad argument (shape, null pointer, unsupported size) */
#define CPB200_ERR_CUDA 2     /* CUDA runtime / launch failure */
#define CPB200_ERR_STATE 3    /* library not usable (no sm_90 device, driver entry point missing) */

#define CPB200_DECODE_MAX_K 128
#define CPB200_DECODE_MAX_J 32

/* Version / diagnostics. */
int cpb200_version(void);
const char *cpb200_last_error(void);
/* Number of kernels this library has launched since load (used by bench.py "gpu_launches"). */
unsigned long long cpb200_launch_count(void);

/* ------------------------------------------------------------------------------------
 * Fused decode.  Replaces lib/models/decode.py:235-308 `multi_pose_decode` together with
 * its helpers `_nms` (:10-16), `_topk` (:99-115), `_topk_channel` (:87-96) and
 * lib/models/utils.py:11-25 `_gather_feat` / `_transpose_and_gather_feat`; with
 * apply_sigmoid != 0 it also absorbs the two `sigmoid_()` calls of
 * lib/detectors/multi_pose.py:35-37 (the heads hand over logits).
 *
 *   heat      (B,1,H,W)   centre heat-map            (required)
 *   wh        (B,2,H,W)   box size                   (required)
 *   kps       (B,2J,H,W)  keypoint offsets           (required)
 *   reg       (B,2,H,W)   centre sub-pixel offset    (NULL -> +0.5, decode.py:253-255)
 *   hm_hp     (B,J,H,W)   keypoint heat-maps         (required: decode.py:307 needs hm_score)
 *   hp_offset (B,2,H,W)   keypoint sub-pixel offset  (NULL -> +0.5, decode.py:278-280)
 *   out       (B,K,5+3J)  [x1,y1,x2,y2, score, J*(x,y), J*kp_score]
 *
 * 1 <= K <= min(H*W, CPB200_DECODE_MAX_K); 1 <= J <= CPB200_DECODE_MAX_J.
 * ONE class channel only (`heat` is (B,1,H,W), the COCO pose task): the reference's _topk additionally merges the per-class
 * top-K lists (decode.py:108-113); a multi-class heat-map is rejected by the host shims instead of being decoded wrongly.
 * Tie order (implementation-defined in the reference) is fixed: value descending, then
 * flat index ascending; nearest-candidate ties -> first (best-scored) candidate.
 * `workspace` must hold cpb200_decode_workspace_bytes(B,J,K) bytes, be 16-byte aligned and
 * ZERO-FILLED ONCE before its first use (the kernel restores the zero state itself);
 * it must not be shared by decodes running concurrently on different streams.
 * ---------------------------------------------------------------------------------- */
size_t cpb200_decode_workspace_bytes(int B, int J, int K);

int cpb200_multi_pose_decode(const float *heat, const float *wh, const float *kps,
                             const float *reg, const float *hm_hp, const float *hp_offset,
                             float *out, int B, int H, int W, int J, int K,
                             int apply_sigmoid, void *workspace, size_t workspace_bytes,
                             void *stream);

/* Same, with the detector's back-projection fused into the epilogue: replaces, in addition,
 * lib/detectors/multi_pose.py:62-71 `post_process` -> lib/utils/post_process.py:8-19
 * `multi_pose_post_process` -> lib/utils/image.py:19-24,63-66 (`transform_preds` / `affine_transform`, a Python
 * loop over 1 900 points per image in the reference).  `affine` is (B,6) fp32 on the device: per image the
 * row-major 2x3 inverse crop matrix of `get_affine_transform(c, s, 0, (out_w, out_h), inv=1)`
 * (lib/utils/image.py:27-60), optionally pre-divided by the test scale.  Every (x,y) of the box corners and
 * keypoints is mapped to original-image pixels; scores are untouched. */
int cpb200_multi_pose_decode_affine(const float *heat, const float *wh, const float *kps,
                                    const float *reg, const float *hm_hp, const float *hp_offset,
                                    const float *affine, float *out, int B, int H, int W, int J, int K,
                                    int apply_sigmoid, void *workspace, size_t workspace_bytes,
                                    void *stream);

/* In-place logistic on n floats — lib/detectors/multi_pose.py:35-37 `hm.sigmoid_()`. */
int cpb200_sigmoid_inplace(float *x, size_t n, void *stream);

/* Flip-test averaging of the head maps in one pass — lib/detectors/multi_pose.py:45-53 with
 * flip_tensor / flip_lr / flip_lr_off (lib/models/utils.py:27-47, which round-trip through numpy on the host).
 * Inputs are the NCHW fp32 maps of 2P images ordered [image, mirrored image] per pair (base_detector.py:54-55);
 * outputs hold P images: o = (a[2p] + flipped(a[2p+1])) / 2, where `flipped` reverses W, maps joint j to
 * flip_perm[j] for hps / hm_hp and negates the x offsets (even hps channels).  hm_hp / o_hm_hp may be NULL.
 * flip_perm is a HOST array of J ints (the permutation generated by flip_idx [[1,2],[3,4],...]). */
int cpb200_flip_merge(const float *hm, const float *wh, const float *hps, const float *hm_hp, float *o_hm, float *o_wh,
                      float *o_hps, float *o_hm_hp, int P, int H, int W, int J, int num_classes, const int *flip_perm,
                      void *stream);

/* Device part of BaseDetector.pre_process (lib/detectors/base_detector.py:44-55): cv2.warpAffine(INTER_LINEAR,
 * constant-0 border) of an 8-bit HWC image with the 2x3 `trans_input` matrix (HOST array of 6 doubles, as returned
 * by get_affine_transform), then ((u/255 - mean)/std) in double -> fp32, HWC -> CHW into out[0]; with flip != 0 the
 * horizontally mirrored copy is written to out[1] (base_detector.py:54-55).  Bit-exact with OpenCV's fixed-point
 * path (verified against cv2 4.13).  img and out are device pointers; mean / stdv are HOST arrays of 3 floats. */
int cpb200_pre_process(const unsigned char *img, int h, int w, const double *trans_input, float *out, int out_h, int out_w,
                       const float *mean, const float *stdv, int flip, void *stream);

/* One image of cpb200_pre_process_batch (64 bytes, lives in caller-owned DEVICE memory). */
typedef struct cpb200_pre_image {
  int64_t offset;            /* byte offset of the image's first pixel in `imgs` */
  int32_t h, w;              /* image size; HWC uint8 BGR, rows packed (pitch 3*w bytes) */
  double trans_input[6];     /* the forward 2x3 matrix of get_affine_transform(c, s, 0, [out_w, out_h]), row-major */
} cpb200_pre_image;

/* cpb200_pre_process for B images in one launch (grid over image x pixel); cpb200_pre_process is its B = 1 case and
 * every image comes out bit-identical to it.  `imgs` is one device buffer holding all images, `table` a DEVICE array
 * of B cpb200_pre_image; all images share the output size (out_h, out_w).  out is (B,3,out_h,out_w), or with
 * flip != 0 (2B,3,out_h,out_w) ordered [img_0, mirror_0, img_1, mirror_1, ...] (the pair layout cpb200_flip_merge
 * reads).  mean / stdv are HOST arrays of 3 floats.  1 <= B <= 65535. */
int cpb200_pre_process_batch(const unsigned char *imgs, const cpb200_pre_image *table, int B, float *out, int out_h,
                             int out_w, const float *mean, const float *stdv, int flip, void *stream);

/* soft_nms_39 (lib/external/nms.pyx:172-275) on a DEVICE (N,56) fp32 array, in place, same semantics as the
 * reference's Cython routine (score decay: 0 hard / 1 linear / 2 gaussian; rows below `threshold` are removed by the
 * swap-with-last walk; columns 0..38 travel with a row, 39..55 stay).  *keep_count (device int, may be NULL)
 * receives the number of surviving rows.  One CTA; N*232 bytes of shared memory (N <= 882). */
int cpb200_soft_nms_39(float *boxes, int N, float sigma, float Nt, float threshold, int method, int *keep_count,
                       void *stream);

/* The same for B images at once: boxes is (B,N,56), one CTA per image, keep_counts (device, B ints, may be NULL)
 * receives each image's surviving rows.  cpb200_soft_nms_39 is its B = 1 case.  N <= 882, B <= 65535. */
int cpb200_soft_nms_39_batch(float *boxes, int B, int N, float sigma, float Nt, float threshold, int method,
                             int *keep_counts, void *stream);


/* ------------------------------------------------------------------------------------
 * Network forward.  Replaces `BackBoneWithHead.forward` (lib/models/model.py:57-59): the
 * backbone modules of lib/models/backbones/pose_dla_dcn.py (DLA-34 + DCN IDAUp) /
 * msra_resnet.py (ResNet-50 + deconvs), the vendored `_ext.dcn_v2_forward`
 * (lib/models/backbones/DCNv2/src/dcn_v2.h:9-39, src/cuda/dcn_v2_cuda.cu:42-172,
 * src/cuda/dcn_v2_im2col_cuda.cu:125-195) and `KeypointHead.forward`
 * (lib/models/heads/keypoint.py:40-42).
 *
 * The host (Python graph builder, centerpose_b200/plan.py) lowers the module tree to a flat
 * program of fused ops — eval-mode BatchNorm folded into weights/bias, ReLU / residual-add /
 * channel-concat fused into the producing or consuming op — and hands it over as an array of
 * cpb200_op.  cpb200_run_ops enqueues the whole program on `stream` (one C call per forward).
 *
 * Activations are NHWC (channels innermost), dtype CPB200_F32 or CPB200_BF16 (fp32
 * accumulate either way).  The network input is the reference's NCHW fp32 image batch and
 * the six head maps are written NCHW fp32, exactly what lib/models/decode.py consumes.
 * ---------------------------------------------------------------------------------- */
#define CPB200_F32 0
#define CPB200_BF16 1
/* Split-operand activations ("x2" precisions): every fp32 value v is stored as TWO 16-bit planes, hi = rn16(v) and
 * lo = rn16(v - hi); a tensor of shape (B,H,W,C) is the hi plane followed by the lo plane, each dense NHWC, i.e. a
 * (2,B,H,W,C) array.  The tensor-core kernels evaluate a*b as a_hi*b_hi + a_hi*b_lo + a_lo*b_hi into one fp32
 * accumulator, which reproduces the reference's fp32 arithmetic (dcn_v2_cuda.cu:58 `scalar_t = float`, cuDNN fp32
 * convs) to ~2^-22 (fp16 planes; activations must stay within +-65504, the epilogues saturate) or ~2^-16 (bf16
 * planes, full fp32 range).  Weights of such ops are packed as two planes as well (centerpose_b200/plan.py). */
#define CPB200_BF16X2 2
#define CPB200_F16X2 3

enum cpb200_op_type {
  CPB200_OP_CONV = 1,        /* k x k conv (+bias)(+residual)(+ReLU); up to 4 channel-concatenated inputs */
  CPB200_OP_STEM = 2,        /* NCHW fp32 image -> NHWC, small-Cin direct conv (+bias+activation); with CPB200_FLAG_TC
                                (7x7, Cin 3, stride 1/2, cout 16/64, bf16) the im2col is built in shared memory and
                                the arithmetic runs on wgmma (weight = pre-swizzled operand image, plan.py)     */
  CPB200_OP_MAXPOOL = 3,     /* k x k / stride s / pad p max-pool, NHWC                                     */
  CPB200_OP_DWDECONV_ADD = 4,/* depthwise ConvTranspose2d(k=2f,s=f,p=f/2) (+ skip add), NHWC  (IDAUp up_*) */
  CPB200_OP_DCN = 5,         /* modulated deformable 3x3 conv (DCNv2 forward) (+bias)(+ReLU)                */
  CPB200_OP_IM2COL_W = 6,    /* NCHW fp32 image -> NHWC act: channel s*cin+c = x[c, h, w+s-pad_w], s < kw, zero-padded
                                to `cout` channels.  Turns the 7x7 stem into a 7x1 tensor-core conv (K = 7 x 32).   */
  CPB200_OP_UPSAMPLE_ADD = 7,/* nearest-neighbour upsample x `stride` (power of two) of src[0] (+ aux skip add)(+ReLU),
                                NHWC  (HRNet fuse_layers, pose_higher_hrnet.py:186-187,224-232)                     */
  CPB200_OP_DWCONV = 8,      /* depthwise k x k conv, stride s, pad k/2 (+bias)(+activation); weight fp32 [k*k][C]
                                (MobileNetV3 Block.conv2, mobilenetv3.py:124-127)                                   */
  CPB200_OP_AVGPOOL = 9,     /* global average pool (B,H,W,C) -> (B,1,1,C)  (SeModule, mobilenetv3.py:100)           */
  CPB200_OP_SCALE_ADD = 10,  /* dst = src[0] * res[b,c] (+ aux skip): SE gate + block shortcut (mobilenetv3.py:111,146);
                                `res` is the (B,1,1,C) gate vector                                                  */
  CPB200_OP_CONVERT = 11,    /* NHWC activation (B,H,W,cin[0]) between fp32 and the split 16-bit pair layout named by
                                act_dtype (CPB200_BF16X2 / CPB200_F16X2): fp32 -> planes, or planes -> fp32 with
                                CPB200_FLAG_TO_F32.  Lets ops without a native split kernel run on fp32 in between.   */
  CPB200_OP_S2D = 12,        /* space-to-depth of the network input for stride-2 stems in split precisions: NCHW fp32
                                (B,3,H,W) (H, W even) -> split NHWC planes (B,H/2,W/2,16), channel (py*2+px)*3 + c =
                                x[c][2h+py][2w+px], channels 12..15 zero.  A k x k / stride-2 / pad k/2 stem
                                (msra_resnet.py:116-117 7x7, pose_higher_hrnet.py:283-284 3x3) is then a stride-1
                                (k+1)/2+1-tap conv over 16 channels on the tensor-core path; src[0] is read live.   */
  CPB200_OP_AVGPOOL2 = 13,   /* 2x2 / stride-2 average pool, NHWC, floor mode, no padding: (B,H,W,C) -> (B,H/2,W/2,C)
                                with Ho == H/2, Wo == W/2, H, W >= 2, C % 4 == 0, one dense input
                                (HarDNet nn.AvgPool2d(2, 2), hardnet.py:141).  All four activation dtypes.          */
  CPB200_OP_RESIZE_BILINEAR = 14 /* bilinear resize with align_corners=True, NHWC: (B,H,W,C) -> (B,Ho,Wo,C), Ho, Wo >= 1,
                                C % 4 == 0, one dense input (HarDNet TransitionUp, hardnet.py:95-100).  PyTorch's
                                arithmetic in fp32: scale = (in-1)/(out-1) (0 when out == 1), src = scale*dst,
                                i0 = (int)src, i1 = i0 + (i0 < in-1), l1 = src - i0, l0 = 1 - l1; the vertical blend
                                of the two horizontal blends.  All four activation dtypes.                          */
};
/* A dense ConvTranspose2d(k4,s2,p1) (msra_resnet.py:168-193) is lowered by the host into four
 * 2x2 CONV ops, one per output parity, using pad_h/pad_w and the strided-output fields below. */

#define CPB200_FLAG_RELU 1u          /* ReLU in the epilogue                                     */
#define CPB200_FLAG_OUT_NCHW_F32 2u  /* write fp32 NCHW into dst (channel slice out_ch_off..)    */
#define CPB200_FLAG_OUT_F32 4u       /* write fp32 NHWC regardless of act_dtype (DCN offsets)    */
#define CPB200_FLAG_TC 8u            /* run on the wgmma tensor-core path (16-bit operands)       */
#define CPB200_FLAG_HSWISH 16u       /* x * relu6(x + 3) / 6 in the epilogue (mobilenetv3.py:84-87)   */
#define CPB200_FLAG_HSIGMOID 32u     /* relu6(x + 3) / 6 in the epilogue     (mobilenetv3.py:90-93)   */
#define CPB200_FLAG_TO_F32 64u       /* CPB200_OP_CONVERT direction: split planes -> fp32                    */

typedef struct cpb200_op {
  int32_t type;              /* enum cpb200_op_type */
  uint32_t flags;
  int32_t act_dtype;         /* CPB200_F32 / CPB200_BF16 / CPB200_BF16X2 / CPB200_F16X2: dtype of src/res/dst activations */
  int32_t B, H, W;           /* input batch / spatial size  */
  int32_t Ho, Wo;            /* output spatial size         */
  int32_t nsrc;              /* number of concatenated inputs (1..4) */
  int32_t cin[4];            /* channels of each input      */
  int32_t cout;              /* output channels             */
  int32_t kh, kw, stride;
  int32_t pad_h, pad_w;      /* top / left zero padding (bottom / right follow from the bounds) */
  int32_t out_ch_off, out_ch_total;   /* NCHW output: channel offset / total channels of dst */
  int32_t Hd, Wd;            /* spatial size of the dst tensor (== Ho,Wo unless strided output) */
  int32_t out_sy, out_sx, out_oy, out_ox; /* output pixel (ho,wo) lands at (ho*out_sy+out_oy, wo*out_sx+out_ox) */
  int32_t aux_pitch;         /* DCN: channel pitch of the offset/mask tensor (27, or 32 when padded for 16-byte rows) */
  const void *src[4];        /* inputs (NHWC act_dtype; STEM: NCHW fp32) */
  const void *res;           /* optional residual, same shape/dtype as the NHWC output */
  const void *aux;           /* DCN: offset/mask tensor (B,H,W,aux_pitch) fp32, channels [0,18) offsets, [18,27) mask; DWDECONV_ADD / UPSAMPLE_ADD: skip */
  void *dst;
  const void *weight;        /* packed by centerpose_b200/plan.py, layout per op type */
  const float *bias;         /* fp32 [cout] (BatchNorm folded), may be NULL */
  void *tc;                  /* opaque tensor-core state prepared by cpb200_prepare_ops, or NULL */
  int32_t src_pitch[4];      /* channel pitch (elements per pixel) of each input when it is a channel SLICE of a wider NHWC
                                tensor (src[i] then points at the slice's first channel); 0 = dense (pitch == cin[i]).
                                Used by the fused head: one 3x3 conv produces all six hidden maps, the 1x1 convs read slices */
  float acc_scale;           /* split-operand ops: the accumulator is multiplied by this (a power of two) before the bias is
                                added — the inverse of the scale the host applied to the weights; 0 is read as 1     */
  int32_t reserved_;
} cpb200_op;

/* Validate the program and build device-side descriptors (TMA tensor maps) for ops flagged
 * CPB200_FLAG_TC.  Must be called once after the INPUT activation / weight pointers in `ops` are final (they are
 * baked into the tensor maps).  `dst`, `res`, `bias`, `aux` and the STEM op's `src[0]` are read from the op at every
 * cpb200_run_ops call and may be re-pointed between runs (the model binds fresh output tensors per forward). */
int cpb200_prepare_ops(cpb200_op *ops, int n);
/* Release what cpb200_prepare_ops attached. */
int cpb200_release_ops(cpb200_op *ops, int n);
/* Enqueue ops[0..n) in order on `stream`. */
int cpb200_run_ops(const cpb200_op *ops, int n, void *stream);
/* sizeof(cpb200_op) as compiled, so the host binding can verify its struct layout. */
size_t cpb200_sizeof_op(void);

/* Hardware probe (diagnostics only, not on the product path): one smem halo tile serving all nine
 * taps of a 3x3 conv through shifted wgmma descriptors.  x (1,18,10,64) bf16 NHWC, w (9,64,64) bf16
 * [tap][cout][cin], out (128,64) fp32 with row = th*8 + tw.  variant 0/1 = descriptor base_offset 0 /
 * (start>>7)&7.  See centerpose_b200/csrc/probe.cu and tools/halo_probe.py. */
int cpb200_probe_halo(const void *x, const void *w, float *out, int variant, void *stream);
/* TMA box-throughput probe: streams a (N,H,W,C) bf16 tensor through 4-D boxes {C,box_w,box_h,1} stepping
 * (step_w,step_h) with an N-deep smem ring on every SM (tools/tma_probe.py). */
int cpb200_probe_tma(const void *x, int C, int W, int H, int N, int box_w, int box_h, int step_w, int step_h,
                     int stages, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CENTERPOSE_B200_H_ */

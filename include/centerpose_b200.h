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
/* Route log (diagnostics and tests): cpb200_route_log_start() clears the log and records every kernel the network-op
 * entry points (cpb200_run_ops) launch from then on; cpb200_route_log_read() stops recording and writes the demangled
 * kernel names into buf, one per line in launch order.  Returns the number of launches, or -1 (cpb200_last_error())
 * when buf is too small or a name cannot be read.  Recording is process-wide. */
void cpb200_route_log_start(void);
int cpb200_route_log_read(char *buf, size_t n);

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

/* One image of cpb200_resize_linear_u8_batch (32 bytes, lives in caller-owned DEVICE memory).  All sizes >= 1. */
typedef struct cpb200_resize_image {
  int64_t src_offset;        /* byte offset of the source image's first pixel in `src` */
  int32_t h, w;              /* source size; HWC uint8 BGR, rows packed (pitch 3*w bytes) */
  int64_t dst_offset;        /* byte offset of the resized image's first pixel in `dst` */
  int32_t new_h, new_w;      /* resized size, rows packed (pitch 3*new_w bytes) */
} cpb200_resize_image;

/* cv2.resize(img, (new_w, new_h)) with the default INTER_LINEAR on 8-bit BGR images, the first step of
 * BaseDetector.pre_process at a test scale != 1 (lib/detectors/base_detector.py:33-34).  Bit-exact with OpenCV's
 * fixed-point path (11-bit coefficients; verified against cv2 4.13 for up- and downscales).  B images of any sizes in
 * one launch: `src` and `dst` are device buffers, `table` a DEVICE array of B cpb200_resize_image whose sizes the
 * caller has checked (the kernel trusts them).  The output regions must not overlap the inputs.  1 <= B <= 65535. */
int cpb200_resize_linear_u8_batch(const unsigned char *src, const cpb200_resize_image *table, int B, unsigned char *dst,
                                  void *stream);

/* One Huffman table of cpb200_jpeg_decode_batch (1424 bytes, 4-byte aligned in `src`).  lut[b] for the next 9 bits b
 * is (code length << 8 | symbol), or 0 when the code is longer than 9 bits; then maxcode[l] (largest code of length
 * l, -1 if none, maxcode[17] = INT32_MAX) and valoff[l] (index in val of the first code of length l, minus that code),
 * T.81 F.2.2.3.  The code lengths form a prefix code; DC symbols are <= 15. */
typedef struct cpb200_jpeg_huff {
  uint16_t lut[512];
  int32_t maxcode[18];
  int32_t valoff[18];
  uint8_t val[256];
} cpb200_jpeg_huff;

/* One scan of a progressive image of cpb200_jpeg_decode_batch (40 bytes, 8-byte aligned in `src`). */
typedef struct cpb200_jpeg_scan {
  int64_t seg_offset;        /* in `src`: nseg x {int64 start, end}, the byte ranges of the scan's entropy-coded
                                segments, 8-byte aligned */
  int32_t nseg;              /* ceil(units / restart_interval), or 1 */
  int32_t restart_interval;  /* units per segment, 0: one segment.  A unit is an MCU when the scan has several
                                components, else one block of that component's own grid, ceil(ceil(w * h_c / hs) / 8)
                                x ceil(ceil(h * v_c / vs) / 8) (T.81 A.2.2) */
  int32_t ncomp;             /* components in the scan, 1..3 (1 for an AC scan) */
  uint8_t comp[4];           /* their indices 0..2, increasing */
  uint8_t dc_tbl[4], ac_tbl[4];  /* per scan component: index of its DC table (first DC scan) or AC table (AC scan)
                                    at the image's huff_offset */
  uint8_t ss, se, ah, al;    /* spectral selection and successive approximation, legal under T.81 G.1.1.1 */
  int32_t pad;
} cpb200_jpeg_scan;

/* One image of cpb200_jpeg_decode_batch (480 bytes, lives in caller-owned DEVICE memory).  Offsets are bytes. */
typedef struct cpb200_jpeg_image {
  int64_t seg_offset;        /* in `src`: nseg x {int64 start, end}, the byte ranges in `src` of the entropy-coded
                                segments (restart intervals; the whole scan without DRI), 8-byte aligned */
  int64_t huff_offset;       /* in `src`: the image's cpb200_jpeg_huff tables, 4-byte aligned */
  int64_t coef_offset;       /* in `workspace`: int16 coefficient blocks, 128 bytes per block, 16-byte aligned */
  int64_t plane_offset;      /* in `workspace`: uint8 component planes, 64 bytes per block */
  int64_t dst_offset;        /* in `dst`: the decoded HWC uint8 BGR image, rows packed, size after orientation */
  int32_t h, w;              /* coded size, 1..65500 */
  int32_t ncomp;             /* 1 (grayscale) or 3 (YCbCr) */
  int32_t hs, vs;            /* luma sampling factors, each 1 or 2 (1, 1 for grayscale); chroma is sampled (1, 1) */
  int32_t orientation;       /* EXIF orientation 1..8, applied as cv2.imread does */
  int32_t restart_interval;  /* MCUs per segment; 0: one segment */
  int32_t nseg;              /* ceil(MCUs / restart_interval), or 1 */
  uint8_t dc_tbl[4], ac_tbl[4];  /* per component: index of its DC / AC table at huff_offset */
  uint16_t qt[3][64];        /* per component: quantisation table in natural (row-major) order */
  int64_t scan_offset;       /* progressive images: in `src`, nscan cpb200_jpeg_scan, 8-byte aligned */
  int32_t nscan;             /* 0: sequential, every field above as described.  > 0: progressive, decoded scan by
                                scan; seg_offset, restart_interval, nseg, dc_tbl and ac_tbl are unused, the scans
                                carry them */
  int32_t pad;
} cpb200_jpeg_image;

/* cv2.imread(path, IMREAD_COLOR) of sequential- and progressive-Huffman JPEG files, byte for byte (libjpeg-turbo's
 * ISLOW IDCT, fancy upsampling and integer YCbCr->BGR, then OpenCV's EXIF orientation; verified against cv2 4.13 with
 * libjpeg-turbo 3.1).  B files in one launch, either kind mixed: `src` holds the file bytes and the Huffman tables,
 * scans and segment lists the table points to, `table` is a DEVICE array of B cpb200_jpeg_image that the caller has
 * checked (the kernels trust it; see centerpose_b200/jpeg.py), `workspace` holds every image's coefficients and
 * planes (an image whose workspace would end past `workspace_bytes` is not decoded and gets status 2).  A sequential
 * image's segments are decoded by one thread each.  A progressive image is decoded by one CTA that zeroes its
 * coefficients and runs its scans in file order, one thread per segment of a scan; its progression must be complete
 * (every coefficient coded down to bit 0), since libjpeg smooths blocks otherwise.  IDCT, upsampling and colour
 * conversion then run over the whole launch.  status[b] (DEVICE int array) is 0 when image b decoded, non-zero when
 * its entropy data was bad (a code longer than 16 bits, a run past the scan's last coefficient, a refinement symbol
 * of size other than 0 or 1, or data ending before a segment's last unit); the image's pixels are then undefined,
 * other images are unaffected.  1 <= B <= 65535. */
int cpb200_jpeg_decode_batch(const unsigned char *src, const cpb200_jpeg_image *table, int B, void *workspace,
                             size_t workspace_bytes, unsigned char *dst, int *status, void *stream);

/* One image of cpb200_png_decode_batch (72 bytes, lives in caller-owned DEVICE memory).  Offsets are bytes. */
typedef struct cpb200_png_image {
  int64_t src_offset;        /* in `src`: the zlib stream (the IDAT payloads back to back), followed by >= 32 bytes
                                the decoder may read but ignores */
  int64_t src_bytes;         /* length of the zlib stream */
  int64_t palette_offset;    /* colour type 3: in `src`, 256 RGB entries (768 bytes), the ones past PLTE zero */
  int64_t ws_offset;         /* in `workspace`: the image's scanlines, 16-byte aligned */
  int64_t ws_bytes;          /* >= the inflated size rounded up to 16, plus 16 */
  int64_t dst_offset;        /* in `dst`: the decoded HWC uint8 BGR image, rows packed, size after orientation */
  int32_t h, w;              /* stored size, 1..1000000, h * w <= 2^30 */
  int32_t color_type;        /* 0 gray, 2 RGB, 3 palette, 4 gray + alpha, 6 RGBA */
  int32_t depth;             /* bits per sample, legal for the colour type: 1, 2, 4, 8 or 16 */
  int32_t interlace;         /* 0 none, 1 Adam7 */
  int32_t orientation;       /* EXIF orientation 1..8 (eXIf chunk), applied as cv2.imread does */
} cpb200_png_image;

/* cv2.imread(path, IMREAD_COLOR) of PNG files, byte for byte (libpng through OpenCV 4.13: 16-bit samples keep their
 * high byte, 1/2/4-bit gray is scaled to 8 bits, palette indices past the palette are black, gray is replicated, alpha
 * is dropped, then OpenCV's EXIF orientation).  B files in one launch: `src` holds each image's zlib stream and
 * palette, `table` is a DEVICE array of B cpb200_png_image that the caller has checked (the kernels trust it; see
 * centerpose_b200/png.py), `workspace` holds every image's scanlines (an image whose workspace would end past
 * `workspace_bytes` is not decoded and gets status 2).  One warp per image inflates its stream (stored, fixed- and
 * dynamic-Huffman blocks), one warp per image then undoes the scanline filters over 32 rows at a time and checks the
 * Adler-32, and the output pass expands the samples over the whole launch.  status[b] (DEVICE int array) is 0 when
 * image b decoded, 1 when its stream was bad (zlib header, block type, Huffman code, a distance before the start of
 * the data or past the window, more or less data than the image holds, data ending early, Adler-32, a filter type
 * above 4); the image's `dst` slot is then left unwritten, other images are unaffected.  1 <= B <= 65535. */
int cpb200_png_decode_batch(const unsigned char *src, const cpb200_png_image *table, int B, void *workspace,
                            size_t workspace_bytes, unsigned char *dst, int *status, void *stream);

/* One image of cpb200_webp_decode_batch (56 bytes, lives in caller-owned DEVICE memory).  Offsets are bytes. */
typedef struct cpb200_webp_image {
  int64_t src_offset;        /* in `src`: the file from its VP8 payload (the frame tag) to its end, followed by >= 32
                                bytes the decoder may read but ignores */
  int64_t src_bytes;         /* length of that data; the last token partition runs to its end, as in libwebp */
  int64_t ws_offset;         /* in `workspace`: the image's macroblock data and planes, 16-byte aligned */
  int64_t ws_bytes;          /* >= 16 + 1184 * (number of 16x16 macroblocks) */
  int64_t dst_offset;        /* in `dst`: the decoded HWC uint8 BGR image, rows packed, size after orientation */
  int32_t h, w;              /* frame size from the key-frame header, 1..16383 */
  int32_t orientation;       /* EXIF orientation 1..8 (the first EXIF chunk of a VP8X file), applied as cv2.imread does */
  int32_t pad;
} cpb200_webp_image;

/* cv2.imread(path, IMREAD_COLOR) of lossy WebP files (one VP8 key frame, RFC 6386), byte for byte (libwebp through
 * OpenCV 4.13: "fancy" 4:2:0 upsampling and libwebp's fixed-point YUV -> BGR, then OpenCV's EXIF orientation).  B
 * files in one launch: `src` holds each image's VP8 data, `table` is a DEVICE array of B cpb200_webp_image that the
 * caller has checked (the kernels trust it; see centerpose_b200/webp.py: the frame tag is a shown key frame, the
 * first partition fits), `workspace` holds every image's coefficients and planes (an image whose workspace would end
 * past `workspace_bytes` is not decoded and gets status 2).  One warp per image decodes the bool-coded header, modes
 * and tokens (serial within an image), one CTA per image then reconstructs and loop-filters its macroblocks along
 * diagonal wavefronts, and the output pass converts to BGR over the whole launch.  status[b] (DEVICE int array) is 0
 * when image b decoded, 1 when its stream was bad (a partition that runs out of data where libwebp's does, partition
 * sizes that do not fit); the image's `dst` slot is then left unwritten, other images are unaffected.
 * 1 <= B <= 65535. */
int cpb200_webp_decode_batch(const unsigned char *src, const cpb200_webp_image *table, int B, void *workspace,
                             size_t workspace_bytes, unsigned char *dst, int *status, void *stream);

/* Prefix-code groups a lossless WebP image may use on the device; each costs 8992 bytes of its workspace. */
#define CPB200_WEBP_LOSSLESS_MAX_GROUPS 64

/* One image of cpb200_webp_lossless_decode_batch (56 bytes, lives in caller-owned DEVICE memory).  Offsets are
 * bytes. */
typedef struct cpb200_webp_lossless_image {
  int64_t src_offset;        /* in `src`: the file from its VP8L payload (the 0x2f signature) to its end, followed by
                                >= 32 zero bytes the decoder may read but ignores */
  int64_t src_bytes;         /* length of that data; libwebp reads the bitstream to the end of the data it is given */
  int64_t ws_offset;         /* in `workspace`: the image's ARGB planes, sub-images and prefix codes, 16-byte aligned */
  int64_t ws_bytes;          /* >= centerpose_b200/webp_lossless.py workspace_bytes(w, h) */
  int64_t dst_offset;        /* in `dst`: the decoded HWC uint8 BGR image, rows packed, size after orientation */
  int32_t h, w;              /* image size from the VP8L header, 1..16384 */
  int32_t orientation;       /* EXIF orientation 1..8 (the first EXIF chunk of a VP8X file), applied as cv2.imread does */
  int32_t pad;
} cpb200_webp_lossless_image;

/* cv2.imread(path, IMREAD_COLOR) of lossless WebP files (VP8L, RFC 9649), byte for byte (libwebp through OpenCV
 * 4.13: the ARGB image with its alpha dropped, then OpenCV's EXIF orientation).  B files in one launch: `src` holds
 * each image's VP8L data, `table` is a DEVICE array of B cpb200_webp_lossless_image that the caller has checked (the
 * kernels trust it; see centerpose_b200/webp_lossless.py: the signature and version of the header, the size),
 * `workspace` holds every image's planes and codes.  One thread per image decodes the transforms, sub-images,
 * prefix codes and the LZ77 / colour-cache coded pixels (serial within an image), one CTA per image then undoes the
 * transforms, and the output pass converts to BGR over the whole launch.  status[b] (DEVICE int array) is 0 when
 * image b decoded, 1 when its stream was bad where libwebp's is (a code-length set that is empty, incomplete or
 * over-subscribed, a repeat or max_symbol past the alphabet, a transform seen twice, colour-cache bits outside 1..11,
 * a backward reference outside the image, more bits read than the data holds), 2 when its entropy image uses more
 * than CPB200_WEBP_LOSSLESS_MAX_GROUPS prefix-code groups or its workspace would end past `workspace_bytes`; the
 * image's `dst` slot is then left unwritten, other images are unaffected.  1 <= B <= 65535. */
int cpb200_webp_lossless_decode_batch(const unsigned char *src, const cpb200_webp_lossless_image *table, int B,
                                      void *workspace, size_t workspace_bytes, unsigned char *dst, int *status,
                                      void *stream);

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
  CPB200_OP_DWDECONV_ADD = 4,/* depthwise ConvTranspose2d(k=2f,s=f,p=f/2) (+ skip add), NHWC  (IDAUp up_*);
                                src[0], aux (the skip) and dst must be 16-byte aligned (16-byte vector accesses).
                                With a non-NULL `bias` (fp32 [C]): dst = act(deconv(src[0]) + bias) (+ skip), the
                                activation from the flags, for any kernel size k = kh, stride and pad_h (MobileNetV2
                                IDAUp: k 2, stride 2, pad 0, folded BN + ReLU, then + the lateral conv,
                                mobilenetv2.py:162-183).  Without a bias the activation flags must be 0.          */
  CPB200_OP_DCN = 5,         /* modulated deformable 3x3 conv (DCNv2 forward) (+bias)(+ReLU)                */
  /* 6 is retired (a horizontal-tap gather for the stem); the number is not reused */
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
  CPB200_OP_RESIZE_BILINEAR = 14,/* bilinear resize with align_corners=True, NHWC: (B,H,W,C) -> (B,Ho,Wo,C), Ho, Wo >= 1,
                                C % 4 == 0, one dense input (HarDNet TransitionUp, hardnet.py:95-100).  PyTorch's
                                arithmetic in fp32: scale = (in-1)/(out-1) (0 when out == 1), src = scale*dst,
                                i0 = (int)src, i1 = i0 + (i0 < in-1), l1 = src - i0, l0 = 1 - l1; the vertical blend
                                of the two horizontal blends.  All four activation dtypes.                          */
  CPB200_OP_HEADS = 15       /* the keypoint heads (keypoint.py:40-42) in one op: for each entry h of the cpb200_head
                                table `aux` (aux_pitch entries, 1..8)  dst_h = conv1x1_h(relu(conv3x3_h(src[0]))),
                                written NCHW fp32 (B, cout_h, Ho, Wo); the hidden maps never leave the chip.  One dense
                                input, C % 16 == 0, C <= 64, 3x3 / stride 1 / pad 1, maps >= 8 x 8; act_dtype BF16 /
                                BF16X2 / F16X2 with CPB200_FLAG_TC.  `weight` = the heads' 3x3 weights packed as for a
                                tensor-core 3x3 conv, one head after the other; `bias` = their biases, [head][hidden];
                                `cout` = the sum of the heads' channels; `dst` is unused (the table holds the outputs).
                                The results are bit-identical to each head's 3x3 conv (+ReLU) followed by its 1x1 conv
                                with NCHW output.                                                                    */
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
#define CPB200_FLAG_RELU6 128u       /* min(max(x, 0), 6) in the epilogue (MobileNetV2 ConvBNReLU, mobilenetv2.py:34-41) */
#define CPB200_FLAG_CLIP01 256u      /* min(max(x, 0), 1) in the epilogue (GhostNet SELayer's clamp, ghost_net.py:43)    */

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

/* One head of a CPB200_OP_HEADS op (a HOST array the op's `aux` points to; it is read at every cpb200_run_ops call, so
 * `dst` may be re-pointed between runs like cpb200_op.dst). */
typedef struct cpb200_head {
  int32_t hidden;            /* 3x3 output channels (the same for every head, a multiple of 128)               */
  int32_t cout;              /* 1x1 output channels, 1..48                                                      */
  const void *weight;        /* the 1x1 weights packed as for a tensor-core 1x1 conv over `hidden` channels    */
  const float *bias;         /* fp32 [cout]                                                                     */
  float acc_scale3;          /* acc_scale of the head's 3x3 conv (split precisions; 0 is read as 1)             */
  float acc_scale1;          /* acc_scale of the head's 1x1 conv                                                */
  float *dst;                /* NCHW fp32 (B, cout, Ho, Wo)                                                     */
} cpb200_head;

/* Validate the program, choose the kernel of every op flagged CPB200_FLAG_TC and build its device-side descriptors
 * (TMA tensor maps).  Must be called once after the INPUT activation / weight pointers in `ops` are final (they are
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

// cpb200_webp_decode_batch: cv2.imread(path, IMREAD_COLOR) of lossy WebP files (one VP8 key frame, RFC 6386) on the
// device, byte for byte as libwebp through OpenCV 4.13, for many files per launch.  Four kernels:
//   webp_entropy_kernel  one warp per image: the lanes clear the image's coefficients, then lane 0 reads the
//                        bool-coded frame header (segmentation, loop filter, partitions, quantisers, coefficient
//                        probability updates), every macroblock's segment, skip flag and intra modes, and its tokens,
//                        and stores the dequantised coefficients (the Y2 block already inverse-WHT'd into the luma DCs)
//                        and each macroblock's modes and loop-filter strength.  Serial within an image, as libwebp is,
//                        so the batch gives the parallelism;
//   webp_recon_kernel    one CTA per image: intra prediction plus the inverse DCT, one thread per macroblock along the
//                        diagonal wavefronts x + 2y = t (a macroblock reads its left, above-left, above and above-right
//                        neighbours, all on earlier wavefronts), into unfiltered Y, U and V planes;
//   webp_filter_kernel   one CTA per image: the normal or simple loop filter over the same wavefronts.  Macroblock
//                        (x, y) filters its left and top edges and its inner edges, reading 4 pixels and writing 3
//                        across each edge; (x - 1, y) and (x + 1, y - 1) touch the pixels it reads and come earlier in
//                        raster order and on earlier wavefronts, and macroblocks on one wavefront touch disjoint pixels,
//                        so the result is the raster-order one.  Prediction read the unfiltered planes already;
//   webp_output_kernel   one thread per output pixel: libwebp's "fancy" 4:2:0 upsampling, its fixed-point YUV -> BGR
//                        and OpenCV's EXIF orientation as an index mapping.
// The host side (centerpose_b200/webp.py) parses the RIFF container and the frame tag and builds the table; the
// kernels trust it.  Intra 4x4 modes are numbered as libwebp does: DC, TM, VE, HE, RD, VR, LD, VL, HD, HU.
#include "common.cuh"

namespace {

static_assert(sizeof(cpb200_webp_image) == 56, "cpb200_webp_image layout is part of the C ABI");

constexpr int kBps = 32;                   // stride of a thread's prediction buffers
constexpr int kMaxMbW = 1024;              // (16383 + 15) / 16
enum { B_DC = 0, B_TM, B_VE, B_HE, B_RD, B_VR, B_LD, B_VL, B_HD, B_HU };

// RFC 6386 14.1: quantiser step of the DC and AC coefficients per index 0..127
__constant__ unsigned char kDcTable[128] = {
    4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 15, 16, 17, 17,
    18, 19, 20, 20, 21, 21, 22, 22, 23, 23, 24, 25, 25, 26, 27, 28,
    29, 30, 31, 32, 33, 34, 35, 36, 37, 37, 38, 39, 40, 41, 42, 43,
    44, 45, 46, 46, 47, 48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58,
    59, 60, 61, 62, 63, 64, 65, 66, 67, 68, 69, 70, 71, 72, 73, 74,
    75, 76, 76, 77, 78, 79, 80, 81, 82, 83, 84, 85, 86, 87, 88, 89,
    91, 93, 95, 96, 98, 100, 101, 102, 104, 106, 108, 110, 112, 114, 116, 118,
    122, 124, 126, 128, 130, 132, 134, 136, 138, 140, 143, 145, 148, 151, 154, 157,
};
__constant__ unsigned short kAcTable[128] = {
    4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19,
    20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35,
    36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48, 49, 50, 51,
    52, 53, 54, 55, 56, 57, 58, 60, 62, 64, 66, 68, 70, 72, 74, 76,
    78, 80, 82, 84, 86, 88, 90, 92, 94, 96, 98, 100, 102, 104, 106, 108,
    110, 112, 114, 116, 119, 122, 125, 128, 131, 134, 137, 140, 143, 146, 149, 152,
    155, 158, 161, 164, 167, 170, 173, 177, 181, 185, 189, 193, 197, 201, 205, 209,
    213, 217, 221, 225, 229, 234, 239, 245, 249, 254, 259, 264, 269, 274, 279, 284,
};
// RFC 6386 13.4: probability that coefficient probability [t][b][c][p] is updated in the frame header
__constant__ unsigned char kCoeffsUpdateProba[4][8][3][11] = {
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    176, 246, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    223, 241, 252, 255, 255, 255, 255, 255, 255, 255, 255,
    249, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 244, 252, 255, 255, 255, 255, 255, 255, 255, 255,
    234, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    253, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 246, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    239, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 248, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    251, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    251, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 254, 253, 255, 254, 255, 255, 255, 255, 255, 255,
    250, 255, 254, 255, 254, 255, 255, 255, 255, 255, 255,
    254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    217, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    225, 252, 241, 253, 255, 255, 254, 255, 255, 255, 255,
    234, 250, 241, 250, 253, 255, 253, 254, 255, 255, 255,
    255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    223, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    238, 253, 254, 254, 255, 255, 255, 255, 255, 255, 255,
    255, 248, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    249, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 253, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    247, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    252, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    253, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 254, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    250, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    186, 251, 250, 255, 255, 255, 255, 255, 255, 255, 255,
    234, 251, 244, 254, 255, 255, 255, 255, 255, 255, 255,
    251, 251, 243, 253, 254, 255, 254, 255, 255, 255, 255,
    255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    236, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    251, 253, 253, 254, 254, 255, 255, 255, 255, 255, 255,
    255, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    248, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    250, 254, 252, 254, 255, 255, 255, 255, 255, 255, 255,
    248, 254, 249, 253, 255, 255, 255, 255, 255, 255, 255,
    255, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    246, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    252, 254, 251, 254, 254, 255, 255, 255, 255, 255, 255,
    255, 254, 252, 255, 255, 255, 255, 255, 255, 255, 255,
    248, 254, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    253, 255, 254, 254, 255, 255, 255, 255, 255, 255, 255,
    255, 251, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    245, 251, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    253, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 251, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    252, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 252, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    249, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 253, 255, 255, 255, 255, 255, 255, 255, 255,
    250, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
    255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255,
};
// RFC 6386 13.5: default coefficient probabilities [type][band][context][node]
__constant__ unsigned char kCoeffsProba0[4][8][3][11] = {
    128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    253, 136, 254, 255, 228, 219, 128, 128, 128, 128, 128,
    189, 129, 242, 255, 227, 213, 255, 219, 128, 128, 128,
    106, 126, 227, 252, 214, 209, 255, 255, 128, 128, 128,
    1, 98, 248, 255, 236, 226, 255, 255, 128, 128, 128,
    181, 133, 238, 254, 221, 234, 255, 154, 128, 128, 128,
    78, 134, 202, 247, 198, 180, 255, 219, 128, 128, 128,
    1, 185, 249, 255, 243, 255, 128, 128, 128, 128, 128,
    184, 150, 247, 255, 236, 224, 128, 128, 128, 128, 128,
    77, 110, 216, 255, 236, 230, 128, 128, 128, 128, 128,
    1, 101, 251, 255, 241, 255, 128, 128, 128, 128, 128,
    170, 139, 241, 252, 236, 209, 255, 255, 128, 128, 128,
    37, 116, 196, 243, 228, 255, 255, 255, 128, 128, 128,
    1, 204, 254, 255, 245, 255, 128, 128, 128, 128, 128,
    207, 160, 250, 255, 238, 128, 128, 128, 128, 128, 128,
    102, 103, 231, 255, 211, 171, 128, 128, 128, 128, 128,
    1, 152, 252, 255, 240, 255, 128, 128, 128, 128, 128,
    177, 135, 243, 255, 234, 225, 128, 128, 128, 128, 128,
    80, 129, 211, 255, 194, 224, 128, 128, 128, 128, 128,
    1, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    246, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    255, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    198, 35, 237, 223, 193, 187, 162, 160, 145, 155, 62,
    131, 45, 198, 221, 172, 176, 220, 157, 252, 221, 1,
    68, 47, 146, 208, 149, 167, 221, 162, 255, 223, 128,
    1, 149, 241, 255, 221, 224, 255, 255, 128, 128, 128,
    184, 141, 234, 253, 222, 220, 255, 199, 128, 128, 128,
    81, 99, 181, 242, 176, 190, 249, 202, 255, 255, 128,
    1, 129, 232, 253, 214, 197, 242, 196, 255, 255, 128,
    99, 121, 210, 250, 201, 198, 255, 202, 128, 128, 128,
    23, 91, 163, 242, 170, 187, 247, 210, 255, 255, 128,
    1, 200, 246, 255, 234, 255, 128, 128, 128, 128, 128,
    109, 178, 241, 255, 231, 245, 255, 255, 128, 128, 128,
    44, 130, 201, 253, 205, 192, 255, 255, 128, 128, 128,
    1, 132, 239, 251, 219, 209, 255, 165, 128, 128, 128,
    94, 136, 225, 251, 218, 190, 255, 255, 128, 128, 128,
    22, 100, 174, 245, 186, 161, 255, 199, 128, 128, 128,
    1, 182, 249, 255, 232, 235, 128, 128, 128, 128, 128,
    124, 143, 241, 255, 227, 234, 128, 128, 128, 128, 128,
    35, 77, 181, 251, 193, 211, 255, 205, 128, 128, 128,
    1, 157, 247, 255, 236, 231, 255, 255, 128, 128, 128,
    121, 141, 235, 255, 225, 227, 255, 255, 128, 128, 128,
    45, 99, 188, 251, 195, 217, 255, 224, 128, 128, 128,
    1, 1, 251, 255, 213, 255, 128, 128, 128, 128, 128,
    203, 1, 248, 255, 255, 128, 128, 128, 128, 128, 128,
    137, 1, 177, 255, 224, 255, 128, 128, 128, 128, 128,
    253, 9, 248, 251, 207, 208, 255, 192, 128, 128, 128,
    175, 13, 224, 243, 193, 185, 249, 198, 255, 255, 128,
    73, 17, 171, 221, 161, 179, 236, 167, 255, 234, 128,
    1, 95, 247, 253, 212, 183, 255, 255, 128, 128, 128,
    239, 90, 244, 250, 211, 209, 255, 255, 128, 128, 128,
    155, 77, 195, 248, 188, 195, 255, 255, 128, 128, 128,
    1, 24, 239, 251, 218, 219, 255, 205, 128, 128, 128,
    201, 51, 219, 255, 196, 186, 128, 128, 128, 128, 128,
    69, 46, 190, 239, 201, 218, 255, 228, 128, 128, 128,
    1, 191, 251, 255, 255, 128, 128, 128, 128, 128, 128,
    223, 165, 249, 255, 213, 255, 128, 128, 128, 128, 128,
    141, 124, 248, 255, 255, 128, 128, 128, 128, 128, 128,
    1, 16, 248, 255, 255, 128, 128, 128, 128, 128, 128,
    190, 36, 230, 255, 236, 255, 128, 128, 128, 128, 128,
    149, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    1, 226, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    247, 192, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    240, 128, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    1, 134, 252, 255, 255, 128, 128, 128, 128, 128, 128,
    213, 62, 250, 255, 255, 128, 128, 128, 128, 128, 128,
    55, 93, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128,
    202, 24, 213, 235, 186, 191, 220, 160, 240, 175, 255,
    126, 38, 182, 232, 169, 184, 228, 174, 255, 187, 128,
    61, 46, 138, 219, 151, 178, 240, 170, 255, 216, 128,
    1, 112, 230, 250, 199, 191, 247, 159, 255, 255, 128,
    166, 109, 228, 252, 211, 215, 255, 174, 128, 128, 128,
    39, 77, 162, 232, 172, 180, 245, 178, 255, 255, 128,
    1, 52, 220, 246, 198, 199, 249, 220, 255, 255, 128,
    124, 74, 191, 243, 183, 193, 250, 221, 255, 255, 128,
    24, 71, 130, 219, 154, 170, 243, 182, 255, 255, 128,
    1, 182, 225, 249, 219, 240, 255, 224, 128, 128, 128,
    149, 150, 226, 252, 216, 205, 255, 171, 128, 128, 128,
    28, 108, 170, 242, 183, 194, 254, 223, 255, 255, 128,
    1, 81, 230, 252, 204, 203, 255, 192, 128, 128, 128,
    123, 102, 209, 247, 188, 196, 255, 233, 128, 128, 128,
    20, 95, 153, 243, 164, 173, 255, 203, 128, 128, 128,
    1, 222, 248, 255, 216, 213, 128, 128, 128, 128, 128,
    168, 175, 246, 252, 235, 205, 255, 255, 128, 128, 128,
    47, 116, 215, 255, 211, 212, 255, 255, 128, 128, 128,
    1, 121, 236, 253, 212, 214, 255, 255, 128, 128, 128,
    141, 84, 213, 252, 201, 202, 255, 219, 128, 128, 128,
    42, 80, 160, 240, 162, 185, 255, 205, 128, 128, 128,
    1, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    244, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128,
    238, 1, 255, 128, 128, 128, 128, 128, 128, 128, 128,
};
// RFC 6386 12.3: key-frame 4x4 mode probabilities [above mode][left mode][tree node]
__constant__ unsigned char kBModesProba[10][10][9] = {
    231, 120, 48, 89, 115, 113, 120, 152, 112,
    152, 179, 64, 126, 170, 118, 46, 70, 95,
    175, 69, 143, 80, 85, 82, 72, 155, 103,
    56, 58, 10, 171, 218, 189, 17, 13, 152,
    114, 26, 17, 163, 44, 195, 21, 10, 173,
    121, 24, 80, 195, 26, 62, 44, 64, 85,
    144, 71, 10, 38, 171, 213, 144, 34, 26,
    170, 46, 55, 19, 136, 160, 33, 206, 71,
    63, 20, 8, 114, 114, 208, 12, 9, 226,
    81, 40, 11, 96, 182, 84, 29, 16, 36,
    134, 183, 89, 137, 98, 101, 106, 165, 148,
    72, 187, 100, 130, 157, 111, 32, 75, 80,
    66, 102, 167, 99, 74, 62, 40, 234, 128,
    41, 53, 9, 178, 241, 141, 26, 8, 107,
    74, 43, 26, 146, 73, 166, 49, 23, 157,
    65, 38, 105, 160, 51, 52, 31, 115, 128,
    104, 79, 12, 27, 217, 255, 87, 17, 7,
    87, 68, 71, 44, 114, 51, 15, 186, 23,
    47, 41, 14, 110, 182, 183, 21, 17, 194,
    66, 45, 25, 102, 197, 189, 23, 18, 22,
    88, 88, 147, 150, 42, 46, 45, 196, 205,
    43, 97, 183, 117, 85, 38, 35, 179, 61,
    39, 53, 200, 87, 26, 21, 43, 232, 171,
    56, 34, 51, 104, 114, 102, 29, 93, 77,
    39, 28, 85, 171, 58, 165, 90, 98, 64,
    34, 22, 116, 206, 23, 34, 43, 166, 73,
    107, 54, 32, 26, 51, 1, 81, 43, 31,
    68, 25, 106, 22, 64, 171, 36, 225, 114,
    34, 19, 21, 102, 132, 188, 16, 76, 124,
    62, 18, 78, 95, 85, 57, 50, 48, 51,
    193, 101, 35, 159, 215, 111, 89, 46, 111,
    60, 148, 31, 172, 219, 228, 21, 18, 111,
    112, 113, 77, 85, 179, 255, 38, 120, 114,
    40, 42, 1, 196, 245, 209, 10, 25, 109,
    88, 43, 29, 140, 166, 213, 37, 43, 154,
    61, 63, 30, 155, 67, 45, 68, 1, 209,
    100, 80, 8, 43, 154, 1, 51, 26, 71,
    142, 78, 78, 16, 255, 128, 34, 197, 171,
    41, 40, 5, 102, 211, 183, 4, 1, 221,
    51, 50, 17, 168, 209, 192, 23, 25, 82,
    138, 31, 36, 171, 27, 166, 38, 44, 229,
    67, 87, 58, 169, 82, 115, 26, 59, 179,
    63, 59, 90, 180, 59, 166, 93, 73, 154,
    40, 40, 21, 116, 143, 209, 34, 39, 175,
    47, 15, 16, 183, 34, 223, 49, 45, 183,
    46, 17, 33, 183, 6, 98, 15, 32, 183,
    57, 46, 22, 24, 128, 1, 54, 17, 37,
    65, 32, 73, 115, 28, 128, 23, 128, 205,
    40, 3, 9, 115, 51, 192, 18, 6, 223,
    87, 37, 9, 115, 59, 77, 64, 21, 47,
    104, 55, 44, 218, 9, 54, 53, 130, 226,
    64, 90, 70, 205, 40, 41, 23, 26, 57,
    54, 57, 112, 184, 5, 41, 38, 166, 213,
    30, 34, 26, 133, 152, 116, 10, 32, 134,
    39, 19, 53, 221, 26, 114, 32, 73, 255,
    31, 9, 65, 234, 2, 15, 1, 118, 73,
    75, 32, 12, 51, 192, 255, 160, 43, 51,
    88, 31, 35, 67, 102, 85, 55, 186, 85,
    56, 21, 23, 111, 59, 205, 45, 37, 192,
    55, 38, 70, 124, 73, 102, 1, 34, 98,
    125, 98, 42, 88, 104, 85, 117, 175, 82,
    95, 84, 53, 89, 128, 100, 113, 101, 45,
    75, 79, 123, 47, 51, 128, 81, 171, 1,
    57, 17, 5, 71, 102, 57, 53, 41, 49,
    38, 33, 13, 121, 57, 73, 26, 1, 85,
    41, 10, 67, 138, 77, 110, 90, 47, 114,
    115, 21, 2, 10, 102, 255, 166, 23, 6,
    101, 29, 16, 10, 85, 128, 101, 196, 26,
    57, 18, 10, 102, 102, 213, 34, 20, 43,
    117, 20, 15, 36, 163, 128, 68, 1, 26,
    102, 61, 71, 37, 34, 53, 31, 243, 192,
    69, 60, 71, 38, 73, 119, 28, 222, 37,
    68, 45, 128, 34, 1, 47, 11, 245, 171,
    62, 17, 19, 70, 146, 85, 55, 62, 70,
    37, 43, 37, 154, 100, 163, 85, 160, 1,
    63, 9, 92, 136, 28, 64, 32, 201, 85,
    75, 15, 9, 9, 64, 255, 184, 119, 16,
    86, 6, 28, 5, 64, 255, 25, 248, 1,
    56, 8, 17, 132, 137, 255, 55, 116, 128,
    58, 15, 20, 82, 135, 57, 26, 121, 40,
    164, 50, 31, 137, 154, 133, 25, 35, 218,
    51, 103, 44, 131, 131, 123, 31, 6, 158,
    86, 40, 64, 135, 148, 224, 45, 183, 128,
    22, 26, 17, 131, 240, 154, 14, 1, 209,
    45, 16, 21, 91, 64, 222, 7, 1, 197,
    56, 21, 39, 155, 60, 138, 23, 102, 213,
    83, 12, 13, 54, 192, 255, 68, 47, 28,
    85, 26, 85, 85, 128, 128, 32, 146, 171,
    18, 11, 7, 63, 144, 171, 4, 4, 246,
    35, 27, 10, 146, 174, 171, 12, 26, 128,
    190, 80, 35, 99, 180, 80, 126, 54, 45,
    85, 126, 47, 87, 176, 51, 41, 20, 32,
    101, 75, 128, 139, 118, 146, 116, 128, 85,
    56, 41, 15, 176, 236, 85, 37, 9, 62,
    71, 30, 17, 119, 118, 255, 17, 18, 138,
    101, 38, 60, 138, 55, 70, 43, 26, 142,
    146, 36, 19, 30, 171, 255, 97, 27, 20,
    138, 45, 61, 62, 219, 1, 81, 188, 64,
    32, 41, 20, 117, 151, 142, 20, 21, 163,
    112, 19, 12, 61, 195, 128, 48, 4, 24,
};

// RFC 6386 13: band of each coefficient position (16 is a sentinel), zigzag order, extra-bit probabilities of
// DCT_CAT3..6
__constant__ unsigned char kBands[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
__constant__ unsigned char kZigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
__constant__ unsigned char kCat3456[4][12] = {{173, 148, 140, 0},
                                              {176, 155, 140, 135, 0},
                                              {180, 157, 141, 134, 130, 0},
                                              {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129, 0}};
// RFC 6386 11.2: the 4x4 mode tree, leaves negated
__constant__ signed char kYModesIntra4[18] = {-B_DC, 1, -B_TM, 2, -B_VE, 3, 4, 6, -B_HE, 5,
                                              -B_RD, -B_VR, -B_LD, 7, -B_VL, 8, -B_HD, -B_HU};

// per macroblock in the workspace: its sixteen 4x4 modes (the 16x16 mode sixteen times), chroma mode, loop-filter
// strength (limit 0: not filtered), and the segment and coded skip flag the mode pass hands to the token pass
struct MbInfo {
  unsigned char imodes[16];
  unsigned char is_i4x4, uvmode, limit, ilevel, hev, inner, segment, skip, pad[8];
};
static_assert(sizeof(MbInfo) == 32, "MbInfo is 32 bytes");

// workspace of one image: 16 bytes of frame flags, then per macroblock its MbInfo and 384 int16 coefficients, then
// the Y, U and V planes padded to whole macroblocks (1184 bytes per macroblock in all; webp.py WorkspaceBytes)
struct Layout {
  int mbw, mbh, ys, uvs;
  int64_t info, coef, y, u, v, total;
};

__device__ __forceinline__ Layout layout(int w, int h) {
  Layout L;
  L.mbw = (w + 15) >> 4;
  L.mbh = (h + 15) >> 4;
  const int64_t n = (int64_t)L.mbw * L.mbh;
  L.ys = L.mbw * 16;
  L.uvs = L.mbw * 8;
  L.info = 16;
  L.coef = L.info + 32 * n;
  L.y = L.coef + 768 * n;
  L.u = L.y + 256 * n;
  L.v = L.u + 64 * n;
  L.total = L.v + 64 * n;
  return L;
}

__device__ __forceinline__ bool fits(const cpb200_webp_image &e, const Layout &L, size_t ws_bytes) {
  return e.ws_offset >= 0 && e.ws_bytes >= L.total && (uint64_t)e.ws_offset + e.ws_bytes <= ws_bytes;
}

// libwebp's boolean decoder (bit_reader): `value` holds `bits` + 8 unread bits, refilled 56 bits at a time while 8
// bytes remain, then byte by byte; past the end it shifts in one zero byte and sets `eof`, which is what makes a
// partition that ran out of data fail
struct BoolReader {
  const unsigned char *buf, *end;
  uint64_t value;
  int bits;
  uint32_t range;                          // range - 1
  int eof;

  __device__ void init(const unsigned char *s, int64_t n) {
    buf = s; end = s + n; value = 0; bits = -8; range = 254; eof = 0;
    load();
  }
  __device__ void load() {
    if (end - buf >= 8) {
      uint64_t v = 0;
#pragma unroll
      for (int k = 0; k < 7; ++k) v = v << 8 | __ldg(buf + k);
      buf += 7;
      value = value << 56 | v;
      bits += 56;
    } else if (buf < end) {
      value = value << 8 | __ldg(buf);
      ++buf;
      bits += 8;
    } else if (!eof) {
      value <<= 8;
      bits += 8;
      eof = 1;
    } else {
      bits = 0;
    }
  }
  __device__ __forceinline__ int bit(int prob) {
    uint32_t r = range;
    if (bits < 0) load();
    const int pos = bits;
    const uint32_t split = (r * (uint32_t)prob) >> 8;
    const uint32_t v = (uint32_t)(value >> pos);
    const int b = v > split;
    if (b) {
      r -= split;
      value -= (uint64_t)(split + 1) << pos;
    } else {
      r = split + 1;
    }
    const int shift = 7 ^ (31 - __clz(r));
    r <<= shift;
    bits -= shift;
    range = r - 1;
    return b;
  }
  __device__ int literal(int n) {          // n bits, most significant first
    int v = 0;
    while (n-- > 0) v |= bit(0x80) << n;
    return v;
  }
  __device__ int signed_literal(int n) {
    const int v = literal(n);
    return bit(0x80) ? -v : v;
  }
  __device__ int flag_value(int n) { return bit(0x80) ? signed_literal(n) : 0; }
};

// RFC 6386 13.2: the size of a token above one
__device__ int large_value(BoolReader &br, const unsigned char *p) {
  int v;
  if (!br.bit(p[3])) {
    v = !br.bit(p[4]) ? 2 : 3 + br.bit(p[5]);
  } else if (!br.bit(p[6])) {
    if (!br.bit(p[7])) {
      v = 5 + br.bit(159);
    } else {
      v = 7 + 2 * br.bit(165);
      v += br.bit(145);
    }
  } else {
    const int bit1 = br.bit(p[8]);
    const int bit0 = br.bit(p[9 + bit1]);
    const int cat = 2 * bit1 + bit0;
    v = 0;
    for (const unsigned char *tab = kCat3456[cat]; *tab; ++tab) v += v + br.bit(*tab);
    v += 3 + (8 << cat);
  }
  return v;
}

// the tokens of one 4x4 block from position n on with probabilities P (one block type) and context ctx; stores the
// dequantised values (truncated to int16 as libwebp does) in raster order and returns the position after the last
// token before the end of block (16 when there is none)
__device__ int get_coeffs(BoolReader &br, const unsigned char *P, int ctx, int dq0, int dq1, int n, int16_t *out) {
  const unsigned char *p = P + (kBands[n] * 3 + ctx) * 11;
  for (; n < 16; ++n) {
    if (!br.bit(p[0])) return n;
    while (!br.bit(p[1])) {
      p = P + kBands[++n] * 33;
      if (n == 16) return 16;
    }
    const unsigned char *pc = P + kBands[n + 1] * 33;
    int v;
    if (!br.bit(p[2])) {
      v = 1;
      p = pc + 11;
    } else {
      v = large_value(br, p);
      p = pc + 22;
    }
    out[kZigzag[n]] = (int16_t)((br.bit(0x80) ? -v : v) * (n > 0 ? dq1 : dq0));
  }
  return 16;
}

// RFC 6386 14.3: inverse Walsh-Hadamard transform of the Y2 block into the DCs of the 16 luma blocks
__device__ void inverse_wht(const int16_t *in, int16_t *out) {
  int tmp[16];
  for (int i = 0; i < 4; ++i) {
    const int a0 = in[0 + i] + in[12 + i], a1 = in[4 + i] + in[8 + i];
    const int a2 = in[4 + i] - in[8 + i], a3 = in[0 + i] - in[12 + i];
    tmp[0 + i] = a0 + a1;
    tmp[8 + i] = a0 - a1;
    tmp[4 + i] = a3 + a2;
    tmp[12 + i] = a3 - a2;
  }
  for (int i = 0; i < 4; ++i) {
    const int dc = tmp[0 + i * 4] + 3;
    const int a0 = dc + tmp[3 + i * 4], a1 = tmp[1 + i * 4] + tmp[2 + i * 4];
    const int a2 = tmp[1 + i * 4] - tmp[2 + i * 4], a3 = dc - tmp[3 + i * 4];
    out[(4 * i + 0) * 16] = (int16_t)((a0 + a1) >> 3);
    out[(4 * i + 1) * 16] = (int16_t)((a3 + a2) >> 3);
    out[(4 * i + 2) * 16] = (int16_t)((a0 - a1) >> 3);
    out[(4 * i + 3) * 16] = (int16_t)((a3 - a2) >> 3);
  }
}

struct Quant {
  int y1[2], y2[2], uv[2];
};

struct FilterStrength {
  unsigned char limit, ilevel, hev;
};

// lane 0 of webp_entropy_kernel: the frame header, then row by row the modes and the tokens; false where libwebp
// fails (a partition ran out of data, partition sizes that do not fit)
__device__ bool decode_frame(const unsigned char *s, int64_t size, const Layout &L, unsigned char *img,
                             unsigned char *proba, unsigned char *intra_t, unsigned char *nz_t,
                             unsigned char *nz_dc_t) {
  const uint32_t tag = s[0] | s[1] << 8 | s[2] << 16;
  const int64_t part0 = tag >> 5;
  MbInfo *info = reinterpret_cast<MbInfo *>(img + L.info);
  int16_t *coef = reinterpret_cast<int16_t *>(img + L.coef);
  BoolReader br;
  br.init(s + 10, part0);
  br.bit(0x80);                             // colour space
  br.bit(0x80);                             // clamping type (libwebp always clamps)
  // segment header (RFC 6386 9.3)
  int use_segment = br.bit(0x80), update_map = 0, absolute = 1;
  int seg_q[4] = {0, 0, 0, 0}, seg_f[4] = {0, 0, 0, 0}, seg_p[3] = {255, 255, 255};
  if (use_segment) {
    update_map = br.bit(0x80);
    if (br.bit(0x80)) {
      absolute = br.bit(0x80);
      for (int k = 0; k < 4; ++k) seg_q[k] = br.flag_value(7);
      for (int k = 0; k < 4; ++k) seg_f[k] = br.flag_value(6);
    }
    if (update_map)
      for (int k = 0; k < 3; ++k) seg_p[k] = br.bit(0x80) ? br.literal(8) : 255;
  }
  if (br.eof) return false;
  // filter header (9.4)
  int simple, level, sharpness, use_lf_delta, ref_delta0 = 0, mode_delta0 = 0, filter_type;
  simple = br.bit(0x80);
  level = br.literal(6);
  sharpness = br.literal(3);
  use_lf_delta = br.bit(0x80);
  if (use_lf_delta && br.bit(0x80)) {
    for (int k = 0; k < 4; ++k) {
      const int d = br.flag_value(6);
      if (k == 0) ref_delta0 = d;          // a key frame uses the intra-frame delta only
    }
    for (int k = 0; k < 4; ++k) {
      const int d = br.flag_value(6);
      if (k == 0) mode_delta0 = d;         // and the B_PRED mode delta
    }
  }
  filter_type = level == 0 ? 0 : simple ? 1 : 2;
  if (br.eof) return false;
  {
    // token partitions (9.5): all but the last have a 3-byte size; the last one takes the rest and may not be empty
    const int nparts = 1 << br.literal(2);
    const int64_t after = 10 + part0, rest = size - after;
    if (rest < 3 * (nparts - 1)) return false;
    BoolReader parts[8];
    int64_t start = after + 3 * (nparts - 1), left = rest - 3 * (nparts - 1);
    for (int p = 0; p < nparts - 1; ++p) {
      const unsigned char *sz = s + after + 3 * p;
      int64_t psize = sz[0] | sz[1] << 8 | sz[2] << 16;
      if (psize > left) psize = left;
      parts[p].init(s + start, psize);
      start += psize;
      left -= psize;
    }
    if (left <= 0) return false;
    parts[nparts - 1].init(s + start, left);
    // quantisers (9.6, 14.1)
    Quant dqm[4];
    {
      const int q0 = br.literal(7);
      const int dy1dc = br.flag_value(4), dy2dc = br.flag_value(4), dy2ac = br.flag_value(4);
      const int duvdc = br.flag_value(4), duvac = br.flag_value(4);
      for (int k = 0; k < 4; ++k) {
        int q = q0;
        if (use_segment) {
          q = seg_q[k];
          if (!absolute) q += q0;
        }
        auto clip = [](int v, int m) { return v < 0 ? 0 : v > m ? m : v; };
        Quant &m = dqm[k];
        m.y1[0] = kDcTable[clip(q + dy1dc, 127)];
        m.y1[1] = kAcTable[clip(q, 127)];
        m.y2[0] = kDcTable[clip(q + dy2dc, 127)] * 2;
        m.y2[1] = kAcTable[clip(q + dy2ac, 127)] * 101581 >> 16;   // x * 155 / 100 for every table entry
        if (m.y2[1] < 8) m.y2[1] = 8;
        m.uv[0] = kDcTable[clip(q + duvdc, 117)];
        m.uv[1] = kAcTable[clip(q + duvac, 127)];
      }
    }
    br.bit(0x80);                           // refresh_entropy_probs: one frame, no effect
    for (int i = 0; i < 4 * 8 * 3 * 11; ++i) {
      const unsigned char *u = &kCoeffsUpdateProba[0][0][0][0], *d = &kCoeffsProba0[0][0][0][0];
      proba[i] = br.bit(u[i]) ? (unsigned char)br.literal(8) : d[i];
    }
    const int use_skip = br.bit(0x80);
    const int skip_p = use_skip ? br.literal(8) : 0;
    // loop-filter strength per segment and per "is 4x4" (libwebp's PrecomputeFilterStrengths)
    FilterStrength fs[4][2];
    for (int k = 0; k < 4; ++k) {
      int base = level;
      if (use_segment) {
        base = seg_f[k];
        if (!absolute) base += level;
      }
      for (int i4 = 0; i4 < 2; ++i4) {
        int lv = base;
        if (use_lf_delta) {
          lv += ref_delta0;
          if (i4) lv += mode_delta0;
        }
        lv = lv < 0 ? 0 : lv > 63 ? 63 : lv;
        FilterStrength &f = fs[k][i4];
        f.limit = f.ilevel = f.hev = 0;
        if (lv > 0 && filter_type) {
          int il = lv;
          if (sharpness > 0) {
            il >>= sharpness > 4 ? 2 : 1;
            if (il > 9 - sharpness) il = 9 - sharpness;
          }
          if (il < 1) il = 1;
          f.ilevel = (unsigned char)il;
          f.limit = (unsigned char)(2 * lv + il);
          f.hev = lv >= 40 ? 2 : lv >= 15 ? 1 : 0;
        }
      }
    }
    *reinterpret_cast<int *>(img) = filter_type;

    for (int mb_y = 0; mb_y < L.mbh; ++mb_y) {
      // the row's modes from the first partition (libwebp's VP8ParseIntraModeRow)
      unsigned char intra_l[4] = {B_DC, B_DC, B_DC, B_DC};
      for (int mb_x = 0; mb_x < L.mbw; ++mb_x) {
        MbInfo &m = info[(int64_t)mb_y * L.mbw + mb_x];
        const int segment = update_map ? (!br.bit(seg_p[0]) ? br.bit(seg_p[1]) : br.bit(seg_p[2]) + 2) : 0;
        const int skip = use_skip ? br.bit(skip_p) : 0;
        const int is_i4x4 = !br.bit(145);
        unsigned char *top = intra_t + 4 * mb_x;
        if (!is_i4x4) {
          const int ymode = br.bit(156) ? (br.bit(128) ? B_TM : B_HE) : (br.bit(163) ? B_VE : B_DC);
          for (int k = 0; k < 4; ++k) top[k] = intra_l[k] = (unsigned char)ymode;
          for (int k = 0; k < 16; ++k) m.imodes[k] = (unsigned char)ymode;
        } else {
          for (int y = 0; y < 4; ++y) {
            int ymode = intra_l[y];
            for (int x = 0; x < 4; ++x) {
              const unsigned char *prob = kBModesProba[top[x]][ymode];
              int i = kYModesIntra4[br.bit(prob[0])];
              while (i > 0) i = kYModesIntra4[2 * i + br.bit(prob[i])];
              ymode = -i;
              top[x] = (unsigned char)ymode;
              m.imodes[4 * y + x] = (unsigned char)ymode;
            }
            intra_l[y] = (unsigned char)ymode;
          }
        }
        m.uvmode = (unsigned char)(!br.bit(142) ? B_DC : !br.bit(114) ? B_VE : br.bit(183) ? B_TM : B_HE);
        m.is_i4x4 = (unsigned char)is_i4x4;
        m.segment = (unsigned char)segment;
        m.skip = (unsigned char)skip;
      }
      if (br.eof) return false;
      // the row's tokens from its partition (VP8DecodeMB / ParseResiduals)
      BoolReader &tb = parts[mb_y & (nparts - 1)];
      unsigned char nz_l = 0, nz_dc_l = 0;
      for (int mb_x = 0; mb_x < L.mbw; ++mb_x) {
        MbInfo &m = info[(int64_t)mb_y * L.mbw + mb_x];
        const int segment = m.segment, is_i4x4 = m.is_i4x4;
        int skip = m.skip;
        if (!skip) {
          const Quant &q = dqm[segment];
          int16_t *dst = coef + ((int64_t)mb_y * L.mbw + mb_x) * 384;
          const unsigned char *ac_proba;
          int first;
          uint32_t non_zero = 0;
          if (!is_i4x4) {
            int16_t dc[16];
            for (int k = 0; k < 16; ++k) dc[k] = 0;
            const int ctx = nz_dc_t[mb_x] + nz_dc_l;
            const int nz = get_coeffs(tb, proba + 1 * 264, ctx, q.y2[0], q.y2[1], 0, dc);
            nz_dc_t[mb_x] = nz_dc_l = (unsigned char)(nz > 0);
            inverse_wht(dc, dst);
            first = 1;
            ac_proba = proba + 0 * 264;
          } else {
            first = 0;
            ac_proba = proba + 3 * 264;
          }
          unsigned tnz = nz_t[mb_x] & 0x0f, lnz = nz_l & 0x0f;
          for (int y = 0; y < 4; ++y) {
            int l = lnz & 1;
            for (int x = 0; x < 4; ++x) {
              const int ctx = l + (tnz & 1);
              const int nz = get_coeffs(tb, ac_proba, ctx, q.y1[0], q.y1[1], first, dst);
              l = nz > first;
              tnz = (tnz >> 1) | (l << 7);
              non_zero |= (nz > 1) | (dst[0] != 0);
              dst += 16;
            }
            tnz >>= 4;
            lnz = (lnz >> 1) | (l << 7);
          }
          unsigned out_t = tnz, out_l = lnz >> 4;
          for (int ch = 0; ch < 4; ch += 2) {
            tnz = nz_t[mb_x] >> (4 + ch);
            lnz = nz_l >> (4 + ch);
            for (int y = 0; y < 2; ++y) {
              int l = lnz & 1;
              for (int x = 0; x < 2; ++x) {
                const int ctx = l + (tnz & 1);
                const int nz = get_coeffs(tb, proba + 2 * 264, ctx, q.uv[0], q.uv[1], 0, dst);
                l = nz > 0;
                tnz = (tnz >> 1) | (l << 3);
                non_zero |= (nz > 1) | (dst[0] != 0);
                dst += 16;
              }
              tnz >>= 2;
              lnz = (lnz >> 1) | (l << 5);
            }
            out_t |= (tnz << 4) << ch;
            out_l |= (lnz & 0xf0) << ch;
          }
          nz_t[mb_x] = (unsigned char)out_t;
          nz_l = (unsigned char)out_l;
          skip = !non_zero;
        } else {
          nz_t[mb_x] = nz_l = 0;
          if (!is_i4x4) nz_dc_t[mb_x] = nz_dc_l = 0;
        }
        const FilterStrength &f = fs[segment][is_i4x4];
        m.limit = f.limit;
        m.ilevel = f.ilevel;
        m.hev = f.hev;
        m.inner = (unsigned char)(is_i4x4 | !skip);
        if (tb.eof) return false;
      }
    }
  }
  return true;
}

// grid B CTAs x 32 threads: CTA b entropy-decodes image b into its workspace.  status 1 for a bad stream (a
// partition that ran out of data, bad partition sizes), 2 when the workspace does not fit
__global__ void __launch_bounds__(32) webp_entropy_kernel(const unsigned char *__restrict__ src,
                                                          const cpb200_webp_image *__restrict__ table,
                                                          unsigned char *__restrict__ ws, size_t ws_bytes,
                                                          int *__restrict__ status) {
  __shared__ unsigned char proba[4 * 8 * 3 * 11];
  __shared__ unsigned char intra_t[4 * kMaxMbW];
  __shared__ unsigned char nz_t[kMaxMbW], nz_dc_t[kMaxMbW];
  const cpb200_webp_image &e = table[blockIdx.x];
  const Layout L = layout(e.w, e.h);
  if (!fits(e, L, ws_bytes)) {
    if (threadIdx.x == 0) status[blockIdx.x] = 2;
    return;
  }
  unsigned char *img = ws + e.ws_offset;
  {
    uint4 *c = reinterpret_cast<uint4 *>(img + L.coef);
    const int64_t n16 = (int64_t)L.mbw * L.mbh * 48;
    for (int64_t i = threadIdx.x; i < n16; i += blockDim.x) c[i] = make_uint4(0, 0, 0, 0);
  }
  for (int i = threadIdx.x; i < 4 * L.mbw; i += blockDim.x) intra_t[i] = B_DC;
  for (int i = threadIdx.x; i < L.mbw; i += blockDim.x) nz_t[i] = nz_dc_t[i] = 0;
  __syncthreads();
  if (threadIdx.x != 0) return;

  status[blockIdx.x] = decode_frame(src + e.src_offset, e.src_bytes, L, img, proba, intra_t, nz_t, nz_dc_t) ? 0 : 1;
}

__device__ __forceinline__ unsigned char clip8(int v) { return (unsigned char)(v < 0 ? 0 : v > 255 ? 255 : v); }
__device__ __forceinline__ int avg3(int a, int b, int c) { return (a + 2 * b + c + 2) >> 2; }
__device__ __forceinline__ int avg2(int a, int b) { return (a + b + 1) >> 1; }

// RFC 6386 14.3 inverse DCT (libwebp's TransformOne), added to the prediction in place
__device__ void idct_add(const int16_t *in, unsigned char *dst) {
  auto mul1 = [](int a) { return ((a * 20091) >> 16) + a; };
  auto mul2 = [](int a) { return (a * 35468) >> 16; };
  int C[16];
  bool any = false;
  for (int i = 0; i < 16; ++i) any |= in[i] != 0;
  if (!any) return;
  for (int i = 0; i < 4; ++i) {
    const int a = in[i] + in[8 + i], b = in[i] - in[8 + i];
    const int c = mul2(in[4 + i]) - mul1(in[12 + i]), d = mul1(in[4 + i]) + mul2(in[12 + i]);
    C[4 * i + 0] = a + d;
    C[4 * i + 1] = b + c;
    C[4 * i + 2] = b - c;
    C[4 * i + 3] = a - d;
  }
  for (int i = 0; i < 4; ++i) {
    const int dc = C[i] + 4;
    const int a = dc + C[8 + i], b = dc - C[8 + i];
    const int c = mul2(C[4 + i]) - mul1(C[12 + i]), d = mul1(C[4 + i]) + mul2(C[12 + i]);
    unsigned char *r = dst + i * kBps;
    r[0] = clip8(r[0] + ((a + d) >> 3));
    r[1] = clip8(r[1] + ((b + c) >> 3));
    r[2] = clip8(r[2] + ((b - c) >> 3));
    r[3] = clip8(r[3] + ((a - d) >> 3));
  }
}

__device__ void true_motion(unsigned char *dst, int size) {
  const unsigned char *top = dst - kBps;
  for (int y = 0; y < size; ++y)
    for (int x = 0; x < size; ++x) dst[y * kBps + x] = clip8(top[x] + dst[y * kBps - 1] - top[-1]);
}

// 16x16 luma or 8x8 chroma prediction; DC at the frame's top or left edge averages what exists (128 at the corner)
__device__ void predict_block(unsigned char *dst, int size, int mode, int mb_x, int mb_y) {
  if (mode == B_DC) {
    const int shift = size == 16 ? 4 : 3;
    int dc;
    if (mb_x > 0 && mb_y > 0) {
      dc = size;
      for (int j = 0; j < size; ++j) dc += dst[j - kBps] + dst[j * kBps - 1];
      dc >>= shift + 1;
    } else if (mb_y > 0) {
      dc = size >> 1;
      for (int j = 0; j < size; ++j) dc += dst[j - kBps];
      dc >>= shift;
    } else if (mb_x > 0) {
      dc = size >> 1;
      for (int j = 0; j < size; ++j) dc += dst[j * kBps - 1];
      dc >>= shift;
    } else {
      dc = 0x80;
    }
    for (int y = 0; y < size; ++y)
      for (int x = 0; x < size; ++x) dst[y * kBps + x] = (unsigned char)dc;
  } else if (mode == B_TM) {
    true_motion(dst, size);
  } else if (mode == B_VE) {
    for (int y = 0; y < size; ++y)
      for (int x = 0; x < size; ++x) dst[y * kBps + x] = dst[x - kBps];
  } else {
    for (int y = 0; y < size; ++y)
      for (int x = 0; x < size; ++x) dst[y * kBps + x] = dst[y * kBps - 1];
  }
}

// RFC 6386 12.3 subblock prediction (libwebp's VP8PredLuma4)
__device__ void predict4(unsigned char *dst, int mode) {
#define DST(x, y) dst[(x) + (y) * kBps]
  const int I = dst[-1], J = dst[-1 + kBps], K = dst[-1 + 2 * kBps], L = dst[-1 + 3 * kBps];
  const int X = dst[-1 - kBps], A = dst[-kBps], B = dst[1 - kBps], C = dst[2 - kBps], D = dst[3 - kBps];
  const int E = dst[4 - kBps], F = dst[5 - kBps], G = dst[6 - kBps], H = dst[7 - kBps];
  switch (mode) {
    case B_DC: {
      int dc = 4;
      for (int i = 0; i < 4; ++i) dc += dst[i - kBps] + dst[-1 + i * kBps];
      dc >>= 3;
      for (int y = 0; y < 4; ++y)
        for (int x = 0; x < 4; ++x) DST(x, y) = (unsigned char)dc;
      break;
    }
    case B_TM: true_motion(dst, 4); break;
    case B_VE: {
      const int v[4] = {avg3(X, A, B), avg3(A, B, C), avg3(B, C, D), avg3(C, D, E)};
      for (int y = 0; y < 4; ++y)
        for (int x = 0; x < 4; ++x) DST(x, y) = (unsigned char)v[x];
      break;
    }
    case B_HE: {
      const int v[4] = {avg3(X, I, J), avg3(I, J, K), avg3(J, K, L), avg3(K, L, L)};
      for (int y = 0; y < 4; ++y)
        for (int x = 0; x < 4; ++x) DST(x, y) = (unsigned char)v[y];
      break;
    }
    case B_RD:
      DST(0, 3) = avg3(J, K, L);
      DST(1, 3) = DST(0, 2) = avg3(I, J, K);
      DST(2, 3) = DST(1, 2) = DST(0, 1) = avg3(X, I, J);
      DST(3, 3) = DST(2, 2) = DST(1, 1) = DST(0, 0) = avg3(A, X, I);
      DST(3, 2) = DST(2, 1) = DST(1, 0) = avg3(B, A, X);
      DST(3, 1) = DST(2, 0) = avg3(C, B, A);
      DST(3, 0) = avg3(D, C, B);
      break;
    case B_LD:
      DST(0, 0) = avg3(A, B, C);
      DST(1, 0) = DST(0, 1) = avg3(B, C, D);
      DST(2, 0) = DST(1, 1) = DST(0, 2) = avg3(C, D, E);
      DST(3, 0) = DST(2, 1) = DST(1, 2) = DST(0, 3) = avg3(D, E, F);
      DST(3, 1) = DST(2, 2) = DST(1, 3) = avg3(E, F, G);
      DST(3, 2) = DST(2, 3) = avg3(F, G, H);
      DST(3, 3) = avg3(G, H, H);
      break;
    case B_VR:
      DST(0, 0) = DST(1, 2) = avg2(X, A);
      DST(1, 0) = DST(2, 2) = avg2(A, B);
      DST(2, 0) = DST(3, 2) = avg2(B, C);
      DST(3, 0) = avg2(C, D);
      DST(0, 3) = avg3(K, J, I);
      DST(0, 2) = avg3(J, I, X);
      DST(0, 1) = DST(1, 3) = avg3(I, X, A);
      DST(1, 1) = DST(2, 3) = avg3(X, A, B);
      DST(2, 1) = DST(3, 3) = avg3(A, B, C);
      DST(3, 1) = avg3(B, C, D);
      break;
    case B_VL:
      DST(0, 0) = avg2(A, B);
      DST(1, 0) = DST(0, 2) = avg2(B, C);
      DST(2, 0) = DST(1, 2) = avg2(C, D);
      DST(3, 0) = DST(2, 2) = avg2(D, E);
      DST(0, 1) = avg3(A, B, C);
      DST(1, 1) = DST(0, 3) = avg3(B, C, D);
      DST(2, 1) = DST(1, 3) = avg3(C, D, E);
      DST(3, 1) = DST(2, 3) = avg3(D, E, F);
      DST(3, 2) = avg3(E, F, G);
      DST(3, 3) = avg3(F, G, H);
      break;
    case B_HU:
      DST(0, 0) = avg2(I, J);
      DST(2, 0) = DST(0, 1) = avg2(J, K);
      DST(2, 1) = DST(0, 2) = avg2(K, L);
      DST(1, 0) = avg3(I, J, K);
      DST(3, 0) = DST(1, 1) = avg3(J, K, L);
      DST(3, 1) = DST(1, 2) = avg3(K, L, L);
      DST(3, 2) = DST(2, 2) = DST(0, 3) = DST(1, 3) = DST(2, 3) = DST(3, 3) = (unsigned char)L;
      break;
    default:  // B_HD
      DST(0, 0) = DST(2, 1) = avg2(I, X);
      DST(0, 1) = DST(2, 2) = avg2(J, I);
      DST(0, 2) = DST(2, 3) = avg2(K, J);
      DST(0, 3) = avg2(L, K);
      DST(3, 0) = avg3(A, B, C);
      DST(2, 0) = avg3(X, A, B);
      DST(1, 0) = DST(3, 1) = avg3(I, X, A);
      DST(1, 1) = DST(3, 2) = avg3(J, I, X);
      DST(1, 2) = DST(3, 3) = avg3(K, J, I);
      DST(1, 3) = avg3(L, K, J);
      break;
  }
#undef DST
}

// the macroblocks of wavefront t (x + 2y = t): y in [ylo, yhi]
__device__ __forceinline__ void wavefront(const Layout &L, int t, int &ylo, int &yhi) {
  ylo = t - (L.mbw - 1) > 0 ? (t - (L.mbw - 1) + 1) >> 1 : 0;
  yhi = min(L.mbh - 1, t >> 1);
}

// one macroblock's prediction and residual in a private buffer whose row -1 and column -1 hold its neighbours as
// libwebp's ReconstructRow sees them (127 above the frame, 129 left of it, 129 above-left of rows below the first),
// then stored into the planes
__device__ void recon_mb(unsigned char *img, const Layout &L, int mb_x, int mb_y) {
  unsigned char yb[17 * kBps], ub[9 * kBps], vb[9 * kBps];
  unsigned char *yd = yb + kBps + 8, *ud = ub + kBps + 8, *vd = vb + kBps + 8;
  unsigned char *Y = img + L.y, *U = img + L.u, *V = img + L.v;
  const int64_t mb = (int64_t)mb_y * L.mbw + mb_x;
  const MbInfo &m = reinterpret_cast<const MbInfo *>(img + L.info)[mb];
  const int16_t *coef = reinterpret_cast<const int16_t *>(img + L.coef) + mb * 384;
  const int x0 = mb_x * 16, y0 = mb_y * 16, cx0 = mb_x * 8, cy0 = mb_y * 8;
  // left column (and, below the first row, the above-left corner)
  for (int j = 0; j < 16; ++j) yd[j * kBps - 1] = mb_x > 0 ? Y[(int64_t)(y0 + j) * L.ys + x0 - 1] : 129;
  for (int j = 0; j < 8; ++j) {
    ud[j * kBps - 1] = mb_x > 0 ? U[(int64_t)(cy0 + j) * L.uvs + cx0 - 1] : 129;
    vd[j * kBps - 1] = mb_x > 0 ? V[(int64_t)(cy0 + j) * L.uvs + cx0 - 1] : 129;
  }
  if (mb_y > 0) {
    const unsigned char *ya = Y + (int64_t)(y0 - 1) * L.ys + x0;
    for (int i = -1; i < 16; ++i) yd[i - kBps] = i < 0 && mb_x == 0 ? 129 : ya[i];
    for (int i = 16; i < 20; ++i) yd[i - kBps] = mb_x < L.mbw - 1 ? ya[i] : ya[15];
    const unsigned char *ua = U + (int64_t)(cy0 - 1) * L.uvs + cx0, *va = V + (int64_t)(cy0 - 1) * L.uvs + cx0;
    for (int i = -1; i < 8; ++i) {
      ud[i - kBps] = i < 0 && mb_x == 0 ? 129 : ua[i];
      vd[i - kBps] = i < 0 && mb_x == 0 ? 129 : va[i];
    }
  } else {
    for (int i = -1; i < 20; ++i) yd[i - kBps] = 127;
    for (int i = -1; i < 8; ++i) ud[i - kBps] = vd[i - kBps] = 127;
  }
  if (m.is_i4x4) {
    // the 4x4 blocks of the right column below the first row take the above-right pixels of the macroblock
    for (int k = 1; k < 4; ++k)
      for (int i = 16; i < 20; ++i) yd[(4 * k - 1) * kBps + i] = yd[i - kBps];
    for (int n = 0; n < 16; ++n) {
      unsigned char *d = yd + (n & 3) * 4 + (n >> 2) * 4 * kBps;
      predict4(d, m.imodes[n]);
      idct_add(coef + 16 * n, d);
    }
  } else {
    predict_block(yd, 16, m.imodes[0], mb_x, mb_y);
    for (int n = 0; n < 16; ++n) idct_add(coef + 16 * n, yd + (n & 3) * 4 + (n >> 2) * 4 * kBps);
  }
  predict_block(ud, 8, m.uvmode, mb_x, mb_y);
  predict_block(vd, 8, m.uvmode, mb_x, mb_y);
  for (int n = 0; n < 4; ++n) {
    idct_add(coef + 256 + 16 * n, ud + (n & 1) * 4 + (n >> 1) * 4 * kBps);
    idct_add(coef + 320 + 16 * n, vd + (n & 1) * 4 + (n >> 1) * 4 * kBps);
  }
  for (int j = 0; j < 16; ++j)
    for (int i = 0; i < 16; ++i) Y[(int64_t)(y0 + j) * L.ys + x0 + i] = yd[j * kBps + i];
  for (int j = 0; j < 8; ++j)
    for (int i = 0; i < 8; ++i) {
      U[(int64_t)(cy0 + j) * L.uvs + cx0 + i] = ud[j * kBps + i];
      V[(int64_t)(cy0 + j) * L.uvs + cx0 + i] = vd[j * kBps + i];
    }
}

// grid B CTAs x 128 threads: CTA b reconstructs image b wavefront by wavefront
__global__ void __launch_bounds__(128) webp_recon_kernel(const cpb200_webp_image *__restrict__ table,
                                                         unsigned char *__restrict__ ws,
                                                         const int *__restrict__ status) {
  if (status[blockIdx.x]) return;
  const cpb200_webp_image &e = table[blockIdx.x];
  const Layout L = layout(e.w, e.h);
  unsigned char *img = ws + e.ws_offset;
  const int steps = L.mbw + 2 * (L.mbh - 1);
  for (int t = 0; t < steps; ++t) {
    int ylo, yhi;
    wavefront(L, t, ylo, yhi);
    for (int y = ylo + (int)threadIdx.x; y <= yhi; y += blockDim.x) recon_mb(img, L, t - 2 * y, y);
    __syncthreads();
  }
}

// libwebp's loop filters (dsp/dec.c); p points at the first pixel past the edge, `step` crosses the edge
__device__ __forceinline__ int sclip1(int v) { return v < -128 ? -128 : v > 127 ? 127 : v; }   // [-1020, 1020]
__device__ __forceinline__ int sclip2(int v) { return v < -16 ? -16 : v > 15 ? 15 : v; }       // [-112, 112]

__device__ __forceinline__ void do_filter2(unsigned char *p, int step) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  const int a = 3 * (q0 - p0) + sclip1(p1 - q1);
  const int a1 = sclip2((a + 4) >> 3), a2 = sclip2((a + 3) >> 3);
  p[-step] = clip8(p0 + a2);
  p[0] = clip8(q0 - a1);
}

__device__ __forceinline__ void do_filter4(unsigned char *p, int step) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  const int a = 3 * (q0 - p0);
  const int a1 = sclip2((a + 4) >> 3), a2 = sclip2((a + 3) >> 3), a3 = (a1 + 1) >> 1;
  p[-2 * step] = clip8(p1 + a3);
  p[-step] = clip8(p0 + a2);
  p[0] = clip8(q0 - a1);
  p[step] = clip8(q1 - a3);
}

__device__ __forceinline__ void do_filter6(unsigned char *p, int step) {
  const int p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step], q2 = p[2 * step];
  const int a = sclip1(3 * (q0 - p0) + sclip1(p1 - q1));
  const int a1 = (27 * a + 63) >> 7, a2 = (18 * a + 63) >> 7, a3 = (9 * a + 63) >> 7;
  p[-3 * step] = clip8(p2 + a3);
  p[-2 * step] = clip8(p1 + a2);
  p[-step] = clip8(p0 + a1);
  p[0] = clip8(q0 - a1);
  p[step] = clip8(q1 - a2);
  p[2 * step] = clip8(q2 - a3);
}

__device__ __forceinline__ bool needs_filter(const unsigned char *p, int step, int t) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  return 4 * abs(p0 - q0) + abs(p1 - q1) <= t;
}

__device__ __forceinline__ bool needs_filter2(const unsigned char *p, int step, int t, int it) {
  const int p3 = p[-4 * step], p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step];
  const int q0 = p[0], q1 = p[step], q2 = p[2 * step], q3 = p[3 * step];
  if (4 * abs(p0 - q0) + abs(p1 - q1) > t) return false;
  return abs(p3 - p2) <= it && abs(p2 - p1) <= it && abs(p1 - p0) <= it && abs(q3 - q2) <= it &&
         abs(q2 - q1) <= it && abs(q1 - q0) <= it;
}

__device__ __forceinline__ bool hev(const unsigned char *p, int step, int thresh) {
  return abs(p[-2 * step] - p[-step]) > thresh || abs(p[step] - p[0]) > thresh;
}

// `size` pixels along an edge: hstride crosses it, vstride walks it; `edge` picks the 6-tap macroblock-edge filter
__device__ void filter_loop(unsigned char *p, int hstride, int vstride, int size, int thresh, int ithresh,
                            int hev_t, bool edge) {
  const int t2 = 2 * thresh + 1;
  for (int i = 0; i < size; ++i, p += vstride) {
    if (!needs_filter2(p, hstride, t2, ithresh)) continue;
    if (hev(p, hstride, hev_t)) do_filter2(p, hstride);
    else if (edge) do_filter6(p, hstride);
    else do_filter4(p, hstride);
  }
}

__device__ void simple_loop(unsigned char *p, int hstride, int vstride, int thresh) {
  const int t2 = 2 * thresh + 1;
  for (int i = 0; i < 16; ++i, p += vstride)
    if (needs_filter(p, hstride, t2)) do_filter2(p, hstride);
}

// libwebp's DoFilter for one macroblock: left edge, inner vertical edges, top edge, inner horizontal edges
__device__ void filter_mb(unsigned char *img, const Layout &L, int type, int mb_x, int mb_y) {
  const MbInfo &m = reinterpret_cast<const MbInfo *>(img + L.info)[(int64_t)mb_y * L.mbw + mb_x];
  const int limit = m.limit, ilevel = m.ilevel, hv = m.hev;
  if (limit == 0) return;
  const int ys = L.ys, uvs = L.uvs;
  unsigned char *y = img + L.y + (int64_t)mb_y * 16 * ys + mb_x * 16;
  if (type == 1) {
    if (mb_x > 0) simple_loop(y, 1, ys, limit + 4);
    if (m.inner)
      for (int k = 4; k < 16; k += 4) simple_loop(y + k, 1, ys, limit);
    if (mb_y > 0) simple_loop(y, ys, 1, limit + 4);
    if (m.inner)
      for (int k = 4; k < 16; k += 4) simple_loop(y + k * ys, ys, 1, limit);
    return;
  }
  unsigned char *u = img + L.u + (int64_t)mb_y * 8 * uvs + mb_x * 8;
  unsigned char *v = img + L.v + (int64_t)mb_y * 8 * uvs + mb_x * 8;
  if (mb_x > 0) {
    filter_loop(y, 1, ys, 16, limit + 4, ilevel, hv, true);
    filter_loop(u, 1, uvs, 8, limit + 4, ilevel, hv, true);
    filter_loop(v, 1, uvs, 8, limit + 4, ilevel, hv, true);
  }
  if (m.inner) {
    for (int k = 4; k < 16; k += 4) filter_loop(y + k, 1, ys, 16, limit, ilevel, hv, false);
    filter_loop(u + 4, 1, uvs, 8, limit, ilevel, hv, false);
    filter_loop(v + 4, 1, uvs, 8, limit, ilevel, hv, false);
  }
  if (mb_y > 0) {
    filter_loop(y, ys, 1, 16, limit + 4, ilevel, hv, true);
    filter_loop(u, uvs, 1, 8, limit + 4, ilevel, hv, true);
    filter_loop(v, uvs, 1, 8, limit + 4, ilevel, hv, true);
  }
  if (m.inner) {
    for (int k = 4; k < 16; k += 4) filter_loop(y + k * ys, ys, 1, 16, limit, ilevel, hv, false);
    filter_loop(u + 4 * uvs, uvs, 1, 8, limit, ilevel, hv, false);
    filter_loop(v + 4 * uvs, uvs, 1, 8, limit, ilevel, hv, false);
  }
}

// grid B CTAs x 128 threads: CTA b loop-filters image b wavefront by wavefront
__global__ void __launch_bounds__(128) webp_filter_kernel(const cpb200_webp_image *__restrict__ table,
                                                          unsigned char *__restrict__ ws,
                                                          const int *__restrict__ status) {
  if (status[blockIdx.x]) return;
  const cpb200_webp_image &e = table[blockIdx.x];
  const Layout L = layout(e.w, e.h);
  unsigned char *img = ws + e.ws_offset;
  const int type = *reinterpret_cast<const int *>(img);
  if (type == 0) return;
  const int steps = L.mbw + 2 * (L.mbh - 1);
  for (int t = 0; t < steps; ++t) {
    int ylo, yhi;
    wavefront(L, t, ylo, yhi);
    for (int y = ylo + (int)threadIdx.x; y <= yhi; y += blockDim.x) filter_mb(img, L, type, t - 2 * y, y);
    __syncthreads();
  }
}

// libwebp's fixed-point YUV -> RGB (yuv.h, 14-bit constants, 6 fractional bits)
__device__ __forceinline__ int mult_hi(int v, int c) { return (v * c) >> 8; }
__device__ __forceinline__ unsigned char yuv_clip(int v) { return (v & ~16383) == 0 ? v >> 6 : v < 0 ? 0 : 255; }

// libwebp's "fancy" upsampling of one chroma plane at output pixel (y, x): the 9-3-3-1 filter between the nearest
// chroma sample and its neighbours across the pixel's row and column parity; at a border without a second column it
// is (3 * near + far) / 4 along the rows
__device__ __forceinline__ int upsample(const unsigned char *c, int stride, int y, int x, int h, int w) {
  const int ny = y >> 1, nx = x >> 1;
  int fy = y == 0 ? 0 : (y & 1) ? ny + 1 : ny - 1;
  if (fy > (h - 1) >> 1) fy = ny;
  int fx = x == 0 ? 0 : (x & 1) ? nx + 1 : nx - 1;
  if (fx > (w - 1) >> 1) fx = nx;
  const int nn = c[(int64_t)ny * stride + nx], fn = c[(int64_t)fy * stride + nx];
  if (fx == nx) return (3 * nn + fn + 2) >> 2;
  const int nf = c[(int64_t)ny * stride + fx], ff = c[(int64_t)fy * stride + fx];
  return (((nn + 3 * nf + 3 * fn + ff + 8) >> 3) + nn) >> 1;
}

// grid (pixel blocks, image) x 256 threads: one thread per output pixel in row-major order of the oriented image
__global__ void __launch_bounds__(256) webp_output_kernel(const cpb200_webp_image *__restrict__ table,
                                                          const unsigned char *__restrict__ ws,
                                                          const int *__restrict__ status,
                                                          unsigned char *__restrict__ dst) {
  if (status[blockIdx.y]) return;
  const cpb200_webp_image &e = table[blockIdx.y];
  const Layout L = layout(e.w, e.h);
  const unsigned char *img = ws + e.ws_offset;
  const int h = e.h, w = e.w, o = e.orientation;
  const int ow = o >= 5 ? h : w;
  const int64_t total = (int64_t)h * w;
  unsigned char *out = dst + e.dst_offset;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(i / ow), ox = (int)(i - (int64_t)oy * ow);
    // cv2's ApplyExifOrientation: transpose for 5..8, then flips
    int sy, sx;
    switch (o) {
      case 2: sy = oy; sx = w - 1 - ox; break;
      case 3: sy = h - 1 - oy; sx = w - 1 - ox; break;
      case 4: sy = h - 1 - oy; sx = ox; break;
      case 5: sy = ox; sx = oy; break;
      case 6: sy = h - 1 - ox; sx = oy; break;
      case 7: sy = h - 1 - ox; sx = w - 1 - oy; break;
      case 8: sy = ox; sx = w - 1 - oy; break;
      default: sy = oy; sx = ox; break;
    }
    const int yy = img[L.y + (int64_t)sy * L.ys + sx];
    const int u = upsample(img + L.u, L.uvs, sy, sx, h, w), v = upsample(img + L.v, L.uvs, sy, sx, h, w);
    const int yv = mult_hi(yy, 19077);
    unsigned char *q = out + i * 3;
    q[0] = yuv_clip(yv + mult_hi(u, 33050) - 17685);
    q[1] = yuv_clip(yv - mult_hi(u, 6419) - mult_hi(v, 13320) + 8708);
    q[2] = yuv_clip(yv + mult_hi(v, 26149) - 14234);
  }
}

}  // namespace

extern "C" int cpb200_webp_decode_batch(const unsigned char *src, const cpb200_webp_image *table, int B,
                                        void *workspace, size_t workspace_bytes, unsigned char *dst, int *status,
                                        void *stream) {
  if (!src || !table || !workspace || !dst || !status || B < 1)
    return cpb::fail(CPB200_ERR_ARG, "webp_decode_batch: bad arguments");
  if (B > 65535) return cpb::fail(CPB200_ERR_ARG, "webp_decode_batch: B = %d images exceed one launch (max 65535)", B);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  webp_entropy_kernel<<<B, 32, 0, st>>>(src, table, ws, workspace_bytes, status);
  int rc = cpb::check_launch("webp_entropy_kernel");
  if (rc) return rc;
  webp_recon_kernel<<<B, 128, 0, st>>>(table, ws, status);
  rc = cpb::check_launch("webp_recon_kernel");
  if (rc) return rc;
  webp_filter_kernel<<<B, 128, 0, st>>>(table, ws, status);
  rc = cpb::check_launch("webp_filter_kernel");
  if (rc) return rc;
  const dim3 grid((unsigned)std::max(1, 132 * 8 / B), (unsigned)B);
  webp_output_kernel<<<grid, 256, 0, st>>>(table, ws, status, dst);
  return cpb::check_launch("webp_output_kernel");
}

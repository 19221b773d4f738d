"""numpy restatement of ``MultiPoseDataset.__getitem__`` for split 'train', the checker of
``centerpose_b200.train_data``.

  * :func:`inputs`: ``cv2.warpAffine`` of ``img`` or ``img[:, ::-1]``, ``/ 255.`` in float32, ``color_aug``
    (lib/utils/image.py), then ``(inp - mean32) / std32``, CHW;
  * :func:`targets`: the val split's targets (``oracle/val_ref.py``) with the flip, the joints through
    ``trans_output_rot`` and the ``rot != 0`` rules;

The rules that decide bit equality, written out instead of left to numpy's or cv2's choices:
  * every in-place step of ``color_aug`` is a float32 operation: ``image *= alpha`` multiplies by float32(alpha) (alpha
    is a Python float), ``blend_`` rounds ``image * alpha``, ``image2 * (1 - alpha)`` and their sum each on its own;
  * lighting adds a float64 vector: per channel ``float32(double(x) + v[c])``;
  * ``cv2.cvtColor(float32, BGR2GRAY)`` is ``fmaf(R, 0.299f, fmaf(B, 0.114f, G * 0.587f))`` (cv2's SIMD loop), computed
    here with an exact product and a corrected float64 sum, so no result depends on the machine's cv2 dispatch;
  * ``gs.mean()`` is numpy's pairwise float32 sum (:func:`pairwise_sum`) divided by float32(n).
"""
from __future__ import annotations

import math

import cv2
import numpy as np

from oracle import val_ref

J = 17
FLIP_IDX = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]


def fmaf(a, b, c):
    """float32 fma(a, b, c) of float32 arrays, correctly rounded: the product is exact in float64, the sum is split
    into its float64 rounding s and error e (TwoSum), and the one case where rounding s to float32 differs from rounding
    s + e (s on a float32 midpoint, e pushing away from the chosen side) is corrected."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    cd = c.astype(np.float64)
    s = p + cd
    bb = s - p
    e = (p - (s - bb)) + (cd - bb)
    f = s.astype(np.float32)
    d = s - f.astype(np.float64)
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64) - f.astype(np.float64)
    dn = f.astype(np.float64) - np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    tie = ((d > 0) & (2 * d == up)) | ((d < 0) & (-2 * d == dn))
    fix = tie & (e != 0) & (np.sign(e) == np.sign(d))
    return np.where(fix, np.nextafter(f, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf))), f)


def grey(img):
    """cv2.cvtColor(img, COLOR_BGR2GRAY) of an (H, W, 3) float32 BGR image."""
    b, g, r = img[..., 0], img[..., 1], img[..., 2]
    return fmaf(r, np.float32(0.299), fmaf(b, np.float32(0.114), g * np.float32(0.587)))


def pairwise_sum(a):
    """numpy's float32 ``pairwise_sum`` (loops_utils.h) of the contiguous float32 vector ``a``."""
    n = len(a)
    if n < 8:
        res = np.float32(0)
        for v in a:
            res = np.float32(res + v)
        return res
    if n <= 128:
        r = a[0:8].copy()
        m = n - n % 8
        for i in range(8, m, 8):
            r = r + a[i:i + 8]
        res = np.float32((r[0] + r[1]) + (r[2] + r[3])) + np.float32((r[4] + r[5]) + (r[6] + r[7]))
        for v in a[m:]:
            res = np.float32(res + v)
        return np.float32(res)
    n2 = n // 2
    n2 -= n2 % 8
    return np.float32(pairwise_sum(a[:n2]) + pairwise_sum(a[n2:]))


def mean(gs):
    """``gs.mean()`` of a contiguous float32 array."""
    a = np.ascontiguousarray(gs, np.float32).reshape(-1)
    return np.float32(pairwise_sum(a) / np.float32(a.size))


def color_aug(inp, order, alphas, light):
    """``color_aug`` on the float32 (H, W, 3) ``inp`` (not modified) with the draws it would make: ``order`` the
    shuffled function indices (0 brightness, 1 contrast, 2 saturation), ``alphas`` the three Python-float
    ``1 + uniform`` in that order, ``light`` the float64 vector ``np.dot(eig_vec, eig_val * alpha)``."""
    x = inp.copy()
    gs = grey(x)
    gs_mean = mean(gs)
    for op, alpha in zip(order, alphas):
        af, bf = np.float32(alpha), np.float32(1 - alpha)
        x = x * af
        if op == 1:
            x = x + np.float32(gs_mean * bf)
        elif op == 2:
            x = x + (gs * bf)[:, :, None]
    return (x.astype(np.float64) + np.asarray(light, np.float64)).astype(np.float32)


def inputs(image, p, res, mean_, std):
    """The network input of a BGR uint8 image under the draws ``p`` (``TrainData.draw``'s keys and
    ``trans_input``): (3, res, res) float32."""
    img = image[:, ::-1] if p["flip"] else image
    inp = cv2.warpAffine(np.ascontiguousarray(img), np.asarray(p["trans_input"], np.float64), (res, res),
                         flags=cv2.INTER_LINEAR)
    inp = inp.astype(np.float32) / np.float32(255.)
    if p["color"]:
        inp = color_aug(inp, p["order"], p["alpha"], p["light"])
    inp = (inp - np.asarray(mean_, np.float32)) / np.asarray(std, np.float32)
    return inp.transpose(2, 0, 1)


def targets(gts, width, flip, rot, trans_output, trans_output_rot, R):
    """One image's targets from its ground-truth rows (``coco_eval.GT`` records, file order), the image width, the
    flip, the rotation (only ``rot != 0`` matters) and the two float64 2x3 matrices."""
    out = val_ref.empty(R)
    t = np.asarray(trans_output, np.float64).reshape(2, 3)
    tr = np.asarray(trans_output_rot, np.float64).reshape(2, 3)
    kept = [g for g in gts if int(g["iscrowd"]) != 1][:val_ref.MAX_OBJS]
    for k, g in enumerate(kept):
        bx, by, bw, bh = [float(v) for v in g["bbox"]]
        box = np.array([bx, by, bx + bw, by + bh], np.float32)
        pts = np.zeros((J, 3), np.float32)
        pts[:, 0], pts[:, 1] = np.float32(g["x"]), np.float32(g["y"])
        pts[:, 2] = [(int(g["visible"]) >> j) & 1 for j in range(J)]
        if flip:
            box[[0, 2]] = width - box[[2, 0]] - 1
            pts[:, 0] = width - pts[:, 0] - 1
            for a, b in FLIP_IDX:
                pts[a], pts[b] = pts[b].copy(), pts[a].copy()
        box[0:2] = val_ref.affine(t, box[0], box[1])
        box[2:4] = val_ref.affine(t, box[2], box[3])
        box = np.clip(box, np.float32(0), np.float32(R - 1))
        h, w = box[3] - box[1], box[2] - box[0]
        if not ((h > 0 and w > 0) or rot != 0):
            continue
        r = val_ref.radius(math.ceil(h), math.ceil(w))
        ct = np.array([(box[0] + box[2]) / np.float32(2), (box[1] + box[3]) / np.float32(2)], np.float32)
        ci = ct.astype(np.int32)
        out["wh"][k] = w, h
        out["ind"][k] = ci[1] * R + ci[0]
        out["reg"][k] = ct - ci.astype(np.float32)
        out["reg_mask"][k] = 1
        if pts[:, 2].sum() == 0:
            out["hm"][0, ci[1], ci[0]] = np.float32(0.9999)
            out["reg_mask"][k] = 0
        for j in range(J):
            if not pts[j, 2] > 0:
                continue
            px, py = val_ref.affine(tr, pts[j, 0], pts[j, 1])
            if not (px >= 0 and px < R and py >= 0 and py < R):
                continue
            pt = np.array([px, py], np.float32)
            pi = pt.astype(np.int32)
            out["hps"][k, 2 * j:2 * j + 2] = pt - ci.astype(np.float32)
            out["hps_mask"][k, 2 * j:2 * j + 2] = 1
            out["hp_offset"][k * J + j] = pt - pi.astype(np.float32)
            out["hp_ind"][k * J + j] = pi[1] * R + pi[0]
            out["hp_mask"][k * J + j] = 1
            val_ref.draw(out["hm_hp"][j], int(pi[0]), int(pi[1]), r)
        val_ref.draw(out["hm"][0], int(ci[0]), int(ci[1]), r)
    if rot != 0:
        out["hm"][:] = np.float32(0.9999)
        out["reg_mask"][:] = 0
        out["hps_mask"][:] = 0
    return out

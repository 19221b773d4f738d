"""numpy restatement of the reference's validation pass per image, the checker of ``centerpose_b200.val``.

  * :func:`targets`: ``MultiPoseDataset.__getitem__``'s targets for the val split (``lib/datasets/multi_pose.py``: rot 0,
    no flip, ``draw_umich_gaussian``), from the ground-truth rows ``coco_eval.gt_table`` makes and ``trans_output``;
  * :func:`inputs`: its network input, ``cv2.warpAffine`` then ``(inp.astype(float32) / 255. - mean32) / std32``;
  * :func:`loss`: ``MultiPoseLoss.forward`` (``lib/trains/multi_pose.py``) with float64 sums, each stat rounded to
    float32 once.

The rules that decide bit equality, written out instead of left to numpy's choices:
  * ``affine_transform`` is ``np.dot(t, float32([x, y, 1]))``; with a BLAS that is ``fma(t0, x, t1 * y) + t2`` in
    float64.  The FMA is computed here with exact rationals, so no result depends on the machine's BLAS kernel.
  * ``gaussian_radius`` is evaluated left to right in Python floats, as the reference writes it.
  * the Gaussian stamp is ``float32(exp(-(x*x + y*y) / (2*sigma*sigma)))``, sigma = (2r + 1) / 6, and
    ``np.maximum(float32, float64)`` cast back to float32 is ``max(h, float32(g))``.
  * the one plain store, ``hm[ct] = 0.9999`` for an object without keypoints, comes right before that object's own
    stamp, whose centre is 1.0; so drawing every stamp as a maximum in any order gives the same maps.
"""
from __future__ import annotations

import math
from fractions import Fraction

import cv2
import numpy as np

J = 17
MAX_OBJS = 32
STATS = ["loss", "hm_loss", "hp_loss", "hm_hp_loss", "hp_offset_loss", "wh_loss", "off_loss"]


def affine(t, x, y):
    """``affine_transform([x, y], t)`` as float32: fma(t[0], x, t[1] * y) + t[2] per output row."""
    out = []
    for r in (0, 1):
        p = float(t[r][1]) * float(np.float32(y))
        s = float(Fraction(float(t[r][0])) * Fraction(float(np.float32(x))) + Fraction(p))
        out.append(np.float32(s + float(t[r][2])))
    return out


def gaussian_radius(height, width, min_overlap=0.7):
    a1 = 1
    b1 = (height + width)
    c1 = width * height * (1 - min_overlap) / (1 + min_overlap)
    r1 = (b1 + math.sqrt(b1 ** 2 - 4 * a1 * c1)) / 2
    a2 = 4
    b2 = 2 * (height + width)
    c2 = (1 - min_overlap) * width * height
    r2 = (b2 + math.sqrt(b2 ** 2 - 4 * a2 * c2)) / 2
    a3 = 4 * min_overlap
    b3 = -2 * min_overlap * (height + width)
    c3 = (min_overlap - 1) * width * height
    r3 = (b3 + math.sqrt(b3 ** 2 - 4 * a3 * c3)) / 2
    return min(r1, r2, r3)


def radius(height, width):
    return max(0, int(gaussian_radius(height, width)))


def stamp(r):
    """The (2r+1, 2r+1) float32 Gaussian ``draw_umich_gaussian`` draws at radius r."""
    sigma = (2 * r + 1) / 6
    y, x = np.ogrid[-r:r + 1, -r:r + 1]
    return np.exp(-(x * x + y * y).astype(np.float64) / (2 * sigma * sigma)).astype(np.float32)


def draw(heatmap, cx, cy, r):
    R = heatmap.shape[0]
    g = stamp(r)
    left, right = min(cx, r), min(R - cx, r + 1)
    top, bottom = min(cy, r), min(R - cy, r + 1)
    win = heatmap[cy - top:cy + bottom, cx - left:cx + right]
    np.maximum(win, g[r - top:r + bottom, r - left:r + right], out=win)


def empty(R):
    """The target arrays of one image, zero, under the reference's batch keys."""
    M = MAX_OBJS
    return {"hm": np.zeros((1, R, R), np.float32), "hm_hp": np.zeros((J, R, R), np.float32),
            "wh": np.zeros((M, 2), np.float32), "reg": np.zeros((M, 2), np.float32), "ind": np.zeros(M, np.int64),
            "reg_mask": np.zeros(M, np.uint8), "hps": np.zeros((M, 2 * J), np.float32),
            "hps_mask": np.zeros((M, 2 * J), np.uint8), "hp_offset": np.zeros((M * J, 2), np.float32),
            "hp_ind": np.zeros(M * J, np.int64), "hp_mask": np.zeros(M * J, np.int64)}


def targets(gts, trans_output, R):
    """One image's targets from its ground-truth rows (``coco_eval.GT`` records, in file order) and its float64 2x3
    ``trans_output``."""
    out = empty(R)
    t = np.asarray(trans_output, np.float64).reshape(2, 3)
    kept = [g for g in gts if int(g["iscrowd"]) != 1][:MAX_OBJS]
    for k, g in enumerate(kept):
        bx, by, bw, bh = [float(v) for v in g["bbox"]]
        box = np.array([bx, by, bx + bw, by + bh], np.float32)
        box[0:2] = affine(t, box[0], box[1])
        box[2:4] = affine(t, box[2], box[3])
        box = np.clip(box, np.float32(0), np.float32(R - 1))
        h, w = box[3] - box[1], box[2] - box[0]
        if not (h > 0 and w > 0):
            continue
        r = radius(math.ceil(h), math.ceil(w))
        ct = np.array([(box[0] + box[2]) / np.float32(2), (box[1] + box[3]) / np.float32(2)], np.float32)
        ci = ct.astype(np.int32)
        out["wh"][k] = w, h
        out["ind"][k] = ci[1] * R + ci[0]
        out["reg"][k] = ct - ci.astype(np.float32)
        out["reg_mask"][k] = 1
        if int(g["visible"]) == 0:
            out["hm"][0, ci[1], ci[0]] = np.float32(0.9999)
            out["reg_mask"][k] = 0
        for j in range(J):
            if not (int(g["visible"]) >> j) & 1:
                continue
            px, py = affine(t, g["x"][j], g["y"][j])
            if not (px >= 0 and px < R and py >= 0 and py < R):
                continue
            pt = np.array([px, py], np.float32)
            pi = pt.astype(np.int32)
            out["hps"][k, 2 * j:2 * j + 2] = pt - ci.astype(np.float32)
            out["hps_mask"][k, 2 * j:2 * j + 2] = 1
            out["hp_offset"][k * J + j] = pt - pi.astype(np.float32)
            out["hp_ind"][k * J + j] = pi[1] * R + pi[0]
            out["hp_mask"][k * J + j] = 1
            draw(out["hm_hp"][j], int(pi[0]), int(pi[1]), r)
        draw(out["hm"][0], int(ci[0]), int(ci[1]), r)
    return out


def inputs(image, trans_input, res, mean, std):
    """The dataset's network input of a BGR uint8 image: (3, res, res) float32."""
    inp = cv2.warpAffine(image, np.asarray(trans_input, np.float64), (res, res), flags=cv2.INTER_LINEAR)
    inp = inp.astype(np.float32) / np.float32(255.)
    inp = (inp - np.asarray(mean, np.float32)) / np.asarray(std, np.float32)
    return inp.transpose(2, 0, 1)


def _focal(logits, gt):
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        x = np.asarray(logits, np.float32)
        p = np.float32(1) / (np.float32(1) + np.exp(-x))
        p = np.where(np.isnan(p), p, np.clip(p, np.float32(1e-4), np.float32(1 - 1e-4)))
        pos = (gt == 1).astype(np.float32)
        neg = (gt < 1).astype(np.float32)
        q, w = np.float32(1) - p, np.float32(1) - gt
        w2 = w * w
        pos_loss = (np.log(p) * (q * q) * pos).astype(np.float64).sum()
        neg_loss = (np.log(q) * (p * p) * (w2 * w2) * neg).astype(np.float64).sum()
    npos = float(pos.sum(dtype=np.float64))
    return np.float32(-neg_loss if npos == 0 else -(pos_loss + neg_loss) / npos)


def _l1(pred_map, ind, mask, target):
    """sum |pred * m - t * m| / (sum(m) + 1e-4) with pred gathered from (C, R, R) at ind; mask already expanded."""
    C = pred_map.shape[0]
    pred = pred_map.reshape(C, -1)[:, ind].T                  # (n, C)
    m = mask.astype(np.float32)
    with np.errstate(invalid="ignore"):
        s = np.abs(pred * m - target * m).astype(np.float64).sum()
    den = np.float32(np.float32(m.sum(dtype=np.float64)) + np.float32(1e-4))
    return np.float32(s / np.float64(den))


def loss(heads, tg, loss_cfg):
    """MultiPoseLoss.forward for one image: ``heads`` the six (C, R, R) float32 maps (logits for hm and hm_hp),
    ``tg`` its targets (:func:`targets`), ``loss_cfg`` the cfg's LOSS section.  Returns the seven float32 stats in
    :data:`STATS` order."""
    hm, wh, hps, reg, hm_hp, hp_offset = [np.asarray(h, np.float32) for h in heads]
    c = loss_cfg
    hm_loss = _focal(hm, tg["hm"])
    hp_loss = _l1(hps, tg["ind"], tg["hps_mask"], tg["hps"])
    z = np.float32(0)
    two = lambda m: np.repeat(np.asarray(m)[:, None], 2, axis=1)
    wh_loss = _l1(wh, tg["ind"], two(tg["reg_mask"]), tg["wh"]) if c["WH_WEIGHT"] > 0 else z
    off_loss = _l1(reg, tg["ind"], two(tg["reg_mask"]), tg["reg"]) if c["REG_OFFSET"] and c["OFF_WEIGHT"] > 0 else z
    hp_offset_loss = _l1(hp_offset, tg["hp_ind"], two(tg["hp_mask"]), tg["hp_offset"]) \
        if c["REG_HP_OFFSET"] and c["OFF_WEIGHT"] > 0 else z
    hm_hp_loss = _focal(hm_hp, tg["hm_hp"]) if c["HM_HP"] and c["HM_HP_WEIGHT"] > 0 else z
    f = np.float32
    total = f(c["HM_WEIGHT"]) * hm_loss
    for wgt, v in ((c["WH_WEIGHT"], wh_loss), (c["OFF_WEIGHT"], off_loss), (c["HP_WEIGHT"], hp_loss),
                   (c["HM_HP_WEIGHT"], hm_hp_loss), (c["OFF_WEIGHT"], hp_offset_loss)):
        total = f(total + f(wgt) * v)
    return np.array([total, hm_loss, hp_loss, hm_hp_loss, hp_offset_loss, wh_loss, off_loss], np.float32)

"""Seeded COCO keypoint ground truths and detection rows for the evaluation tests.

``make_case(seed)`` returns ``(gt, results)``: a single-category ``person_keypoints``-style dict and
``{image_id: {1: (N, 56) float32 rows}}``.  Every case reaches: crowd ground truths, ``num_keypoints == 0``, partly
visible ones, ones with no visible joint but ``num_keypoints > 0`` (computeOks' box branch), areas exactly 32^2 and
96^2, images with no ground truth (with and without detections), ground truths without detections, up to ``max_rows``
rows per image (the cut to 20), two-decimal score ties (and -0.0 against 0.0, and a NaN score), detections equal to a
ground truth (OKS exactly 1), a ground truth with id 0, float32 values at '{:.2f}' midpoints, and a NaN keypoint.

``check_margins`` asserts that no OKS lies within 1e-9 of a threshold (exact 1.0 and NaN apart) and that no two
different OKS >= 0.5 of one detection lie within 1e-9 of each other, so a 1-ulp difference of exp() cannot change a match.
"""
from __future__ import annotations

import numpy as np

THRESHOLDS = np.linspace(.5, 0.95, 10)
MIDPOINTS = np.array([0.125, 0.375, 0.625, 0.875, 0.005, 0.015, 0.245, 0.995], np.float64)


def _gt(rng, image_id, ann_id, kind, area):
    w = float(np.sqrt(area * rng.uniform(0.5, 2.0)))
    h = float(area / w)
    x, y = float(rng.integers(0, 400)), float(rng.integers(0, 300))
    kx = np.rint(x + rng.random(17) * w)
    ky = np.rint(y + rng.random(17) * h)
    if kind == "full":
        v = np.full(17, 2.0)
    elif kind == "partial":
        v = rng.choice([0.0, 1.0, 2.0], 17)
        v[rng.integers(0, 17)] = 2.0
    else:                                   # "hidden" (num_keypoints > 0) or "empty" (num_keypoints == 0)
        v = np.zeros(17)
        kx[:] = 0.0
        ky[:] = 0.0
    kp = np.stack([kx, ky, v], 1).reshape(-1)
    nk = int(np.count_nonzero(v > 0)) if kind != "hidden" else int(rng.integers(1, 6))
    return {"id": int(ann_id), "image_id": int(image_id), "category_id": 1, "iscrowd": 0,
            "keypoints": [float(a) if a != int(a) else int(a) for a in kp], "num_keypoints": nk,
            "area": float(area), "bbox": [x, y, round(w, 2), round(h, 2)]}


def _row(rng, gt, noise, score):
    r = np.zeros(56, np.float32)
    if gt is not None and noise == 0.0 and gt["num_keypoints"] > 0 and any(gt["keypoints"][2::3]):
        kx = np.asarray(gt["keypoints"][0::3], np.float64)
        ky = np.asarray(gt["keypoints"][1::3], np.float64)
    else:
        if gt is not None:
            bx, by, bw, bh = gt["bbox"]
            if any(gt["keypoints"][2::3]):
                cx = np.asarray(gt["keypoints"][0::3], np.float64)
                cy = np.asarray(gt["keypoints"][1::3], np.float64)
            else:
                cx = bx + rng.random(17) * bw
                cy = by + rng.random(17) * bh
            s = np.sqrt(max(gt["area"], 1.0))
        else:
            cx, cy, s = rng.uniform(0, 600, 17), rng.uniform(0, 400, 17), 50.0
        kx = cx + rng.normal(0, 1, 17) * s * max(noise, 1e-3)
        ky = cy + rng.normal(0, 1, 17) * s * max(noise, 1e-3)
    r[5:39:2], r[6:39:2] = kx, ky
    # a few coordinates exactly at, or at the float32 nearest to, a '{:.2f}' midpoint
    for j in rng.choice(17, 2, replace=False):
        r[5 + 2 * j] = np.float32(np.floor(kx[j]) + rng.choice(MIDPOINTS))
    x1, x2 = float(kx.min()), float(kx.max())
    y1, y2 = float(ky.min()), float(ky.max())
    pad = rng.uniform(-2, 8)
    r[0:4] = [x1 - pad, y1 - pad, x2 + pad, y2 + pad]
    r[4] = score
    r[39:56] = rng.random(17)
    return r


def _score(rng):
    c = rng.random()
    if c < 0.5:
        return np.float32(rng.integers(0, 101) / 100)       # two-decimal ties
    if c < 0.65:
        return np.float32(rng.choice(MIDPOINTS))
    return np.float32(rng.random())


def make_case(seed, n_images=40, max_rows=200, gts_per_image=(1, 6), rows_per_image=None):
    """``rows_per_image``: every image with detections gets exactly that many (else 1 to ``max_rows``)."""
    rng = np.random.default_rng(seed)
    ids = rng.choice(10 ** 6, n_images, replace=False)
    images = [{"id": int(i), "width": 640, "height": 480, "file_name": "%012d.jpg" % i} for i in ids]
    anns, results = [], {}
    next_id = 1
    for k, image_id in enumerate(ids):
        role = k % 5                       # 0: nothing, 1: detections only, 2: ground truths only, 3-4: both
        gts = []
        if role >= 2:
            for g in range(int(rng.integers(*gts_per_image))):
                kind = rng.choice(["full", "partial", "partial", "hidden", "empty"])
                area = float(rng.choice([32.0 ** 2, 96.0 ** 2, rng.uniform(200, 40000), rng.uniform(1000, 9000)]))
                gt = _gt(rng, image_id, next_id, kind, area)
                next_id += 1
                if rng.random() < 0.12:
                    gt["iscrowd"] = 1
                if rng.random() < 0.1:
                    gt["ignore"] = 1                  # overwritten by _prepare
                gts.append(gt)
        anns += gts
        if role in (0, 2):
            continue
        n = int(rng.integers(1, max_rows + 1)) if rng.random() < 0.5 else int(rng.integers(1, 30))
        n = rows_per_image or n
        rows = []
        for _ in range(n):
            gt = gts[int(rng.integers(0, len(gts)))] if gts and rng.random() < 0.8 else None
            noise = float(rng.choice([0.0, 0.02, 0.05, 0.1, 0.2, 0.5]))
            rows.append(_row(rng, gt, noise, _score(rng)))
        results[int(image_id)] = {1: np.stack(rows)}
    # the edge values, in the first image with ground truths and detections
    with_gt = {a["image_id"] for a in anns}
    rows = results[next(i for i in results if i in with_gt)][1]
    rows[0, 4] = np.float32(-0.001)             # rounds to -0.0, ties with 0.0
    if len(rows) > 1:
        rows[1, 4] = np.float32(0.0)
    if len(rows) > 2:
        rows[2, 4] = np.float32(np.nan)
    if len(rows) > 3:
        rows[3, 7] = np.float32(np.nan)         # a NaN OKS: `ious < iou` is False, so it is taken
        rows[3, 4] = np.float32(0.99)
    anns[len(anns) // 2]["id"] = 0             # a ground truth with id 0
    order = rng.permutation(len(images))       # images listed out of id order
    gt = {"images": [images[i] for i in order], "annotations": anns,
          "categories": [{"id": 1, "name": "person", "supercategory": "person"}]}
    return gt, results


def check_margins(ious):
    """Asserts the OKS margins above on ``COCOeval.ious`` (``{(image, cat): (D, G) array or []}``)."""
    for key, m in ious.items():
        m = np.asarray(m, np.float64)
        if m.size == 0:
            continue
        v = m[np.isfinite(m) & (m != 1.0)]
        near = np.abs(v[:, None] - THRESHOLDS[None, :]).min(1) if v.size else np.zeros(0)
        assert not np.any(near < 1e-9), "image %r: an OKS within 1e-9 of a threshold" % (key,)
        for row in m:
            f = np.sort(row[np.isfinite(row) & (row >= 0.5 - 1e-9)])      # only OKS above 0.5 are compared
            d = np.diff(f)
            assert not np.any((d > 0) & (d < 1e-9)), "image %r: two OKS within 1e-9" % (key,)

"""ORACLE (test infrastructure, not product): cv2 restatement of what the reference's ``MultiPoseDetector.show_results``
draws (``lib/detectors/multi_pose.py:96-107`` with ``lib/utils/debugger.py`` ``add_coco_bbox`` / ``add_coco_hp`` for
the one-class 'coco_hp' Debugger).  ``tests/golden/render_poses.npz`` pins it to the unmodified reference Debugger;
the device renderer (``csrc/render.cu``) is checked against it byte for byte.
"""
from __future__ import annotations

import math

import cv2
import numpy as np

from centerpose_b200.render import EDGES, theme_color


def add_coco_bbox(img, bbox, conf, theme):
    bbox = np.array(bbox, dtype=np.int32)
    c = list(theme_color(theme))
    txt = "p{:.1f}".format(conf)
    font = cv2.FONT_HERSHEY_SIMPLEX
    size = cv2.getTextSize(txt, font, 0.5, 2)[0]
    cv2.rectangle(img, (bbox[0], bbox[1]), (bbox[2], bbox[3]), c, 2)
    cv2.rectangle(img, (bbox[0], bbox[1] - size[1] - 2), (bbox[0] + size[0], bbox[1] - 2), c, -1)
    cv2.putText(img, txt, (bbox[0], bbox[1] - 2), font, 0.5, (0, 0, 0), thickness=1, lineType=cv2.LINE_AA)


def add_coco_hp(img, points, points_prob):
    """Returns the drawn image (each limb's addWeighted makes a new array)."""
    pts = np.array(points, dtype=np.int32).reshape(17, 2)
    prob = np.array(points_prob, dtype=np.float32).reshape(17)
    for j in range(17):
        if prob[j] > 0.:
            cv2.circle(img, (pts[j, 0], pts[j, 1]), 2, (255, 255, 255), -1)
    canvas = img.copy()
    for a, b in EDGES:
        if prob[a] > 0. and prob[b] > 0.:
            ys = [pts[a, 1], pts[b, 1]]
            xs = [pts[a, 0], pts[b, 0]]
            length = ((ys[0] - ys[1]) ** 2 + (xs[0] - xs[1]) ** 2) ** 0.5
            angle = math.degrees(math.atan2(ys[0] - ys[1], xs[0] - xs[1]))
            poly = cv2.ellipse2Poly((int(np.mean(xs)), int(np.mean(ys))), (int(length / 2), 2), int(angle), 0, 360, 1)
            cv2.fillConvexPoly(canvas, poly, (255, 255, 255))
            img = cv2.addWeighted(img, 0.8, canvas, 0.2, 0)
    return img


def show_results(image, results, vis_thresh=0.3, theme="white"):
    """The image ``show_results`` leaves in ``debugger.imgs['multi_pose']`` for ``results`` (rows of 56)."""
    img = image.copy()
    for det in results:
        if det[4] > vis_thresh:
            add_coco_bbox(img, det[:4], det[4], theme)
            img = add_coco_hp(img, det[5:39], det[39:56])
    return img

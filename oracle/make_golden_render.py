"""Generate ``tests/golden/render_poses.npz``: the reference's own ``Debugger`` (UNMODIFIED,
``/root/reference/lib/utils/debugger.py``, made with ``ipynb=True`` so it does not import matplotlib) drawing seeded
rows the way ``MultiPoseDetector.show_results`` does, and pin :mod:`oracle.debugger_ref` against it before anything is
written.

Run:  python -m oracle.make_golden_render      (from the repo root; needs /root/reference)

Cases (``tests/render_cases.py``): both themes; small images with random persons (every label string, joints with
score <= 0, zero-length limbs, overlapping persons, persons partly and wholly off the image, rows at and just above
VIS_THRESH 0.3) and the hand-placed ``edge_rows`` (label boxes cut by the top row, inside-out and point boxes).
Stored per case k: ``image_k``, ``rows_k``, ``theme_k``, ``out_k``.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/lib"
OUT = os.path.join(ROOT, "tests", "golden", "render_poses.npz")


def reference_show_results(image, results, theme, vis_thresh=0.3):
    """``show_results`` (multi_pose.py:96-107) with the reference's Debugger, minus the final ``show_all_imgs``."""
    sys.path.insert(0, os.path.join(REF, "utils"))
    try:
        from debugger import Debugger
    finally:
        sys.path.pop(0)
    dbg = Debugger(ipynb=True, theme=theme, num_classes=1, dataset="coco_hp", down_ratio=4)
    dbg.add_img(image, img_id="multi_pose")
    for det in results:
        if det[4] > vis_thresh:
            dbg.add_coco_bbox(det[:4], 0, det[4], img_id="multi_pose")
            dbg.add_coco_hp(det[5:39], det[39:], img_id="multi_pose")
    return dbg.imgs["multi_pose"]


def cases():
    sys.path.insert(0, ROOT)
    from tests import render_cases as rc
    out = []
    for k, (h, w, n, off) in enumerate([(48, 64, 6, 0.0), (61, 47, 12, 0.3), (40, 90, 20, 0.5), (72, 56, 3, 0.0)]):
        for theme in ("white", "black"):
            out.append((rc.image(h, w, 100 + k), rc.rows(h, w, n, 200 + k, spread=0.6, off=off), theme))
    for theme in ("white", "black"):
        out.append((rc.image(50, 70, 300), rc.edge_rows(50, 70), theme))
    return out


def main():
    from oracle import debugger_ref
    store = {}
    for k, (img, rows, theme) in enumerate(cases()):
        want = reference_show_results(img.copy(), rows.tolist(), theme)
        got = debugger_ref.show_results(img, rows.tolist(), 0.3, theme)
        if not np.array_equal(want, got):
            raise SystemExit("oracle.debugger_ref != reference Debugger on case %d" % k)
        store.update({"image_%d" % k: img, "rows_%d" % k: rows, "theme_%d" % k: np.array(theme), "out_%d" % k: want})
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(store) // 4, "cases")


if __name__ == "__main__":
    main()

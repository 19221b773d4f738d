"""Generate ``tests/golden/heatmap_views.npz``: the reference's own ``Debugger`` (UNMODIFIED,
``/root/reference/lib/utils/debugger.py``, made with ``ipynb=True`` so it does not import matplotlib) making the views
``MultiPoseDetector.debug`` makes (``gen_colormap`` / ``gen_colormap_hp`` and ``add_blend_img`` after ``debug()``'s
de-normalization line), and pin :mod:`oracle.heatmaps_ref` against it before anything is written.

Run:  python -m oracle.make_golden_heatmaps      (from the repo root; needs /root/reference)

Cases, each with both themes ('white' and 'black'): square, landscape and portrait maps, 8x40 and 40x8, a 1x1 map,
a down ratio of 2 and 3 keypoint maps; map values exactly 0 and 1, on and just below k/255 and k/128 (the products
that land on an integer), MSE-mode raw maps with negative values and values above 1; inputs from the pre-process
normalization of a uint8 image and inputs that de-normalize far outside [0, 255].
Stored per case k: ``x_k``, ``hm_k``, ``hp_k``, ``dr_k`` and ``<theme>_<view>_k``; ``mean`` and ``std`` once.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/lib"
OUT = os.path.join(ROOT, "tests", "golden", "heatmap_views.npz")
MEAN = np.array([0.408, 0.447, 0.470], np.float32)
STD = np.array([0.289, 0.274, 0.278], np.float32)
THEMES = ("white", "black")


def reference_views(x, hm, hm_hp, dr, theme):
    """``debug()``'s views (multi_pose.py:82-94, with ``output[0]`` / ``output[4]`` for ``output['hm']`` /
    ``output['hm_hp']``) from the reference's Debugger."""
    sys.path.insert(0, os.path.join(REF, "utils"))
    try:
        from debugger import Debugger
    finally:
        sys.path.pop(0)
    dbg = Debugger(ipynb=True, theme=theme, num_classes=1, dataset="coco_hp", down_ratio=dr)
    img = x.transpose(1, 2, 0)
    img = np.clip(((img * STD.reshape(1, 1, 3) + MEAN.reshape(1, 1, 3)) * 255.), 0, 255).astype(np.uint8)
    dbg.add_blend_img(img, dbg.gen_colormap(hm), "pred_hm")
    dbg.add_blend_img(img, dbg.gen_colormap_hp(hm_hp), "pred_hmhp")
    return {v: dbg.imgs[v] for v in ("pred_hm", "pred_hmhp")}


def edge_values():
    """0, 1, and k/255, k/128 as float32 with their next float below: products with the colours that land on or just
    below an integer."""
    k = np.arange(256, dtype=np.float64)
    on = np.concatenate([k / 255, k[:129] / 128]).astype(np.float32)
    return np.concatenate([[0, 1], on, np.nextafter(on, np.float32(0))]).astype(np.float32)


def maps(rng, c, h, w, raw=False):
    """(c, h, w) maps: half edge values, half uniform [0, 1]; ``raw``: MSE-mode maps, also negative and above 1."""
    m = np.where(rng.random((c, h, w)) < 0.5, rng.choice(edge_values(), (c, h, w)), rng.random((c, h, w)))
    if raw:
        m = np.where(rng.random((c, h, w)) < 0.5, m, rng.normal(0, 1.5, (c, h, w)))
        m.reshape(-1)[:6] = [-1.5 / 255, 300.7 / 255, -300 / 255, 2.0, -0.001, 1.0001]
    return m.astype(np.float32)


def normalized(rng, H, W):
    """A uint8 image through pre_process's normalization (base_detector.py:53), as (3, H, W) float32."""
    img = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    img[0, :min(W, 4)] = [[0, 0, 0], [255, 255, 255], [254, 1, 128], [255, 0, 255]][:min(W, 4)]
    return ((img / 255. - MEAN) / STD).astype(np.float32).transpose(2, 0, 1).copy()


def cases():
    """(x, hm, hm_hp, dr) per case."""
    rng = np.random.default_rng(2024)
    out = []
    for h, w, c, dr, raw, wild in [(10, 10, 17, 4, False, False), (8, 12, 17, 4, False, False),
                                   (12, 8, 17, 4, False, False), (8, 40, 17, 4, False, False),
                                   (40, 8, 17, 4, False, False), (1, 1, 17, 4, False, False),
                                   (6, 10, 17, 4, True, False), (9, 13, 3, 2, False, True),
                                   (7, 7, 17, 4, True, True)]:
        H, W = h * dr, w * dr
        x = rng.normal(0, 4, (3, H, W)).astype(np.float32) if wild else normalized(rng, H, W)
        out.append((x, maps(rng, 1, h, w), maps(rng, c, h, w, raw), dr))
    return out


def main():
    from oracle import heatmaps_ref
    store = {"mean": MEAN, "std": STD}
    for k, (x, hm, hp, dr) in enumerate(cases()):
        store.update({"x_%d" % k: x, "hm_%d" % k: hm, "hp_%d" % k: hp, "dr_%d" % k: np.array(dr)})
        for theme in THEMES:
            want = reference_views(x, hm, hp, dr, theme)
            got = heatmaps_ref.heatmap_views(x, hm, hp, dr, theme, MEAN, STD)
            for v in want:
                if not np.array_equal(want[v], got[v]):
                    raise SystemExit("oracle.heatmaps_ref != reference Debugger on case %d %s %s" % (k, theme, v))
                store["%s_%s_%d" % (theme, v, k)] = want[v]
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(cases()), "cases")


if __name__ == "__main__":
    main()

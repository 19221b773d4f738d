"""Heat-map view throughput: centerpose_b200.heatmaps.views (cpb200_heatmap_views_batch, including its one copy back)
against the reference's path (download the input and the maps, then the numpy / cv2 views of oracle/heatmaps_ref.py
on one host thread), for N 512x512 network inputs with 128x128 maps; and run_images on COCO-sized JPEG files with
and without return_heatmaps.  Three alternating rounds; outputs are compared in the same run.  Prints the card and its
power limit.

    python tools/bench_heatmaps.py [--n 256] [--rounds 3] [--run-images 64]
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from centerpose_b200 import heatmaps  # noqa: E402
from centerpose_b200.config import default_cfg  # noqa: E402
from centerpose_b200.detector import detector_factory  # noqa: E402
from oracle import heatmaps_ref  # noqa: E402
from oracle.init_recipe import conditioned_state_dict  # noqa: E402
from tests import render_cases as rc  # noqa: E402
from tools.bench_render import SHAPES, card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--run-images", type=int, default=64)
    a = ap.parse_args()
    print("card:", card())
    cfg = default_cfg("dla_34")
    theme, mean, std = cfg.DEBUG_THEME, np.array(cfg.DATASET.MEAN, np.float32), np.array(cfg.DATASET.STD, np.float32)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((a.n, 3, 512, 512), device="cuda", generator=g)
    hm = torch.rand((a.n, 1, 128, 128), device="cuda", generator=g)
    hp = torch.rand((a.n, 17, 128, 128), device="cuda", generator=g)
    inputs, hms, hps = list(x), list(hm), list(hp)
    heatmaps.views(inputs[:8], hms[:8], hps[:8], 4, theme, mean, std)          # warm-up: module load
    threads = cv2.getNumThreads()
    dev, host = [], []
    for _ in range(a.rounds):
        t, got = timed(lambda: heatmaps.views(inputs, hms, hps, 4, theme, mean, std))
        dev.append(a.n / t)
        cv2.setNumThreads(1)
        t0 = time.perf_counter()
        xs, hs, ps = x.cpu().numpy(), hm.cpu().numpy(), hp.cpu().numpy()
        want = [heatmaps_ref.heatmap_views(xs[i], hs[i], ps[i], 4, theme, mean, std) for i in range(a.n)]
        host.append(a.n / (time.perf_counter() - t0))
        cv2.setNumThreads(threads)
        assert all(np.array_equal(gv[v], wv[v]) for gv, wv in zip(got, want) for v in heatmaps.VIEWS), "views != oracle"
    print("heatmap views, N=%d at 512x512: device %s images/s; download + numpy/cv2 on 1 thread %s images/s (identical)"
          % (a.n, "/".join("%.0f" % v for v in dev), "/".join("%.1f" % v for v in host)))

    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for k in range(a.run_images):
            p = os.path.join(tmp, "im%d.jpg" % k)
            cv2.imwrite(p, rc.image(*SHAPES[k % 3], 1000 + k), [cv2.IMWRITE_JPEG_QUALITY, 90])
            paths.append(p)
        det.run_images(paths[:8])
        det.run_images(paths[:8], return_heatmaps=True)
        plain, views = [], []
        for _ in range(a.rounds):
            t, rows = timed(lambda: det.run_images(paths))
            plain.append(len(paths) / t)
            t, (rows2, _) = timed(lambda: det.run_images(paths, return_heatmaps=True))
            views.append(len(paths) / t)
            assert all(np.array_equal(r, s) for r, s in zip(rows, rows2)), "return_heatmaps changed the rows"
    print("run_images %d JPEG files (FLIP_TEST %s, FIX_RES %s): %s images/s, with return_heatmaps %s images/s "
          "(rows identical)" % (len(paths), det.cfg.TEST.FLIP_TEST, det.cfg.TEST.FIX_RES,
                                "/".join("%.0f" % v for v in plain), "/".join("%.0f" % v for v in views)))


if __name__ == "__main__":
    main()

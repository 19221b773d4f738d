"""Pose drawing throughput: MultiPoseDetector.render_poses (cpb200_render_poses_batch) against the cv2 oracle of the
reference's show_results (oracle/debugger_ref.py) on one host thread and on cv2's default threads, and run_images
with and without return_images.  Seeded COCO-sized images (640x480 / 480x640 / 640x427) with 1, 5 and 10 drawn
persons each; three alternating rounds; outputs are compared in the same run.  Prints the card and its power limit.

    python tools/bench_render.py [--n 256] [--rounds 3]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from centerpose_b200.config import default_cfg  # noqa: E402
from centerpose_b200.detector import detector_factory  # noqa: E402
from oracle import debugger_ref  # noqa: E402
from oracle.init_recipe import conditioned_state_dict  # noqa: E402
from tests import render_cases as rc  # noqa: E402
from tools.bench_images import TEST_SECTIONS  # noqa: E402

SHAPES = [(480, 640), (640, 480), (427, 640)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def workload(n, persons):
    images = [rc.image(*SHAPES[k % 3], 1000 + k) for k in range(n)]
    results = []
    for k, im in enumerate(images):
        r = rc.rows(im.shape[0], im.shape[1], persons, 2000 + k, spread=0.4)
        r[:, 4] = 0.31 + 0.68 * np.random.default_rng(k).random(persons)
        results.append(r)
    return images, results


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--run-images", type=int, default=64)
    a = ap.parse_args()
    print("card:", card())
    cfg = default_cfg("dla_34")
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    threads = cv2.getNumThreads()
    for persons in (1, 5, 10):
        images, results = workload(a.n, persons)
        det.render_poses(images[:8], results[:8])                    # warm-up: module load, text tables
        dev, one, many = [], [], []
        for _ in range(a.rounds):
            t, got = timed(lambda: det.render_poses(images, results))
            dev.append(a.n / t)
            for store, nt in ((one, 1), (many, threads)):
                cv2.setNumThreads(nt)
                t0 = time.perf_counter()
                want = [debugger_ref.show_results(im, r.tolist(), 0.3, cfg.DEBUG_THEME) for im, r in zip(images, results)]
                store.append(a.n / (time.perf_counter() - t0))
            cv2.setNumThreads(threads)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), "render_poses != oracle"
        print("render %2d persons/image, N=%d: device %s images/s; cv2 oracle 1 thread %s, %d threads %s (identical)"
              % (persons, a.n, "/".join("%.0f" % v for v in dev), "/".join("%.1f" % v for v in one), threads,
                 "/".join("%.1f" % v for v in many)))
    # run_images with and without the drawing, dla_34's test section
    for k, v in TEST_SECTIONS["dla_34"].items():
        det.cfg.TEST[k] = v
    det.scales = det.cfg.TEST.TEST_SCALES
    images, _ = workload(a.run_images, 1)
    det.run_images(images[:8])
    det.run_images(images[:8], return_images=True)
    plain, drawn = [], []
    for _ in range(a.rounds):
        t, rows = timed(lambda: det.run_images(images))
        plain.append(len(images) / t)
        t, (rows2, imgs) = timed(lambda: det.run_images(images, return_images=True))
        drawn.append(len(images) / t)
        assert all(np.array_equal(x, y) for x, y in zip(rows, rows2)), "return_images changed the rows"
    print("run_images %d images (FLIP_TEST %s, NMS %s): %s images/s, with return_images %s images/s (rows identical)"
          % (len(images), det.cfg.TEST.FLIP_TEST, det.cfg.TEST.NMS, "/".join("%.0f" % v for v in plain),
             "/".join("%.0f" % v for v in drawn)))


if __name__ == "__main__":
    main()

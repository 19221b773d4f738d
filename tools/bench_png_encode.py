"""PNG encoding throughput: png.encode (cpb200_png_encode_batch; upload, launch and both copies back included)
against cv2.imencode('.png') on one host thread and on a pool of os.cpu_count() threads, at 1, 16 and 256 images,
and run_images(return_images=True, encode_png=True) against run_images(return_images=True) followed by host
cv2.imencode.  The images are seeded COCO-sized photos (640x480 / 480x640 / 640x427) with 5 persons drawn by
render_poses each, and 512 x 512 heat-map views from heatmaps.views.  Three alternating rounds; the files are
compared byte for byte in every round.  Prints the card and its power limit.

    python tools/bench_png_encode.py [--rounds 3] [--run-images 64]
"""
from __future__ import annotations

import argparse
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from centerpose_b200 import heatmaps, png, render  # noqa: E402
from centerpose_b200.config import default_cfg  # noqa: E402
from centerpose_b200.detector import detector_factory  # noqa: E402
from oracle.init_recipe import conditioned_state_dict  # noqa: E402
from tools.bench_images import TEST_SECTIONS  # noqa: E402
from tools.bench_render import card, timed, workload  # noqa: E402


def drawn_images(n):
    images, results = workload(n, 5)
    shapes = [im.shape[:2] for im in images]
    pixels, offsets = render.launch(render.build(shapes, results, 0.3, "white"), images=images)
    return render.download(pixels, offsets, shapes)


def views(n):
    rng = np.random.default_rng(5)
    x = [torch.from_numpy(rng.normal(0, 1, (3, 512, 512)).astype(np.float32)).cuda() for _ in range(n)]
    hm = [torch.from_numpy((rng.random((1, 128, 128)) ** 4).astype(np.float32)).cuda() for _ in range(n)]
    hp = [torch.from_numpy((rng.random((17, 128, 128)) ** 6).astype(np.float32)).cuda() for _ in range(n)]
    v = heatmaps.views(x, hm, hp, 4, "white", np.array([0.408, 0.447, 0.470]), np.array([0.289, 0.274, 0.278]))
    return [d[k] for d in v for k in heatmaps.VIEWS]


def host_encode(images, pool=None):
    enc = lambda im: cv2.imencode(".png", im)[1].tobytes()
    return list(pool.map(enc, images)) if pool else [enc(im) for im in images]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--run-images", type=int, default=64)
    a = ap.parse_args()
    print("card:", card())
    threads = os.cpu_count()
    pool = ThreadPoolExecutor(threads)
    cv2.setNumThreads(1)          # one image per host thread; the pool supplies the parallelism
    for what, make in (("drawn poses", drawn_images), ("heat-map views", lambda n: views(n // 2))):
        pool_imgs = make(256)
        png.encode(pool_imgs[:4])                                        # warm-up
        for n in (1, 16, 256):
            imgs = pool_imgs[:n]
            dev, one, many = [], [], []
            for _ in range(a.rounds):
                t, got = timed(lambda: png.encode(imgs))
                dev.append(n / t)
                t0 = time.perf_counter()
                want = host_encode(imgs)
                one.append(n / (time.perf_counter() - t0))
                t0 = time.perf_counter()
                want2 = host_encode(imgs, pool)
                many.append(n / (time.perf_counter() - t0))
                assert got == want == want2, "png.encode != cv2.imencode"
            print("%s, %d images: png.encode %s images/s; cv2.imencode 1 thread %s, %d threads %s (identical)"
                  % (what, n, "/".join("%.0f" % v for v in dev), "/".join("%.1f" % v for v in one), threads,
                     "/".join("%.1f" % v for v in many)))
    cfg = default_cfg("dla_34")
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    for k, v in TEST_SECTIONS["dla_34"].items():
        det.cfg.TEST[k] = v
    det.scales = det.cfg.TEST.TEST_SCALES
    images, _ = workload(a.run_images, 1)
    det.run_images(images[:8], return_images=True)
    det.run_images(images[:8], return_images=True, encode_png=True)
    dev, host = [], []
    for _ in range(a.rounds):
        t, (rows, files) = timed(lambda: det.run_images(images, return_images=True, encode_png=True))
        dev.append(len(images) / t)
        t0 = time.perf_counter()
        rows2, drawn = det.run_images(images, return_images=True)
        want = host_encode(drawn, pool)
        host.append(len(images) / (time.perf_counter() - t0))
        assert all(np.array_equal(x, y) for x, y in zip(rows, rows2)), "encode_png changed the rows"
        assert files == want, "encode_png != cv2.imencode of the drawn images"
    print("run_images %d images (FLIP_TEST %s, NMS %s) to PNG files: encode_png %s images/s; return_images + "
          "cv2.imencode on %d threads %s images/s (rows and bytes identical)"
          % (len(images), det.cfg.TEST.FLIP_TEST, det.cfg.TEST.NMS, "/".join("%.0f" % v for v in dev), threads,
             "/".join("%.0f" % v for v in host)))
    pool.shutdown()


if __name__ == "__main__":
    main()

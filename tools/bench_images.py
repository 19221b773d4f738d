"""Raw-image detection throughput on one GPU: ``MultiPoseDetector.run_images`` against a per-image ``run()`` loop.

    python tools/bench_images.py [--images 64] [--rounds 3] [--max-batch 32] [--precision fp16x2]

DLA-34 with conditioned weights (``centerpose_b200.synth``) and the test section of the reference's
``experiments/dla_34_512x512.yaml``: flip test, soft-NMS, ``FIX_RES: false`` (each image padded to (h|31)+1 x
(w|31)+1), scales [1].  The images are seeded uint8 noise at COCO-like sizes, 640x480, 480x640 and 640x427 in turn.
Both paths take the same host arrays and return the same rows (original-image pixels, after soft-NMS), so each time
covers upload, pre-process, forward, flip merge, decode, back-projection, NMS and the copy back.

After one warm-up pass of each (plans are built per input shape and batch), the two are timed in alternating rounds
with a host clock; every call ends in a device-to-host copy of its results, so the clock covers the device work.
Agreement: per image, the number of rows whose score is at least soft-NMS's 0.001 threshold in each path, and the
largest absolute difference of any value.  The card's name, power limit and SM clocks are read (nvidia-smi
--query-gpu, read-only) before and after the timed rounds.  Prints one JSON line.  Fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_hardnet import gpu_info  # noqa: E402

SIZES = [(480, 640), (640, 480), (427, 640)]     # (h, w)


def detector(precision):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from centerpose_b200.synth import conditioned_state_dict
    cfg = default_cfg("dla_34")
    cfg.TEST.FLIP_TEST = True                     # experiments/dla_34_512x512.yaml, TEST section
    cfg.TEST.NMS = True
    cfg.TEST.FIX_RES = False
    cfg.TEST.TEST_SCALES = [1]
    cfg.B200.PRECISION = precision
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    det.model.set_precision(precision)
    return det


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--precision", default="fp16x2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_images.py needs a CUDA device (there is no CPU path to time)")
    torch.cuda.set_device(0)
    rng = np.random.RandomState(317)
    images = [rng.randint(0, 256, size=SIZES[i % len(SIZES)] + (3,)).astype(np.uint8) for i in range(args.images)]
    det = detector(args.precision)
    hw_before = gpu_info(0)

    def batched():
        return det.run_images(images, max_batch=args.max_batch)

    def loop():
        return [np.asarray(det.run(im)["results"][1], dtype=np.float32) for im in images]

    got, want = batched(), loop()                 # warm-up (plans for every shape and batch) and the parity sample
    times = {"run_images": [], "run_loop": []}
    for _ in range(args.rounds):
        for name, fn in (("run_images", batched), ("run_loop", loop)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
    kept_a = [int((g[:, 4] >= 0.001).sum()) for g in got]
    kept_b = [int((w[:, 4] >= 0.001).sum()) for w in want]
    result = {
        "metric": "images/sec, raw uint8 images -> rows after flip test + soft-NMS, DLA-34, dla_34_512x512 test section",
        "precision": args.precision, "images": args.images, "sizes_hw": SIZES, "max_batch": args.max_batch,
        "rounds": args.rounds,
        "run_images_images_per_s": [args.images / t for t in times["run_images"]],
        "run_loop_images_per_s": [args.images / t for t in times["run_loop"]],
        "median_speedup": statistics.median(times["run_loop"]) / statistics.median(times["run_images"]),
        "rows_per_image": int(got[0].shape[0]),
        "kept_rows_equal_images": int(sum(a == b for a, b in zip(kept_a, kept_b))),
        "kept_rows_total": [sum(kept_a), sum(kept_b)],
        "max_abs_diff": float(max(np.abs(g - w).max() for g, w in zip(got, want))),
        "max_abs_ref": float(max(np.abs(w).max() for w in want)),
        "gpu_before": hw_before, "gpu_after": gpu_info(0),
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()

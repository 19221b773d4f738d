"""COCO keypoint evaluation time: the reference's host path (coco_format.convert_eval_format into result dicts, then
the numpy restatement of COCOeval in oracle/cocoeval_ref.py, and pycocotools itself when it is importable) against
KeypointEval.evaluate on the device (the upload of the rows and the copy back included; the ground truth is parsed
and uploaded once, outside the timing, as a user evaluating several checkpoints would).  The input is N synthetic
images (default 5000, val2017's count) with 100 rows each against a matching synthetic ground truth
(tests/coco_eval_cases.py).  Three alternating rounds; the results are compared bit for bit in the same run.  Prints
the card and its power limit.

    python tools/bench_coco_eval.py [--n 5000] [--rows 100] [--rounds 3]
"""
from __future__ import annotations

import argparse
import contextlib
import io
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from centerpose_b200.coco_eval import KeypointEval  # noqa: E402
from centerpose_b200.coco_format import convert_eval_format  # noqa: E402
from oracle import cocoeval_ref  # noqa: E402
from tests.coco_eval_cases import make_case  # noqa: E402
from tools.bench_render import card, timed  # noqa: E402


def pycocotools_eval(gt, dets):
    try:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
    except ImportError:
        return None
    coco = COCO()
    coco.dataset = gt
    coco.createIndex()
    E = COCOeval(coco, coco.loadRes(dets), "keypoints")
    E.evaluate()
    E.accumulate()
    E.summarize()
    return E


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=5000)
    ap.add_argument("--rows", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print("card:", card())
    gt, res = make_case(11, n_images=a.n, gts_per_image=(1, 4), rows_per_image=a.rows)    # TOPK rows per image
    n_rows = sum(len(v[1]) for v in res.values())
    print("workload: %d images, %d with detections, %d rows, %d ground truths"
          % (a.n, len(res), n_rows, len(gt["annotations"])))
    ev = KeypointEval(gt)
    ev.evaluate(res)                                  # warm-up: module load, first allocations
    dev, fmt, ora, pyc = [], [], [], []
    for _ in range(a.rounds):
        t, stats = timed(lambda: ev.evaluate(res))
        dev.append(t)
        t0 = time.perf_counter()
        dets = convert_eval_format(res)
        t1 = time.perf_counter()
        E = cocoeval_ref.evaluate(gt, dets, out=None)
        t2 = time.perf_counter()
        fmt.append(t1 - t0)
        ora.append(t2 - t1)
        for k in ("precision", "recall", "scores"):
            assert np.array_equal(ev.eval[k], E.eval[k], equal_nan=True), k + " != oracle"
        assert np.array_equal(stats, E.stats), "stats != oracle"
        with contextlib.redirect_stdout(io.StringIO()):
            t0 = time.perf_counter()
            P = pycocotools_eval(gt, dets)
            t1 = time.perf_counter()
        if P is not None:
            pyc.append(t1 - t0)
            for k in ("precision", "recall", "scores"):
                assert np.array_equal(ev.eval[k], P.eval[k], equal_nan=True), k + " != pycocotools"
    s = lambda v: "/".join("%.3f" % x for x in v)
    print("KeypointEval.evaluate (upload, kernels, copy back): %s s" % s(dev))
    print("host: convert_eval_format %s s + numpy COCOeval restatement %s s" % (s(fmt), s(ora)))
    print("pycocotools loadRes + evaluate/accumulate/summarize: %s" % (s(pyc) + " s" if pyc else "not importable"))
    print("results identical in every round; AP %.4f" % stats[0])


if __name__ == "__main__":
    main()

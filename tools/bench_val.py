"""Validation-pass throughput: ``MultiPoseDetector.run_val`` against the same pass with the targets built on the host
by the numpy restatement (oracle/val_ref.py) and uploaded, which is the work the reference's data loader does; the
forward, the loss and the decode run on the device in both.  Then the targets and loss kernels alone, timed with
CUDA events, with their bytes over the H100 SXM data-sheet bandwidth (3.35 TB/s) as the share of the HBM bound.

Workload: N seeded COCO-sized JPEG files (default 256) with 2..8 synthetic people each, DLA-34 at 512x512 in
``fp16x2``, batches of 32.  Three alternated rounds; the two arms' stats and rows are compared in the same run.
Prints the card and its power limit.

    python tools/bench_val.py [--n 256] [--rounds 3]
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from centerpose_b200 import val  # noqa: E402
from centerpose_b200.coco_eval import KeypointEval, gt_table  # noqa: E402
from centerpose_b200.config import default_cfg  # noqa: E402
from centerpose_b200.detector import detector_factory  # noqa: E402
from centerpose_b200.image import get_affine_transform  # noqa: E402
from centerpose_b200.synth import conditioned_state_dict  # noqa: E402
from oracle import val_ref  # noqa: E402
from oracle.make_golden_val import image  # noqa: E402
from tests.val_cases import _ann, _dataset, _person  # noqa: E402
from tools.bench_render import card, timed  # noqa: E402

SHAPES = [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375)]
HBM = 3.35e12


def workload(n, d):
    rng = np.random.default_rng(5)
    paths, images, anns, aid = [], [], [], 1
    for k in range(n):
        h, w = SHAPES[k % len(SHAPES)]
        paths.append(os.path.join(d, "%d.jpg" % k))
        cv2.imwrite(paths[-1], image(5000 + k, h, w), [cv2.IMWRITE_JPEG_QUALITY, 90])
        images.append((k + 1, h, w))
        for _ in range(int(rng.integers(2, 9))):
            bw, bh = rng.uniform(0.1, 0.5) * w, rng.uniform(0.2, 0.9) * h
            x, y = rng.uniform(0, w - bw), rng.uniform(0, h - bh)
            anns.append(_ann(aid, k + 1, [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)],
                             _person(rng, x, y, bw, bh, "partial"), crowd=int(rng.random() < 0.05)))
            aid += 1
    return paths, _dataset(images, anns)


def host_targets_factory(ds):
    """``val.targets`` with the numpy restatement on the host and one upload per array."""
    per = {im["id"]: gt_table([a for a in ds["annotations"] if a["image_id"] == im["id"]]) for im in ds["images"]}

    def targets(ev, image_ids, shapes, cfg):
        R = int(cfg.MODEL.OUTPUT_RES)
        tgs = []
        for i, (h, w) in zip(image_ids, shapes):
            c, s = val.center_scale(h, w)
            tgs.append(val_ref.targets(per[i], get_affine_transform(c, s, 0, [R, R]), R))
        return {k: torch.from_numpy(np.stack([t[k] for t in tgs])).to(ev.device, non_blocking=True)
                for k, _, _ in val.TARGETS}
    return targets


def kernel_times(det, ev, ds, cfg, reps=50):
    """The targets and loss kernels on one batch of 32 images, their tables already on the device: mean ms per
    call (CUDA events around ``reps`` calls of each entry point) and the bytes each moves at least."""
    import ctypes
    from centerpose_b200 import _lib
    L = _lib.lib()
    ids = [im["id"] for im in ds["images"][:32]]
    shapes = [(im["height"], im["width"]) for im in ds["images"][:32]]
    R = int(cfg.MODEL.OUTPUT_RES)
    with torch.no_grad():
        outputs = det.model(torch.zeros((32, 3, 512, 512), device="cuda"))
    tg = val.targets(ev, ids, shapes, cfg)
    table = torch.from_numpy(val.image_table(ev, ids, shapes, R).view(np.uint8).reshape(-1).copy()).cuda()
    ptrs = val.targets_struct(tg)
    heads = _lib.Heads(*[o.data_ptr() for o in outputs])
    lcfg = val.loss_cfg(cfg)
    stats = torch.empty((32, len(val.STATS)), device="cuda")
    ws = torch.empty(L.cpb200_multi_pose_loss_workspace_bytes(32), dtype=torch.uint8, device="cuda")
    calls = {"targets": lambda: _lib.launch("multi_pose_targets_batch", table.device, table, 32, ev.gts, R, ptrs),
             "loss": lambda: _lib.launch("multi_pose_loss_batch", table.device, heads, ptrs, 32, R, ctypes.byref(lcfg),
                                         stats, ws)}
    res = {}
    for name, fn in calls.items():
        fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        res[name] = a.elapsed_time(b) / reps
    nbytes = lambda ts: sum(t.numel() * t.element_size() for t in ts)
    # the targets are written once; the loss reads both heat maps and their targets once, and the sparse targets
    return res, {"targets": nbytes(tg.values()),
                 "loss": nbytes([outputs[0], outputs[4]] + list(tg.values()))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print("card:", card())
    cfg = default_cfg("dla_34")
    cfg.B200.PRECISION = "fp16x2"
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    with tempfile.TemporaryDirectory() as d:
        paths, ds = workload(a.n, d)
        ids = [im["id"] for im in ds["images"]]
        ev = KeypointEval(ds)
        print("workload: %d JPEG files, %d annotations, DLA-34 fp16x2 at 512x512, batches of 32"
              % (len(paths), len(ds["annotations"])))
        device_targets, host_targets = val.targets, host_targets_factory(ds)
        det.run_val(paths[:32], ids[:32], ev)                        # warm-up: module load, first allocations
        dev_t, host_t = [], []
        for r in range(a.rounds):
            val.targets = device_targets
            t, (log_d, preds_d) = timed(lambda: det.run_val(paths, ids, ev))
            dev_t.append(t)
            val.targets = host_targets
            t, (log_h, preds_h) = timed(lambda: det.run_val(paths, ids, ev))
            host_t.append(t)
            val.targets = device_targets
            same = all(log_d[k] == log_h[k] for k in val.STATS) and \
                all(np.array_equal(preds_d[i][1], preds_h[i][1]) for i in ids)
            print("round %d: run_val %.1f images/s, host targets %.1f images/s, outputs identical: %s"
                  % (r, a.n / dev_t[-1], a.n / host_t[-1], same))
            assert same
        print("run_val: %.1f-%.1f images/s; with the targets on the host: %.1f-%.1f images/s"
              % (a.n / max(dev_t), a.n / min(dev_t), a.n / max(host_t), a.n / min(host_t)))
        print("stats:", {k: round(v, 6) for k, v in log_d.items() if k != "time"})
        ms, nbytes = kernel_times(det, ev, ds, cfg)
        for k in ("targets", "loss"):
            print("%s kernels, 32 images: %.3f ms, %.1f MB, %.1f%% of the HBM bound (%.3f ms at 3.35 TB/s)"
                  % (k, ms[k], nbytes[k] / 1e6, 100 * nbytes[k] / HBM / (ms[k] / 1e3), nbytes[k] / HBM * 1e3))


if __name__ == "__main__":
    main()

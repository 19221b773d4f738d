"""Training-batch throughput: ``TrainData.batch`` (decode, warp, colour augmentation and targets on the device)
against the host loader it replaces, the reference's ``__getitem__`` work in numpy and cv2 per image (``cv2.imread``,
``cv2.warpAffine``, ``color_aug``'s in-place float32 steps with ``cv2.cvtColor`` and ``gs.mean()``, the normalisation,
and the targets of ``oracle/train_ref.py``) on 1 and on 8 threads.  The host draws are made once per batch in both
arms, in order, so the two produce the same batch; it is compared element for element in every round.  Then the new
kernels alone (``cpb200_train_augment_batch``, ``cpb200_multi_pose_targets_train_batch``) timed with CUDA events, with
the bytes they must move computed from the shapes.

Workload: N seeded COCO-sized JPEG files (default 64) with 2..8 synthetic people each, INPUT_RES 512, batches of 32,
the reference's default augmentation (random crop, flip 0.5, colour on).  Three alternated rounds.  Prints the card and
its power limit.

    python tools/bench_train_data.py [--n 64] [--rounds 3]
"""
from __future__ import annotations

import argparse
import ctypes
import os
import random
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from centerpose_b200 import _lib, train_data, val  # noqa: E402
from centerpose_b200.coco_eval import gt_table  # noqa: E402
from centerpose_b200.config import default_cfg  # noqa: E402
from centerpose_b200.detector import load_images_device  # noqa: E402
from centerpose_b200.image import get_affine_transform  # noqa: E402
from oracle import train_ref  # noqa: E402
from tools.bench_render import card, timed  # noqa: E402
from tools.bench_val import workload  # noqa: E402

B = 32


def host_item(path, p, gts, cfg):
    """One image as the reference's __getitem__ computes it, from the draws ``p``."""
    S, R = cfg.MODEL.INPUT_RES, cfg.MODEL.OUTPUT_RES
    img = cv2.imread(path)
    if p["flip"]:
        img = img[:, ::-1, :]
    inp = cv2.warpAffine(img, get_affine_transform(p["c"], p["s"], p["rot"], [S, S]), (S, S), flags=cv2.INTER_LINEAR)
    inp = inp.astype(np.float32) / 255.
    if p["color"]:
        gs = cv2.cvtColor(inp, cv2.COLOR_BGR2GRAY)
        gs_mean = gs.mean()
        for op, alpha in zip(p["order"], p["alpha"]):
            inp *= alpha
            if op == 1:
                inp += gs_mean * (1 - alpha)
            elif op == 2:
                gs *= (1 - alpha)
                inp += gs[:, :, None]
        inp += p["light"]
    inp = (inp - np.array(cfg.DATASET.MEAN, np.float32)) / np.array(cfg.DATASET.STD, np.float32)
    out = train_ref.targets(gts, img.shape[1], p["flip"], p["rot"], get_affine_transform(p["c"], p["s"], 0, [R, R]),
                            get_affine_transform(p["c"], p["s"], p["rot"], [R, R]), R)
    out["input"] = inp.transpose(2, 0, 1)
    return out


def host_batch(paths, ds, draws, per, cfg, pool):
    """The host loader: draws in order, then the images on the pool, then default_collate's stack."""
    ps = [draws.draw(im["height"], im["width"]) for im in ds["images"][:len(paths)]]
    ids = [im["id"] for im in ds["images"][:len(paths)]]
    items = list(pool.map(lambda a: host_item(a[0], a[1], per[a[2]], cfg), zip(paths, ps, ids)))
    return {k: np.stack([it[k] for it in items]) for k in items[0]}


def kernels_alone(tr, paths, ids, reps=20):
    """CUDA-event times of the two kernels on a loaded batch; bytes from the shapes."""
    cfg = tr.cfg
    S, R = cfg.MODEL.INPUT_RES, cfg.MODEL.OUTPUT_RES
    loaded, offsets, pixels = load_images_device(paths)
    table = np.zeros(len(paths), train_data.TRAIN_IMAGE)
    for n in range(len(paths)):
        h, w = loaded[n].shape[0:2]
        tr.table_row(table[n], tr.draws.draw(h, w), h, w, offsets[n], ids[n])
    dev = pixels.device
    up = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).to(dev)
    plan = torch.from_numpy(train_data.mean_plan(S * S)).to(dev)
    L = _lib.lib()
    n = len(paths)
    inp = torch.empty((n, 3, S, S), dtype=torch.float32, device=dev)
    ws = torch.empty(L.cpb200_train_augment_workspace_bytes(n, S), dtype=torch.uint8, device=dev)
    tg = {k: torch.empty((n,) + shape(R), dtype=dt, device=dev) for k, dt, shape in val.TARGETS}
    mean = (ctypes.c_float * 3)(*np.float32(cfg.DATASET.MEAN))
    std = (ctypes.c_float * 3)(*np.float32(cfg.DATASET.STD))
    stream = torch.cuda.current_stream().cuda_stream
    ptrs = val._pointers(_lib.Targets, tg, [k for k, _, _ in val.TARGETS])

    def aug():
        _lib.check(L.cpb200_train_augment_batch(pixels.data_ptr(), up.data_ptr(), n, S, plan.data_ptr(), mean, std,
                                                inp.data_ptr(), ws.data_ptr(), ws.numel(), stream))

    def tgt():
        _lib.check(L.cpb200_multi_pose_targets_train_batch(up.data_ptr(), n, tr.ev.gts.data_ptr(), R, ptrs, stream))

    out = {}
    src_bytes = sum(int(np.prod(v.shape)) for v in loaded)
    # warp: sampled source (at most the images) + uint8 and grey planes; mean: grey planes; colour: uint8 and grey
    # planes in, the float32 input out
    aug_bytes = src_bytes + n * S * S * (3 + 4) + n * S * S * 4 + n * S * S * (3 + 4) + inp.numel() * 4
    tgt_bytes = sum(t.numel() * t.element_size() for t in tg.values())
    for name, fn, nbytes in (("augment", aug, aug_bytes), ("targets", tgt, tgt_bytes)):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = {"ms": round(ms, 4), "bytes": int(nbytes), "GB/s": round(nbytes / ms / 1e6, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print("card:", card())
    cfg = default_cfg("dla_34")
    with tempfile.TemporaryDirectory() as d:
        paths, ds = workload(a.n, d)
        per = {im["id"]: gt_table([x for x in ds["annotations"] if x["image_id"] == im["id"]]) for im in ds["images"]}
        ids = [im["id"] for im in ds["images"]]
        tr = train_data.TrainData(cfg, ds)
        tr.batch(paths[:B], ids[:B])                              # warm-up: library load, first launches
        pools = {1: ThreadPoolExecutor(1), 8: ThreadPoolExecutor(8)}
        times = {"device": [], "host_1": [], "host_8": []}
        for r in range(a.rounds):
            for arm in ("device", "host_1", "host_8"):
                got, total = [], 0.0
                for s in range(0, a.n, B):
                    np.random.seed(100 + r * 1000 + s)
                    random.seed(200 + r * 1000 + s)
                    if arm == "device":
                        tr.draws = train_data.TrainDraws(cfg)
                        t, out = timed(lambda: tr.batch(paths[s:s + B], ids[s:s + B]))
                        out = {k: v.cpu().numpy() for k, v in out.items()}
                    else:
                        draws = train_data.TrainDraws(cfg)
                        t0 = time.perf_counter()
                        out = host_batch(paths[s:s + B], {"images": ds["images"][s:s + B]}, draws, per, cfg,
                                         pools[int(arm[-1])])
                        t = time.perf_counter() - t0
                    total += t
                    got.append(out)
                times[arm].append(a.n / total)
                if arm == "device":
                    ref = got
                else:
                    for x, y in zip(ref, got):
                        for k in x:
                            assert np.array_equal(np.ascontiguousarray(x[k]).view(np.uint8),
                                                  np.ascontiguousarray(y[k]).view(np.uint8)), (arm, r, k)
            print("round %d: images/s device %.1f, host 1 thread %.1f, host 8 threads %.1f (identical)"
                  % (r, times["device"][-1], times["host_1"][-1], times["host_8"][-1]))
        tr.draws = train_data.TrainDraws(cfg)
        print("kernels alone, B = %d:" % B, kernels_alone(tr, paths[:B], ids[:B]))


if __name__ == "__main__":
    main()

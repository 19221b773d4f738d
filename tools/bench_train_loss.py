"""Time the trainer's loss on the device: ``train_loss.MultiPoseLoss`` forward + backward against the torch op sequence
the reference runs (``oracle/train_loss_ref.loss_torch`` with autograd) on the same device, and the new kernels alone.

    python tools/bench_train_loss.py [--B 32] [--res 512] [--steps 50] [--warmup 10] [--rounds 3]

Workload: B TrainData images (seeded synthetic JPEG files with people, INPUT_RES 512, so R = 128) and seeded logits.
Per round and arm: CUDA-event time per step after a warm-up, the outputs of the two arms compared, and the rise of
``torch.cuda.max_memory_allocated`` over one step.  Rounds alternate the arms.  The kernels alone are timed with
events around the C entry points, and their bytes (the dense maps they read and write; the gathers are negligible) are
set against the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.  Prints
one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import random
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch is enough to label the numbers
        q = "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)
    return q


def workload(B, res, d):
    from centerpose_b200 import train_data
    from centerpose_b200.config import default_cfg
    from oracle.make_golden_val import image
    from tests.train_cases import case_cfg, seeded_case
    from tests.train_loss_cases import logits
    cfg = case_cfg(default_cfg("dla_34"), {"AUG_ROT": 0.3, "ROTATE": 30., "FLIP": 0.5}, res)
    ds = seeded_case(700, B, lo=200, hi=700, people=(1, 12))
    paths = []
    for im in ds["images"]:
        p = os.path.join(d, "%d.jpg" % im["id"])
        cv2.imwrite(p, image(9000 + im["id"], im["height"], im["width"]), [cv2.IMWRITE_JPEG_QUALITY, 90])
        paths.append(p)
    np.random.seed(60)
    random.seed(70)
    batch = train_data.TrainData(cfg, ds).batch(paths, [im["id"] for im in ds["images"]])
    R = cfg.MODEL.OUTPUT_RES
    heads = [torch.from_numpy(h).cuda() for h in logits(31, B, R)]
    return cfg, batch, heads


def step_fn(cfg, batch, heads, device_arm):
    from centerpose_b200 import train_loss
    from oracle import train_loss_ref
    crit = train_loss.MultiPoseLoss(cfg, 0)
    leaves = [h.clone().requires_grad_(True) for h in heads]

    def clear():
        for x in leaves:
            x.grad = None

    def step():
        clear()
        if device_arm:
            loss, st = crit(leaves, batch)
        else:
            loss, st = train_loss_ref.loss_torch(leaves, batch, cfg.LOSS)
        loss.backward()
        return st, leaves
    step.clear = clear
    return step


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def peak_rise(step):
    """The rise of the allocator's peak over one step from no gradient held: the six gradient maps and whatever the
    arm keeps for its backward."""
    step.clear()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def compare(dev, ref):
    (sd, gd), (sr, gr) = dev, ref
    stats = max(abs(float(sd[k]) - float(sr[k])) / max(abs(float(sr[k])), 1e-30) for k in sd)
    grads = {}
    for name, x, y in zip(("hm", "wh", "hps", "reg", "hm_hp", "hp_offset"), gd, gr):
        d = (x.grad - y.grad).abs().max().item()
        grads[name] = d / max(y.grad.abs().max().item(), 1e-30)
    return stats, grads


def kernels_alone(cfg, batch, heads, reps):
    from centerpose_b200 import _lib, val
    from centerpose_b200.train_loss import _targets_struct, target_keys
    L = _lib.lib()
    B, R = heads[0].shape[0], heads[0].shape[-1]
    ws = torch.empty(L.cpb200_multi_pose_loss_train_workspace_bytes(B), dtype=torch.uint8, device="cuda")
    stats = torch.empty(7, device="cuda")
    loss = torch.empty((), device="cuda")
    one = torch.ones((), device="cuda")
    grads = [torch.empty_like(h) for h in heads]
    hs = _lib.Heads(*[h.data_ptr() for h in heads])
    gs = _lib.Heads(*[g.data_ptr() for g in grads])
    ts = _targets_struct(batch, target_keys(cfg))
    lc = val.loss_cfg(cfg)
    s = torch.cuda.current_stream().cuda_stream

    def fwd():
        _lib.check(L.cpb200_multi_pose_loss_train_batch(hs, ts, B, R, ctypes.byref(lc), stats.data_ptr(),
                                                        loss.data_ptr(), ws.data_ptr(), s))

    def bwd():
        _lib.check(L.cpb200_multi_pose_loss_train_backward(hs, ts, B, R, ctypes.byref(lc), one.data_ptr(),
                                                           ws.data_ptr(), gs, s))
    out = {}
    fwd()
    plane = B * R * R * 4
    # forward: logits and targets of hm and hm_hp; backward: those again, their gradients, and the 40 regression
    # channels zero-filled
    for name, fn, nbytes in (("forward", fwd, 2 * 18 * plane), ("backward", bwd, 3 * 18 * plane + 40 * plane)):
        ms = time_steps(fn, reps, 5)
        out[name] = {"ms": round(ms, 4), "bytes": nbytes, "GB_s": round(nbytes / ms / 1e6, 1),
                     "share_of_3.35TB_s": round(nbytes / (ms * 1e-3) / HBM_BPS, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loss: needs a CUDA device")
    with tempfile.TemporaryDirectory() as d:
        cfg, batch, heads = workload(a.B, a.res, d)
    arms = {"device": step_fn(cfg, batch, heads, True), "torch": step_fn(cfg, batch, heads, False)}
    rounds = []
    for r in range(a.rounds):
        row = {}
        for name in (("device", "torch") if r % 2 == 0 else ("torch", "device")):
            row[name + "_ms"] = round(time_steps(arms[name], a.steps, a.warmup), 4)
            row[name + "_peak_rise_MB"] = round(peak_rise(arms[name]) / 2 ** 20, 1)
        row["stats_rel_diff"], row["grad_rel_diff"] = compare(arms["device"](), arms["torch"]())
        rounds.append(row)
    res = {"bench": "train_loss", "card": card(), "B": a.B, "R": a.res // 4, "rounds": rounds,
           "kernels": kernels_alone(cfg, batch, heads, 200)}
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

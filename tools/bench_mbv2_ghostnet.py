"""MobileNetV2 and GhostNet throughput and parity on one GPU: forward + fused decode of device-resident 512x512 batches,
fp16x2 and bf16.

    python tools/bench_mbv2_ghostnet.py [--steps 20] [--warmup 3] [--batch 64] [--rounds 3]

Prints one JSON line.  Every (backbone, precision) model is built and warmed up first; then ``--rounds`` rounds each
time every model once, in turn, so that the models alternate and the spread between rounds shows the noise of the
shared host.  Per model: images/s of each round (CUDA events around ``--steps`` steps, inputs rotated over four
resident batches), their range, and the parity of the head maps / decoded rows against
tests/golden/{mbv2,ghostnet}_512.npz (the unmodified reference on the CPU).  The card's name, power limit and SM clocks
are read (nvidia-smi --query-gpu, read-only) before and after the timed rounds.  Fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_hardnet import gpu_info  # noqa: E402

IMG = 512
K_DET = 100
GOLDEN = {"mobilenetv2": "mbv2_512", "ghostnet": "ghostnet_512"}


def build(dev, arch, precision):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from centerpose_b200.synth import conditioned_state_dict
    cfg = default_cfg(arch)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    m.load_state_dict(conditioned_state_dict(m.state_dict(), 317))
    return m.to(dev).set_precision(precision)


def parity(model, dev, arch):
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.synth import synth_images
    from tests.util import match_rows
    g = np.load(os.path.join(ROOT, "tests", "golden", GOLDEN[arch] + ".npz"))
    st = int(g["stride"])
    outs = model(synth_images(1, IMG, IMG, 317).to(dev))
    maps = torch.cat(outs, dim=1).cpu().numpy()[:, :, ::st, ::st].astype(np.float64)
    ref = g["maps"].astype(np.float64)
    dets = multi_pose_decode(outs[0], outs[1], outs[2], reg=outs[3], hm_hp=outs[4], hp_offset=outs[5], K=K_DET,
                             apply_sigmoid=True)[0].cpu().numpy()
    rows, elems = match_rows(dets, g["dets"][0], tol=1e-3, box_tol=2e-2)
    return {"head_maps_rel_l2": float(np.linalg.norm(maps - ref) / np.linalg.norm(ref)),
            "head_maps_max_abs_over_max": float(np.abs(maps - ref).max() / np.abs(ref).max()),
            "rows_matched": rows, "elements_within_1e-3": elems,
            "tolerance": "rows matched on bbox + score within 2e-2, then |err| <= 1e-3 * max(1, |ref|) per value"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--archs", default="mobilenetv2,ghostnet")
    ap.add_argument("--precisions", default="fp16x2,bf16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_mbv2_ghostnet.py needs a CUDA device (there is no CPU path to time)")
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.synth import synth_images
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    inputs = [synth_images(B, IMG, IMG, 317 + i).to(dev) for i in range(4)]
    models = {(a, p): build(dev, a, p) for a in args.archs.split(",") for p in args.precisions.split(",")}

    def step(model, i):
        hm, wh, hps, reg, hm_hp, hp_off = model(inputs[i % len(inputs)])
        return multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_off, K=K_DET, apply_sigmoid=True)

    for model in models.values():
        for i in range(max(args.warmup, 1)):
            step(model, i)
    torch.cuda.synchronize()
    hw_before = gpu_info(0)
    rates = {key: [] for key in models}
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for key, model in models.items():
            e0.record()
            for i in range(args.steps):
                step(model, i)
            e1.record()
            torch.cuda.synchronize()
            rates[key].append(B * args.steps / (e0.elapsed_time(e1) / 1e3))
    hw_after = gpu_info(0)
    result = {"metric": "images/sec 512x512 forward + decode, device-resident batches", "batch": B, "steps": args.steps,
              "warmup": args.warmup, "rounds": args.rounds, "models": {}}
    for (arch, precision), model in models.items():
        plan = next(iter(model._plans.values()))
        r = rates[(arch, precision)]
        result["models"][f"{arch}/{precision}"] = {
            "images_per_s": r, "images_per_s_range": [min(r), max(r)], "ops": int(plan.n),
            "convert_ops": int(sum(1 for o in plan.ops if o.type == 11)),
            "parity_vs_512_golden": parity(model, dev, arch)}
    result["gpu_before"] = hw_before
    result["gpu_after"] = hw_after
    print(json.dumps(result))


if __name__ == "__main__":
    main()

"""HarDNet throughput and parity on one GPU: forward + fused decode of device-resident 512x512 batches, fp16x2 and bf16.

    python tools/bench_hardnet.py [--steps 20] [--warmup 3] [--batch 64]

Prints one JSON line.  Per precision: images/s over the timed window (CUDA events, after warm-up, inputs rotated over
four resident batches so they do not sit in L2), the achieved TFLOP/s at 31.0 GFLOP per image (the reference's conv
shapes: 4.39 GMAC backbone + 11.11 GMAC heads at 512x512), that rate as a WHOLE-PROGRAM share of the H100 SXM's 989
TFLOP/s dense FP16 data-sheet rate, and the parity of the head maps / decoded rows against tests/golden/hardnet_512.npz
(the unmodified reference on the CPU).  The card's name, power limit and SM clocks are read (nvidia-smi --query-gpu,
read-only) in the same run, before and after the timed windows.  Fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GFLOP_PER_IMG = 31.0
PEAK_FP16_TFLOPS = 989.0
IMG = 512
K_DET = 100


def gpu_info(index: int):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, sm, sm_max = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit_w": float(plim), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}
    except Exception as e:                      # the numbers stay valid, but say that the hardware could not be read
        return {"error": f"nvidia-smi unavailable: {e}"}


def build(dev, precision):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from centerpose_b200.synth import conditioned_state_dict
    cfg = default_cfg("hardnet")
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    m.load_state_dict(conditioned_state_dict(m.state_dict(), 317))
    return m.to(dev).set_precision(precision)


def parity(model, dev):
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.synth import synth_images
    from tests.util import match_rows
    g = np.load(os.path.join(ROOT, "tests", "golden", "hardnet_512.npz"))
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
    ap.add_argument("--precisions", default="fp16x2,bf16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_hardnet.py needs a CUDA device (there is no CPU path to time)")
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.synth import synth_images
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    hw_before = gpu_info(0)
    inputs = [synth_images(B, IMG, IMG, 317 + i).to(dev) for i in range(4)]
    result = {"metric": "images/sec 512x512 HarDNet forward + decode, device-resident batches", "batch": B,
              "steps": args.steps, "warmup": args.warmup, "gflop_per_image": GFLOP_PER_IMG, "precisions": {}}
    for precision in args.precisions.split(","):
        model = build(dev, precision)

        def step(i):
            hm, wh, hps, reg, hm_hp, hp_off = model(inputs[i % len(inputs)])
            return multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_off, K=K_DET, apply_sigmoid=True)

        for i in range(max(args.warmup, 1)):
            step(i)
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            step(i)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        ips = B * args.steps / (ms / 1e3)
        tflops = ips * GFLOP_PER_IMG / 1e3
        plan = next(iter(model._plans.values()))
        result["precisions"][precision] = {
            "images_per_s": ips, "ms_per_step": ms / args.steps, "achieved_tflops": tflops,
            "whole_program_share_of_989_tflops_fp16_dense_datasheet": tflops / PEAK_FP16_TFLOPS,
            "ops": int(plan.n), "convert_ops": int(sum(1 for o in plan.ops if o.type == 11)),
            "parity_vs_hardnet_512_golden": parity(model, dev)}
        del model
        torch.cuda.empty_cache()
    result["gpu_before"] = hw_before
    result["gpu_after"] = gpu_info(0)
    print(json.dumps(result))


if __name__ == "__main__":
    main()

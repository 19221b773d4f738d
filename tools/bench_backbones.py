"""Throughput and parity on one GPU of the backbones bench.py does not take: forward + fused decode of device-resident
512x512 batches, fp16x2 and bf16.

    python tools/bench_backbones.py [--archs hardnet,mobilenetv2,ghostnet] [--steps 20] [--warmup 3] [--batch 64]
                                    [--rounds 3]

Prints one JSON line.  Every (backbone, precision) model is built and warmed up first; then ``--rounds`` rounds each
time every model once, in turn, so that the models alternate and the spread between rounds shows the noise of the
shared host.  Per model: images/s of each round (CUDA events around ``--steps`` steps, inputs rotated over four
resident batches so they do not sit in L2), their range, the program's op and CONVERT-op counts, and the parity of the
head maps / decoded rows against tests/golden/<golden>_512.npz (the unmodified reference on the CPU).  For a backbone
with a known FLOP count per image (GFLOP_PER_IMAGE), also the achieved TFLOP/s of each round and that rate as a
WHOLE-PROGRAM share of the H100 SXM's 989 TFLOP/s dense FP16 data-sheet rate.  The card's name, power limit and SM
clocks are read (nvidia-smi --query-gpu, read-only) before and after the timed rounds.  Fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.util import golden_check, match_rows, model  # noqa: E402

IMG = 512
K_DET = 100
PEAK_FP16_TFLOPS = 989.0
GOLDEN = {"hardnet": "hardnet_512", "mobilenetv2": "mbv2_512", "ghostnet": "ghostnet_512"}
# the reference's conv shapes at 512x512: HarDNet 4.39 GMAC backbone + 11.11 GMAC heads
GFLOP_PER_IMAGE = {"hardnet": 31.0}


def gpu_info(index: int):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, sm, sm_max = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit_w": float(plim), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}
    except Exception as e:                      # the numbers stay valid, but say that the hardware could not be read
        return {"error": f"nvidia-smi unavailable: {e}"}


def parity(m, arch):
    _, mx, rel, rows = golden_check(m, GOLDEN[arch])
    r, e = match_rows(*rows, tol=1e-3, box_tol=2e-2)
    return {"head_maps_rel_l2": float(rel), "head_maps_max_abs_over_max": float(mx),
            "rows_matched": r, "elements_within_1e-3": e,
            "tolerance": "rows matched on bbox + score within 2e-2, then |err| <= 1e-3 * max(1, |ref|) per value"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--archs", default="hardnet,mobilenetv2,ghostnet")
    ap.add_argument("--precisions", default="fp16x2,bf16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_backbones.py needs a CUDA device (there is no CPU path to time)")
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.synth import synth_images
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    inputs = [synth_images(B, IMG, IMG, 317 + i).to(dev) for i in range(4)]
    models = {(a, p): model(a, p)[0] for a in args.archs.split(",") for p in args.precisions.split(",")}

    def step(m, i):
        hm, wh, hps, reg, hm_hp, hp_off = m(inputs[i % len(inputs)])
        return multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_off, K=K_DET, apply_sigmoid=True)

    for m in models.values():
        for i in range(max(args.warmup, 1)):
            step(m, i)
    torch.cuda.synchronize()
    hw_before = gpu_info(0)
    rates = {key: [] for key in models}
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for key, m in models.items():
            e0.record()
            for i in range(args.steps):
                step(m, i)
            e1.record()
            torch.cuda.synchronize()
            rates[key].append(B * args.steps / (e0.elapsed_time(e1) / 1e3))
    hw_after = gpu_info(0)
    result = {"metric": "images/sec 512x512 forward + decode, device-resident batches", "batch": B, "steps": args.steps,
              "warmup": args.warmup, "rounds": args.rounds, "models": {}}
    for (arch, precision), m in models.items():
        plan = next(iter(m._plans.values()))
        r = rates[(arch, precision)]
        entry = {"images_per_s": r, "images_per_s_range": [min(r), max(r)], "ops": int(plan.n),
                 "convert_ops": int(sum(1 for o in plan.ops if o.type == 11))}
        if arch in GFLOP_PER_IMAGE:
            tflops = [ips * GFLOP_PER_IMAGE[arch] / 1e3 for ips in r]
            entry.update({"gflop_per_image": GFLOP_PER_IMAGE[arch], "achieved_tflops": tflops,
                          "whole_program_share_of_989_tflops_fp16_dense_datasheet": [t / PEAK_FP16_TFLOPS for t in tflops]})
        entry["parity_vs_512_golden"] = parity(m, arch)
        result["models"][f"{arch}/{precision}"] = entry
    result["gpu_before"] = hw_before
    result["gpu_after"] = hw_after
    print(json.dumps(result))


if __name__ == "__main__":
    main()

"""Time the training DCNv2 (``centerpose_b200.dcn``) forward, and forward + backward, against
``torchvision.ops.deform_conv2d`` on the same card, on every DCN shape of DLA-34 (B = 32) and MobileNetV3 (B = 64) at
a 512x512 input.

    python tools/bench_dcn_train.py [--steps 10] [--warmup 3] [--rounds 3] [--out FILE]

Arms: the device path at ``precision="default"`` (tf32 split, tensor cores) and ``"fp32"`` (CUDA cores), and
torchvision (skipped, and said so, where torchvision is absent).  Per shape, round and arm: CUDA-event time per call
after a warm-up, through autograd as a training step runs it; rounds alternate the arms.  Also per arm: the rise of
``torch.cuda.max_memory_allocated`` over one forward + backward, and the largest max-normalised difference of the
output and the five gradients from the default arm.  FLOP/s count 2 * B * Co * C * 9 * H * W for the forward and
twice that for the backward (data and weight gradient).  A torch.profiler pass times each kernel of the default arm;
its share of the data-sheet bound is useful FLOPs over kernel time over 495 TFLOP/s (dense TF32, H100 SXM; the split
issues three tf32 MMAs per useful one, so its ceiling is a third of that) or over 67 TFLOP/s (FP32) for the fp32 arm.
The card's name and power limit are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

TF32_PEAK = 495e12
FP32_PEAK = 67e12
DLA34 = [(512, 256, 16, 16), (256, 256, 32, 32), (256, 128, 32, 32), (128, 128, 64, 64), (128, 64, 64, 64),
         (256, 64, 32, 32), (64, 64, 128, 128)]
MOBILENETV3 = [(40, 24, 64, 64), (160, 24, 32, 32), (960, 24, 16, 16), (24, 24, 128, 128), (24, 24, 64, 64),
               (24, 24, 32, 32)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)


def inputs(B, C, Co, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = dict(device="cuda", generator=g)
    stdv = 1.0 / math.sqrt(9 * C)
    return dict(input=torch.randn(B, C, H, W, **d), weight=(torch.rand(Co, C, 3, 3, **d) * 2 - 1) * stdv,
                bias=torch.randn(Co, **d) * 0.1, offset=torch.randn(B, 18, H, W, **d) * 2,
                mask=torch.rand(B, 9, H, W, **d), grad_out=torch.randn(B, Co, H, W, **d))


def arm_fn(arm):
    from centerpose_b200 import dcn
    if arm == "torchvision":
        from torchvision.ops import deform_conv2d
        return lambda x, o, m, w, b: deform_conv2d(x, o, w, b, stride=1, padding=1, dilation=1, mask=m)
    return lambda x, o, m, w, b: dcn.dcn_v2_conv(x, o, m, w, b, 1, 1, 1, 1, arm)


def leaves(t):
    return [t[k].detach().clone().requires_grad_(True) for k in ("input", "offset", "mask", "weight", "bias")]


def run(fn, t, lv, backward):
    if backward:
        for x in lv:
            x.grad = None
        fn(*lv).backward(t["grad_out"])
    else:
        with torch.no_grad():
            fn(*lv)


def timed(fn, t, lv, backward, steps, warmup):
    for _ in range(warmup):
        run(fn, t, lv, backward)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        run(fn, t, lv, backward)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def results(fn, t):
    lv = leaves(t)
    out = fn(*lv)
    out.backward(t["grad_out"])
    return [out.detach()] + [x.grad for x in lv]


def peak_extra(fn, t):
    lv = leaves(t)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    run(fn, t, lv, True)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def kernel_times(fn, t, iters=3):
    """Mean device time per call of each kernel of one forward + backward, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    lv = leaves(t)
    run(fn, t, lv, True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(iters):
            run(fn, t, lv, True)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        k = re.search(r"(dcn_\w+_kernel)(<\d>)?", e.key)
        if e.device_type.name == "CUDA" and k:
            name = k.group(1)
            dur = getattr(e, "device_time_total", None)
            if dur is None:
                dur = e.cuda_time_total
            out[name] = out.get(name, 0.0) + dur / 1e3 / iters
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcn_train: needs a CUDA device")
    arms = ["default", "fp32"]
    try:
        import torchvision.ops  # noqa: F401
        arms.append("torchvision")
        skipped = None
    except ImportError:
        skipped = "torchvision is not installed: its arm is skipped"
    rows = []
    for net, B, shapes in (("dla_34", 32, DLA34), ("mobilenetv3", 64, MOBILENETV3)):
        for (C, Co, H, W) in shapes:
            t = inputs(B, C, Co, H, W, seed=C + Co + H)
            flop_f = 2.0 * B * Co * C * 9 * H * W
            fns = {arm: arm_fn(arm) for arm in arms}
            ref = results(fns["default"], t)
            row = dict(net=net, B=B, C=C, Co=Co, H=H, W=W, gflop_fwd=flop_f / 1e9, gflop_fwd_bwd=3 * flop_f / 1e9,
                       arms={})
            for arm in arms:
                got = results(fns[arm], t)
                agree = max(((g - r).abs().max() / r.abs().max().clamp_min(1e-30)).item() for g, r in zip(got, ref))
                row["arms"][arm] = dict(fwd_ms=[], fwd_bwd_ms=[], peak_extra_mib=peak_extra(fns[arm], t) / 2**20,
                                        max_rel_diff_vs_default=agree)
                del got
            for _ in range(a.rounds):
                for arm in arms:
                    lv = leaves(t)
                    row["arms"][arm]["fwd_ms"].append(timed(fns[arm], t, lv, False, a.steps, a.warmup))
                    row["arms"][arm]["fwd_bwd_ms"].append(timed(fns[arm], t, lv, True, a.steps, a.warmup))
            for arm in arms:
                r = row["arms"][arm]
                r["fwd_tflops"] = flop_f / (min(r["fwd_ms"]) * 1e-3) / 1e12
                r["fwd_bwd_tflops"] = 3 * flop_f / (min(r["fwd_bwd_ms"]) * 1e-3) / 1e12
            kt = {}
            for arm, peak in (("default", TF32_PEAK), ("fp32", FP32_PEAK)):
                ks = kernel_times(fns[arm], t)
                useful = {"dcn_fwd_kernel": flop_f, "dcn_bwd_data_kernel": flop_f, "dcn_bwd_weight_kernel": flop_f}
                kt[arm] = {k: dict(ms=v, share_of_peak=(useful[k] / (v * 1e-3) / peak) if k in useful else None)
                           for k, v in ks.items()}
            row["kernels"] = kt
            rows.append(row)
            print(json.dumps({k: row[k] for k in ("net", "C", "Co", "H", "W")}) + " " +
                  " ".join("%s fwd %.3f fwd+bwd %.3f ms" % (arm, min(row["arms"][arm]["fwd_ms"]),
                                                           min(row["arms"][arm]["fwd_bwd_ms"])) for arm in arms),
                  file=sys.stderr)
            del t, ref
            torch.cuda.empty_cache()
    res = dict(card=card(), torch=torch.__version__, steps=a.steps, warmup=a.warmup, rounds=a.rounds,
               skipped=skipped, shapes=rows)
    line = json.dumps(res)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()

"""Time the bandwidth-bound ops of the DLA-34 program at benchmark size (B = 32, 512x512, fp16x2), each on its own.

Every STEM, MAXPOOL and DWDECONV_ADD op of the plan, and ops 1 and 2 (the 16 -> 16 @ 512^2 and 16 -> 32 stride-2
small-channel convs, the next bandwidth-bound layers), is launched back to back between two CUDA events until the window
is well above 10 ms.  Per op: shape, microseconds per launch, algorithmic bytes from the shapes (every input, skip and
output once; 4 bytes per element on split planes and for the fp32 image), GB/s and the share of the H100 SXM data-sheet
3 350 GB/s.  The card's name, power limit and SM clock are queried in the same call.  Needs a GPU.

    python tools/bench_eltwise.py [--arch dla_34] [--batch 32] [--precision fp16x2] [--min-ms 30]
"""
import argparse
import ctypes
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import _lib                                                   # noqa: E402
from centerpose_b200 import plan as P                                              # noqa: E402

DATA_SHEET_GBS = 3350.0
NAMES = {P.OP_CONV: "conv", P.OP_STEM: "stem", P.OP_MAXPOOL: "maxpool", P.OP_DWDECONV_ADD: "dwdeconv+add"}
CLASS = (P.OP_STEM, P.OP_MAXPOOL, P.OP_DWDECONV_ADD)


def op_bytes(o):
    """algorithmic bytes of one launch: inputs, the skip / residual and the output once, 4 bytes per element"""
    cin = sum(o.cin[j] for j in range(o.nsrc))
    n_out = o.B * o.Ho * o.Wo * o.cout
    extra = n_out if (o.type == P.OP_DWDECONV_ADD and o.aux) or (o.type == P.OP_CONV and o.res) else 0
    return 4 * (o.B * o.H * o.W * cin + n_out + extra)


def time_op(plan, i, min_ms):
    one = ctypes.cast(ctypes.addressof(plan.ops) + i * ctypes.sizeof(P.OpStruct), ctypes.POINTER(P.OpStruct))
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    n = 8
    while True:
        e0.record()
        for _ in range(n):
            _lib.launch("run_ops", plan.device, one, 1)
        e1.record(); e1.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= min_ms:
            return ms / n, n
        n = max(2 * n, int(n * 1.5 * min_ms / max(ms, 1e-3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="dla_34")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--precision", default="fp16x2")
    ap.add_argument("--min-ms", type=float, default=30.0, help="shortest timed window per op")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eltwise: no CUDA device")
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from centerpose_b200.synth import conditioned_state_dict, synth_images
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("card (name, power limit, max SM clock, SM clock now):", q)
    dev = torch.device("cuda:0")
    cfg = default_cfg(a.arch)
    model = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    model.load_state_dict(conditioned_state_dict(model.state_dict(), 317))
    model = model.to(dev).set_precision(a.precision)
    model(synth_images(a.batch, 512, 512, 317).to(dev))
    plan = model._plan(a.batch, 512, 512, dev)
    plan.run()
    torch.cuda.synchronize()
    picked = [i for i in range(plan.n) if plan.ops[i].type in CLASS or (i in (1, 2) and plan.ops[i].type == P.OP_CONV)]
    print(f"{a.arch} [{a.precision}] B={a.batch}, {plan.n} ops; share = GB/s over the data-sheet {DATA_SHEET_GBS:.0f} GB/s (not measured peak)")
    cls_us = cls_b = 0.0
    n_cls = 0
    for i in picked:
        o = plan.ops[i]
        ms, n = time_op(plan, i, a.min_ms)
        by = op_bytes(o)
        gbs = by / ms / 1e6
        cin = sum(o.cin[j] for j in range(o.nsrc))
        in_class = o.type in CLASS
        print(f"op {i:3d} {NAMES[o.type]:13s} {cin:3d}->{o.cout:3d} {o.H}x{o.W}->{o.Ho}x{o.Wo} k{o.kh} s{o.stride}: "
              f"{ms * 1e3:8.1f} us  {by / 1e6:7.1f} MB  {gbs:7.0f} GB/s  {100 * gbs / DATA_SHEET_GBS:5.1f} % of data sheet"
              f"  ({n} launches){'' if in_class else '  [not in the class sum]'}")
        if in_class:
            cls_us += ms * 1e3; cls_b += by; n_cls += 1
    print(f"class sum (stem + max-pool + dwdeconv, {n_cls} ops): {cls_us / 1e3:.3f} ms, {cls_b / 1e9:.2f} GB, "
          f"{cls_b / 1e9 / DATA_SHEET_GBS * 1e3:.3f} ms at the data-sheet rate")


if __name__ == "__main__":
    main()

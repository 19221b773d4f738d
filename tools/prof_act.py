"""Time one 1x1 conv (64 -> 256 @64^2, B=64: MobileNetV3's 40->240 expand conv on padded channels) per activation."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200.plan import PlanBuilder

dev = torch.device("cuda:0")
prec = os.environ.get("PROF_PREC", "fp16x2")
B, ci, co, hw = 64, 64, 256, 64
g = torch.Generator().manual_seed(0)
for act in (None, "relu", "hswish", "hsigmoid"):
    pb = PlanBuilder(B, 512, 512, prec, dev, tc=True)
    adt = torch.float32 if prec in ("fp16x2", "bf16x2") else torch.bfloat16
    xin = torch.randn(B, hw, hw, ci, generator=g).to(dev, adt)
    y = pb.conv([pb.external(xin)], torch.randn(co, ci, 1, 1, generator=g).to(dev) * 0.05, torch.zeros(co, device=dev), act=act)
    plan = pb.build()
    for _ in range(2):
        plan.run()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        plan.run()
    e1.record(); torch.cuda.synchronize()
    print(f"PROFACT [{prec}] act={act}: {e0.elapsed_time(e1) / 5 * 1e3:.1f} us")

"""Run ONE fused op of the DLA-34 program at benchmark size (B=32, 512x512 input) a few times, for
`ncu --set full -k regex:<kernel> -s 2 -c 1 python tools/prof_op.py <op>` captures and quick timing.
ops: dcn64 (64->64 @128^2), dcn128 (128->128 @64^2), head3x3 (64->256 @128^2), conv64 (64->64 @128^2),
     conv256 (256->256 @32^2), om64 (64->27 @128^2), level0 (16->16 @512^2), level1 (16->32 s2), stem, head1x1
     heads: the keypoint-head ops of the whole DLA-34 program (PROF_ARCH overrides the backbone), each timed on its own
            with Plan.profile_ops, with the card's name and power limit"""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200.plan import PlanBuilder

OPS = {
    "dcn64": ("dcn", 64, 64, 128), "dcn128": ("dcn", 128, 128, 64), "dcn256": ("dcn", 256, 256, 32),
    "head3x3": ("conv", 64, 256, 128, 3, 1), "conv64": ("conv", 64, 64, 128, 3, 1), "conv128": ("conv", 128, 128, 64, 3, 1),
    "conv256": ("conv", 256, 256, 32, 3, 1), "conv512": ("conv", 512, 512, 16, 3, 1), "om64": ("conv", 64, 27, 128, 3, 1),
    "level0": ("conv", 16, 16, 512, 3, 1), "level1": ("conv", 16, 32, 512, 3, 2), "root448": ("conv", 448, 128, 64, 1, 1),
    "up64": ("up", 64, 64, 2), "up64x4": ("up", 64, 32, 4), "pool32": ("pool", 32, 256), "head1x1": ("conv", 256, 34, 128, 1, 1), "reshead": ("conv", 256, 64, 128, 3, 1), "res1x1": ("conv", 64, 256, 128, 1, 1), "stem": ("stem",),
}


def heads(B, prec, reps):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from centerpose_b200.synth import conditioned_state_dict, synth_images
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("card:", q)
    dev = torch.device("cuda:0")
    arch = os.environ.get("PROF_ARCH", "dla_34")
    cfg = default_cfg(arch)
    model = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    model.load_state_dict(conditioned_state_dict(model.state_dict(), 317))
    model = model.to(dev).set_precision(prec)
    x = synth_images(B, 512, 512, 317).to(dev)
    model(x)
    plan = model._plan(B, 512, 512, dev)
    prof = plan.profile_ops(torch.cuda.current_stream().cuda_stream, reps=reps)
    # the heads are the program's tail from its first NCHW-output op: the fused HEADS op, or a 1x1 conv whose 3x3 conv
    # comes right before it
    first = min(i for i in range(plan.n) if plan.ops[i].flags & 2)
    first -= plan.ops[first].type == 1
    sums = {}
    for i in range(first, plan.n):
        typ, fl, b_, ho, wo, co, ci, kh, kw, ms = prof[i]
        kind = "1x1 nchw" if fl & 2 else ("type%d %dx%d" % (typ, kh, kw))
        sums[kind] = sums.get(kind, 0.0) + ms
        print(f"op {i:3d} type {typ} {kind:8s} {ci:4d}->{co:4d} @ {ho}x{wo}: {ms * 1e3:8.1f} us")
    for k, v in sums.items():
        print(f"HEADS {arch} [{prec}] B={B}: {k} total {v * 1e3:.1f} us")
    print(f"whole program (sum of per-op times): {sum(p[-1] for p in prof) * 1e3:.1f} us over {plan.n} ops")


def main():
    name = sys.argv[1]
    B = int(os.environ.get("PROF_B", "32"))
    if name == "heads":
        return heads(B, os.environ.get("PROF_PREC", "fp16x2"), int(os.environ.get("PROF_REPS", "5")))
    reps = int(os.environ.get("PROF_REPS", "5"))
    dev = torch.device("cuda:0")
    spec = OPS[name]
    g = torch.Generator().manual_seed(0)
    prec = os.environ.get("PROF_PREC", "bf16")
    split = prec in ("fp16x2", "bf16x2")
    adt = torch.float32 if split else torch.bfloat16          # split precisions: external() takes fp32 and splits it
    pb = PlanBuilder(B, 512, 512, prec, dev, tc=True)
    flops = 0.0
    if spec[0] == "stem":
        x = torch.randn(B, 3, 512, 512, generator=g).to(dev)
        y = pb.stem(pb.input(3), torch.randn(16, 3, 7, 7, generator=g).to(dev) * 0.1, torch.zeros(16, device=dev), 7, 1, 3)
        flops = 2.0 * B * 512 * 512 * 16 * 147
        name = name + ("(tc)" if (pb.ops[0].flags & 8 or len(pb.ops) == 2) else "(simt)")
    elif spec[0] == "up":                        # IDAUp depthwise ConvTranspose2d(k=2f, s=f) + skip add
        _, c, hw, f = spec
        xin = torch.randn(B, hw, hw, c, generator=g).to(dev, adt)
        sk = torch.randn(B, hw * f, hw * f, c, generator=g).to(dev, adt)
        y = pb.up_add(pb.external(xin), pb.external(sk), torch.randn(c, 1, 2 * f, 2 * f, generator=g).to(dev) * 0.2)
        flops = 2.0 * B * (hw * f) ** 2 * c * 4
    elif spec[0] == "pool":
        _, c, hw = spec
        xin = torch.randn(B, hw, hw, c, generator=g).to(dev, adt)
        y = pb.maxpool(pb.external(xin), 2, 2)
        flops = 1.0 * B * (hw // 2) ** 2 * c * 4
    elif spec[0] == "dcn":
        _, ci, co, hw = spec
        xin = torch.randn(B, hw, hw, ci, generator=g).to(dev, adt)
        y = pb.dcn(pb.external(xin), torch.randn(co, ci, 3, 3, generator=g).to(dev) * 0.05, torch.zeros(co, device=dev),
                   torch.randn(27, ci, 3, 3, generator=g).to(dev) * 0.01, torch.randn(27, generator=g).to(dev) * 0.5)
        flops = 2.0 * B * hw * hw * co * ci * 9
    else:
        _, ci, co, hw, k, s = spec
        xin = torch.randn(B, hw, hw, ci, generator=g).to(dev, adt)
        out = "f32" if co == 27 else ("nchw" if co == 34 else "act")
        dst = pb.output(co, hw // s, hw // s, "o") if out == "nchw" else None
        y = pb.conv([pb.external(xin)], torch.randn(co, ci, k, k, generator=g).to(dev) * 0.05, torch.zeros(co, device=dev),
                    stride=s, pad=k // 2, relu=True, out=out, dst=dst)
        flops = 2.0 * B * (hw // s) * (hw // s) * co * ci * k * k
    plan = pb.build()
    outs = {"o": torch.empty(B, 34, 128, 128, device=dev)} if spec[0] == "conv" and spec[2] == 34 else {}
    plan.bind(x if spec[0] == "stem" else torch.zeros(1, device=dev), outs)
    st = torch.cuda.current_stream().cuda_stream
    which = int(os.environ.get("PROF_OP_INDEX", "-1"))     # dcn: 0 = offset conv, 1 = DCN itself
    for _ in range(2):
        plan.run(st)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        plan.run(st)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print(f"PROFOP {name} [{prec}]: {ms * 1e3:.1f} us per plan run ({plan.n} ops), {flops / ms / 1e9:.1f} TFLOP/s on the main op's flops")


if __name__ == "__main__":
    main()

"""Hardware characterisation (GPU): how much does the wgmma fp32 accumulator's round-toward-zero behaviour shrink a
K-long dot product of split operands?  For iid random-sign data the error of the tensor-core result has a component
proportional to the exact result (a coherent shrink factor) — the part that adds up linearly through a deep network.
Prints, per K and operand statistics, the projection coefficient  <got - ref, ref> / <ref, ref>  and the residual.

    python tools/rz_probe.py
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import torch                                                    # noqa: E402
import torch.nn.functional as F                                 # noqa: E402

from centerpose_b200.plan import PlanBuilder                    # noqa: E402

DEV = torch.device("cuda:0")


def one(prec, ci, k, kind, co=128, H=32, W=32, B=2):
    g = torch.Generator().manual_seed(ci * 10 + k)
    x = torch.randn(B, ci, H, W, generator=g)
    if kind == "relu":
        x = F.relu(x)
    elif kind == "pos":
        x = x.abs() + 0.5
    w = torch.randn(co, ci, k, k, generator=g) / (ci * k * k) ** 0.5
    if kind == "pos":
        w = w.abs()
    ref = F.conv2d(x.double(), w.double(), None, padding=k // 2)
    pb = PlanBuilder(B, 1, 1, prec, DEV)
    y = pb.conv([pb.external(x.permute(0, 2, 3, 1).contiguous().to(DEV))], w.to(DEV), torch.zeros(co, device=DEV), pad=k // 2)
    plan = pb.build(); plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
    got = plan.tensor(y).double().permute(0, 3, 1, 2).cpu()
    d = got - ref
    coef = (d * ref).sum().item() / (ref * ref).sum().item()
    resid = (d - coef * ref).norm().item() / ref.norm().item()
    return coef, resid


def main():
    for prec in ("fp16x2", "bf16x2"):
        for kind in ("gauss", "relu", "pos"):
            for ci, k in ((64, 1), (256, 1), (1280, 1), (64, 3), (128, 3), (256, 3), (512, 3)):
                K = ci * k * k
                coef, resid = one(prec, ci, k, kind)
                print(f"{prec} {kind:5s} K={K:5d} ksteps={K // 16:4d}  shrink coef {coef:+.3e}  per kstep {coef / (K / 16):+.3e}  "
                      f"per sqrt(kstep) {coef / (K / 16) ** 0.5:+.3e}  residual relL2 {resid:.3e}")


if __name__ == "__main__":
    main()

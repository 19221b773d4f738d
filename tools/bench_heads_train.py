"""Time the training keypoint heads (``centerpose_b200.heads_train.KeypointHead``) forward, and forward + backward
through autograd, against the reference's ``KeypointHead`` in torch on the same card, at the head shapes of DLA-34
(B = 18), MobileNetV3 (B = 21) and ResNet-50 (B = 14) at R = 128 (a 512x512 input).

    python tools/bench_heads_train.py [--steps 10] [--warmup 3] [--rounds 3] [--out FILE]

Arms: the device heads at ``precision="default"`` (tf32 split, tensor cores) and ``"fp32"`` (CUDA cores); torch's
module (the reference's six Conv2d -> ReLU -> Conv2d sequences) with cuDNN in fp32 (``allow_tf32=False``) and at
torch's default, where cuDNN's convs run TF32.  Per shape, round and arm: CUDA-event time per call after a warm-up;
rounds alternate the arms.  Per arm: the rise of ``torch.cuda.max_memory_allocated`` over one forward + backward, and
the largest max-normalised difference of the six outputs and the input gradient from torch's fp32 arm.  The card's
name and power limit are read in the same run.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SHAPES = {"dla_34": (18, 64, 256), "mobilenetv3": (21, 24, 256), "res_50": (14, 256, 64)}   # (B, C, hc)
R = 128
ARMS = ("default", "fp32", "torch_fp32", "torch_tf32")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)


class TorchHeads(torch.nn.Module):
    """The reference's KeypointHead layers in torch (the same children and parameter names)."""

    def __init__(self, C, hc):
        super().__init__()
        from centerpose_b200.heads_train import HEADS, OUTPUTS
        self.names = HEADS
        for name, c in zip(HEADS, OUTPUTS):
            setattr(self, name, torch.nn.Sequential(torch.nn.Conv2d(C, hc, 3, padding=1), torch.nn.ReLU(inplace=True),
                                                    torch.nn.Conv2d(hc, c, 1)))

    def forward(self, x):
        return [getattr(self, n)(x) for n in self.names]


def make(arch):
    from centerpose_b200 import heads_train
    B, C, hc = SHAPES[arch]
    torch.manual_seed(0)
    mine = heads_train.KeypointHead(C, hc).cuda()
    ref = TorchHeads(C, hc).cuda()
    ref.load_state_dict(mine.state_dict())
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, C, R, R, device="cuda", generator=g).relu_()
    gos = [torch.randn(B, c, R, R, device="cuda", generator=g) for c in heads_train.OUTPUTS]
    return mine, ref, x, gos


def call(arm, mine, ref, x, gos, backward):
    m = ref if arm.startswith("torch") else mine
    if arm in ("default", "fp32"):
        mine.precision = arm
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=(arm == "torch_tf32")):
        if not backward:
            with torch.no_grad():
                return m(x)
        xl = x.detach().requires_grad_(True)
        for p in m.parameters():
            p.grad = None
        outs = m(xl)
        torch.autograd.backward(outs, gos)
        return [o.detach() for o in outs] + [xl.grad]


def timed(arm, mine, ref, x, gos, backward, steps, warmup):
    for _ in range(warmup):
        call(arm, mine, ref, x, gos, backward)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        call(arm, mine, ref, x, gos, backward)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def peak_rise(arm, mine, ref, x, gos):
    torch.cuda.synchronize()
    for m in (mine, ref):
        for p in m.parameters():
            p.grad = None
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    res = call(arm, mine, ref, x, gos, True)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    del res
    return rise


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_heads_train: no CUDA device; nothing is measured")
    result = {"card": card(), "R": R, "shapes": {}}
    for arch in SHAPES:
        mine, ref, x, gos = make(arch)
        want = call("torch_fp32", mine, ref, x, gos, True)
        entry = {"B_C_hc": SHAPES[arch], "arms": {}}
        for arm in ARMS:
            got = call(arm, mine, ref, x, gos, True)
            diff = max(((g - w).abs().max() / w.abs().max().clamp_min(1e-30)).item() for g, w in zip(got, want))
            entry["arms"][arm] = {"fwd_ms": [], "step_ms": [], "max_rel_diff_vs_torch_fp32": diff,
                                  "peak_rise_MiB": peak_rise(arm, mine, ref, x, gos) / 2 ** 20}
            del got
        for _ in range(a.rounds):
            for arm in ARMS:
                e = entry["arms"][arm]
                e["fwd_ms"].append(timed(arm, mine, ref, x, gos, False, a.steps, a.warmup))
                e["step_ms"].append(timed(arm, mine, ref, x, gos, True, a.steps, a.warmup))
        for e in entry["arms"].values():
            e["fwd_ms_min"], e["step_ms_min"] = min(e["fwd_ms"]), min(e["step_ms"])
        result["shapes"][arch] = entry
        for arm, e in entry["arms"].items():
            print("%s %s: forward %.2f ms, forward + backward %.2f ms, peak rise %.0f MiB, max rel diff %.2g"
                  % (arch, arm, e["fwd_ms_min"], e["step_ms_min"], e["peak_rise_MiB"],
                     e["max_rel_diff_vs_torch_fp32"]), file=sys.stderr)
        del mine, ref, x, gos, want
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

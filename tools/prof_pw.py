"""Per-op table of the pointwise convs (1x1 / stride 1 / pad 0, NHWC output) on the tap-per-stage kernel's 1 x 128 pixel
tiles against the same ops on its 2-D tiles (csrc/net_tc.cu).

    python tools/prof_pw.py [--arch dla_34] [--precision fp16x2] [--batch 32] [--reps 20] [--json out.json]

Builds the program twice in one process, once with CPB200_NO_PW=1 (2-D tiles for every op) and once without,
checks that the two programs' outputs are bit-identical, then times every CONV op with a 1x1 filter and an NHWC output
on its own: ``--reps`` back-to-back launches between CUDA events, best of five windows.  GB/s are algorithmic bytes
(each input, residual and the weights read once, the output written once; split planes = 4 bytes per element, bf16 =
2, fp32 = 4) over that time.  Prints the card's name, power limit and SM clock beside the numbers."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import _lib  # noqa: E402
from centerpose_b200.plan import FLAG_TC, OP_CONV, OpStruct  # noqa: E402

FLAG_NCHW = 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def op_bytes(o):
    es = 2 if o.act_dtype == 1 else 4                       # bf16 = 2; fp32 and the split planes = 4
    cin = sum(o.cin[j] for j in range(o.nsrc))
    px = o.B * o.Ho * o.Wo
    out_es = 4 if o.flags & 4 else es
    wr = px * o.cout * out_es
    return px * cin * es + wr + (wr if o.res else 0) + o.cout * cin * es


def time_op(plan, i, stream, reps):
    L = _lib.lib()
    one = ctypes.cast(ctypes.addressof(plan.ops) + i * ctypes.sizeof(OpStruct), ctypes.POINTER(OpStruct))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = None
    for _ in range(5):
        e0.record()
        for _ in range(reps):
            _lib.check(L.cpb200_run_ops(one, 1, stream), "cpb200_run_ops")
        e1.record(); e1.synchronize()
        t = e0.elapsed_time(e1) / reps
        best = t if best is None or t < best else best
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="dla_34")
    ap.add_argument("--precision", default="fp16x2")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from centerpose_b200.synth import conditioned_state_dict, synth_images

    dev = torch.device("cuda:0")
    cfg = default_cfg(args.arch)
    B, S = args.batch, args.size
    x = synth_images(B, S, S, 317).to(dev)
    plans, outs = {}, {}
    for layout in ("2d", "pw"):
        if layout == "2d":
            os.environ["CPB200_NO_PW"] = "1"
        else:
            os.environ.pop("CPB200_NO_PW", None)
        model = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
        model.load_state_dict(conditioned_state_dict(model.state_dict(), 317))
        model = model.to(dev).set_precision(args.precision)
        with torch.no_grad():
            outs[layout] = [t.clone() for t in model(x)]        # prepares the program in this layout
        plans[layout] = (model, model._plan(B, S, S, dev))
    same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(outs["2d"], outs["pw"]))
    stream = torch.cuda.current_stream().cuda_stream
    plan_2d, plan_p = plans["2d"][1], plans["pw"][1]
    rows = []
    for i in range(plan_2d.n):
        o = plan_2d.ops[i]
        if o.type != OP_CONV or o.kh != 1 or o.kw != 1 or o.flags & FLAG_NCHW or not o.flags & FLAG_TC:
            continue
        t_2d = time_op(plan_2d, i, stream, args.reps)
        t_pw = time_op(plan_p, i, stream, args.reps)
        nb = op_bytes(o)
        cins = [o.cin[j] for j in range(o.nsrc)]
        rows.append({"op": i, "cin": cins, "cout": o.cout, "H": o.Ho, "W": o.Wo, "res": bool(o.res), "bytes": nb,
                     "us_2d": t_2d * 1e3, "pw_us": t_pw * 1e3,
                     "gbs_2d": nb / (t_2d * 1e-3) / 1e9, "pw_gbs": nb / (t_pw * 1e-3) / 1e9})
    info = card()
    print(f"card: {info}")
    print(f"{args.arch} [{args.precision}] B={B} {S}x{S}: outputs bit-identical between the tile layouts: {same}")
    print(f"{'op':>4} {'inputs -> cout @ map':34s} {'MB':>7} {'2-D us':>8} {'GB/s':>6} {'PW us':>8} {'GB/s':>6}")
    for r in rows:
        shape = f"{r['cin']} -> {r['cout']} @ {r['H']}x{r['W']}" + (" +res" if r["res"] else "")
        print(f"{r['op']:4d} {shape:34s} {r['bytes'] / 1e6:7.1f} {r['us_2d']:8.1f} {r['gbs_2d']:6.0f} {r['pw_us']:8.1f} "
              f"{r['pw_gbs']:6.0f}")
    tb = sum(r["bytes"] for r in rows)
    tt, tp = sum(r["us_2d"] for r in rows), sum(r["pw_us"] for r in rows)
    print(f"sum  {len(rows)} ops {'':24s} {tb / 1e6:7.1f} {tt:8.1f} {tb / tt / 1e3:6.0f} {tp:8.1f} {tb / tp / 1e3:6.0f}")
    print(f"card after timing: {card()}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "identical": same, "rows": rows}, f, indent=1)
    if not same:
        sys.exit("the pointwise and 2-D tile layouts disagree")


if __name__ == "__main__":
    main()

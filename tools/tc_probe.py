"""Diagnostic probe of the wgmma conv path: integer-valued inputs/weights and fp32 output, so
every result is exactly representable and any mismatch is a real defect (layout, descriptor,
pipeline).  Each case runs in a subprocess with a timeout so that a hung kernel cannot take the
whole GPU call down.  Usage: python tools/tc_probe.py [case_index]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [
    # name, cins, cout, k, stride, H, W, B, weights
    ("1x1_c64_identity_onetile", [64], 64, 1, 1, 8, 16, 1, "identity"),
    ("1x1_c64_rand_onetile", [64], 64, 1, 1, 8, 16, 1, "rand"),
    ("1x1_c16_rand", [16], 16, 1, 1, 8, 16, 1, "rand"),
    ("1x1_c32_rand", [32], 32, 1, 1, 8, 16, 1, "rand"),
    ("1x1_c128_rand_k2blocks", [128], 64, 1, 1, 8, 16, 1, "rand"),
    ("3x3_c64_onetile", [64], 64, 3, 1, 8, 16, 1, "rand"),
    ("3x3_c64_multi_tile", [64], 64, 3, 1, 24, 40, 2, "rand"),
    ("3x3_c16_s2", [16], 32, 3, 2, 32, 32, 1, "rand"),
    ("3x3_c64_s2", [64], 128, 3, 2, 32, 64, 2, "rand"),
    ("1x1_concat4", [128, 128, 64, 128], 128, 1, 1, 16, 16, 2, "rand"),
    ("3x3_cout256", [64], 256, 3, 1, 16, 16, 2, "rand"),
    ("3x3_cout512_two_ntiles", [128], 512, 3, 1, 16, 16, 1, "rand"),
    ("3x3_cout27", [64], 27, 3, 1, 16, 16, 1, "rand"),
    ("w8_tiles", [256], 256, 3, 1, 8, 8, 4, "rand"),
    ("persistent_many_tiles", [64], 64, 3, 1, 128, 128, 12, "rand"),
    ("7x7_c16", [16], 16, 7, 1, 16, 32, 1, "rand"),
    ("3x3_c16_s1_halo_sw32", [16], 16, 3, 1, 32, 32, 2, "rand"),
    ("3x3_c32_s1_halo_sw64", [32], 64, 3, 1, 32, 24, 2, "rand"),
    ("3x3_c128_c64_halo_ring", [128], 64, 3, 1, 32, 32, 2, "rand"),
    ("3x3_c128_c128_halo", [128], 128, 3, 1, 40, 24, 2, "rand"),
    ("3x3_c512_c512_halo", [512], 512, 3, 1, 16, 16, 2, "rand"),
    ("3x3_c64_odd_size_halo", [64], 64, 3, 1, 19, 13, 3, "rand"),
]


def run_case(i):
    import torch
    import torch.nn.functional as F
    from centerpose_b200.plan import PlanBuilder
    name, cins, cout, k, stride, H, W, B, wkind = CASES[i]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(i + 1)
    xs = [torch.randint(-4, 5, (B, c, H, W), generator=g).float() for c in cins]
    ci = sum(cins)
    if wkind == "identity":
        w = torch.zeros(cout, ci, k, k)
        for c in range(min(cout, ci)):
            w[c, c, k // 2, k // 2] = 1.0
    else:
        w = torch.randint(-2, 3, (cout, ci, k, k), generator=g).float()
    b = torch.randint(-3, 4, (cout,), generator=g).float()
    pad = k // 2
    ref = F.conv2d(torch.cat(xs, 1), w, b, stride=stride, padding=pad)
    pb = PlanBuilder(B, 1, 1, "bf16", dev, tc=True)
    sx = [pb.external(x.permute(0, 2, 3, 1).contiguous().to(dev, torch.bfloat16)) for x in xs]
    y = pb.conv(sx, w.to(dev), b.to(dev), stride=stride, pad=pad, relu=False, out="f32")
    assert pb.ops[-1].flags & 8
    plan = pb.build()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = plan.tensor(y).float().permute(0, 3, 1, 2).cpu()
    diff = (got - ref).abs()
    res = {"case": name, "max_err": float(diff.max()), "ref_max": float(ref.abs().max()),
           "bad_frac": float((diff > 0).float().mean())}
    if diff.max() > 0:
        bad = (diff > 0)
        res["bad_by_channel"] = [int(v) for v in bad.sum(dim=(0, 2, 3))[:32].tolist()]
        res["bad_by_row"] = [int(v) for v in bad.sum(dim=(0, 1, 3))[:32].tolist()]
        res["bad_by_col"] = [int(v) for v in bad.sum(dim=(0, 1, 2))[:32].tolist()]
        idx = bad.nonzero()[:6].tolist()
        res["samples"] = [(ix, float(got[tuple(ix)]), float(ref[tuple(ix)])) for ix in idx]
        # is `got` a pixel/channel permutation of ref?  (sorted values equal)
        res["same_multiset"] = bool(torch.equal(got.flatten().sort().values, ref.flatten().sort().values))
        res["got_all_zero"] = bool((got == 0).all())
    print("PROBE " + json.dumps(res), flush=True)


def main():
    if len(sys.argv) > 1:
        return run_case(int(sys.argv[1]))
    for i, c in enumerate(CASES):
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), str(i)], capture_output=True, text=True, timeout=90)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("PROBE ")]
            if lines:
                print(lines[-1])
            else:
                print("PROBE " + json.dumps({"case": c[0], "error": (r.stderr or r.stdout)[-600:]}))
        except subprocess.TimeoutExpired:
            print("PROBE " + json.dumps({"case": c[0], "error": "TIMEOUT (kernel hang?)"}))
        sys.stdout.flush()


if __name__ == "__main__":
    main()

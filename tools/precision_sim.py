"""CPU emulation of the split-operand tensor-core arithmetic (design aid, not product / not a test).

Runs the oracle's DLA-34 forward with every conv / DCN GEMM replaced by the arithmetic a split-precision
wgmma path would perform — operands decomposed into 16-bit planes, the cross products accumulated in fp32 —
and reports the head-map error and the decoded-row agreement against the reference golden (dla34_512.npz).

    python tools/precision_sim.py [mode ...]     modes: fp32 bf16 bf16x2 fp16x2 bf16x3
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from oracle import dla_ref, dcn_ref, decode_ref            # noqa: E402
from oracle.init_recipe import conditioned_state_dict, synth_images   # noqa: E402
from tests.util import match_rows                          # noqa: E402

AMAX = 0.0
_conv2d = F.conv2d
_matmul = torch.matmul


def split(x, dt, n):
    parts = []
    r = x
    for _ in range(n):
        p = r.to(dt).float()
        parts.append(p)
        r = r - p
    return parts


def make_ops(mode):
    if mode == "fp32":
        return _conv2d, _matmul
    dt = torch.bfloat16 if mode.startswith("bf16") else torch.float16
    n = int(mode.split("x")[1][0]) if "x" in mode else 1
    wscale = mode.endswith("s")          # fp16x2s: weights pre-scaled by a power of two so max|w| lands in [2^12, 2^13)

    def wsplit(w):
        if not wscale:
            return split(w, dt, n), 1.0
        e = torch.floor(torch.log2(w.abs().max().clamp_min(1e-30)))
        sc = float(2.0 ** (12 - e))
        return split(w * sc, dt, n), 1.0 / sc
    # products kept: all (i, j) with i + j < n  (x2: hh, hl, lh;  x3: hh, hm, mh, hl, mm, lh)
    def conv(x, w, b=None, stride=1, padding=0, **kw):
        xs = split(x, dt, n); ws, inv = wsplit(w)
        out = None
        for i in range(n):
            for j in range(n - i):
                t = _conv2d(xs[i], ws[j], None, stride=stride, padding=padding, **kw)
                out = t if out is None else out + t
        out = out * inv
        global AMAX
        AMAX = max(AMAX, float(x.abs().max()))
        if b is not None:
            out = out + b.view(1, -1, 1, 1)
        return out

    def mm(a, b):
        (as_, inv), bs = wsplit(a), split(b, dt, n)
        out = None
        for i in range(n):
            for j in range(n - i):
                t = _matmul(as_[i], bs[j])
                out = t if out is None else out + t
        return out * inv
    return conv, mm


class _FProxy:
    def __init__(self, conv):
        self._conv = conv

    def __getattr__(self, k):
        if k == "conv2d":
            return self._conv
        return getattr(F, k)


class _TProxy:
    def __init__(self, mm):
        self._mm = mm

    def __getattr__(self, k):
        if k == "matmul":
            return self._mm
        return getattr(torch, k)


def run(mode, sd, x):
    conv, mm = make_ops(mode)
    dla_ref.F = _FProxy(conv); dcn_ref.F = _FProxy(conv); dcn_ref.torch = _TProxy(mm)
    try:
        return dla_ref.forward(sd, x)
    finally:
        dla_ref.F = F; dcn_ref.F = F; dcn_ref.torch = torch


def main():
    modes = sys.argv[1:] or ["fp32", "bf16x2", "fp16x2"]
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    cfg = default_cfg("dla_34")
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    sd = conditioned_state_dict(m.state_dict(), 317)
    x = synth_images(1, 512, 512, 317)
    g = np.load(os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "dla34_512.npz"))
    torch.set_num_threads(os.cpu_count())
    with torch.no_grad():
        ref64 = None
        for mode in modes:
            outs = run(mode, sd, x)
            maps = torch.cat(outs, 1).numpy()
            sub = maps[:, :, ::4, ::4]
            rel = np.linalg.norm(sub - g["maps"]) / np.linalg.norm(g["maps"])
            mx = np.abs(sub - g["maps"]).max() / np.abs(g["maps"]).max()
            hm, wh, hps, reg, hm_hp, hp_off = [o.numpy() for o in outs]
            sig = lambda a: 1.0 / (1.0 + np.exp(-a.astype(np.float32)))
            dets = decode_ref.multi_pose_decode(sig(hm).astype(np.float32), wh, hps, reg, sig(hm_hp).astype(np.float32), hp_off, K=100)
            rows, elems = match_rows(dets[0], g["dets"][0], tol=1e-3, box_tol=2e-2)
            # per-head max abs error on the subsampled maps
            names = [("hm", 1), ("wh", 2), ("hps", 34), ("reg", 2), ("hm_hp", 17), ("hp_offset", 2)]
            o = 0; per = []
            for nme, c in names:
                per.append(f"{nme}:{np.abs(sub[:, o:o + c] - g['maps'][:, o:o + c]).max():.2e}")
                o += c
            # exact-position rows
            d = np.abs(dets[0] - g["dets"][0])
            same_rows = (d.max(axis=1) <= 1e-3).mean()
            print(f"{mode:8s} relL2 {rel:.3e}  max/max {mx:.3e}  rows matched {rows:.3f} elems<=1e-3 {elems:.4f}  "
                  f"rows identical(1e-3, same index) {same_rows:.3f}  | " + " ".join(per) + f" amax {AMAX:.1f}", flush=True)


if __name__ == "__main__":
    main()

"""Generate ``tests/golden/dcn_train.npz``: the DCNv2 forward and its five gradients on small constructed cases.

Run:  python -m oracle.make_golden_dcn_train      (from the repo root)

The reference's own backward (``DCNv2/src/cuda/dcn_v2_cuda.cu:206-330``) cannot be built anywhere: its CUDA sources
use the THC API that torch removed and its CPU entry point is ``AT_ERROR``.  So the values are those of the literal
float64 restatements, ``oracle.dcn_train_ref.dcn_v2_backward_loops`` and ``oracle.dcn_ref.dcn_v2_forward_loops``.
Before anything is written, the literal form is checked against the vectorised one (float64 autograd through
``dcn_v2_forward``) and against torchvision's CPU ``deform_conv2d`` forward and backward in float64, on every case
(grad_offset apart from the taps whose sample sits exactly at -1, where torchvision's coordinate weight skips the
reference's range test).
Where the reference tree is mounted, the product's ``dcn.DCN`` is also checked against the reference's ``dcn_v2.py``
``DCN`` module: parameter names, shapes and, from the same seed, the same initial values (constructing the module
never calls ``_ext``).

The cases (all 3x3 / stride 1 / pad 1, float32 inputs, dyadic where a sample position is constructed):
  edges     samples at exactly -1, inside (-1, 0), at integers, at H-1, inside (H-1, H), exactly at H, and far outside;
            negative fractions where (int) truncation and floor differ; some masks exactly 0
  pile      every sample of every tap lands on the same few input pixels
  one       1x1 maps
  random    seeded normal offsets on a 5x7 map, two images
Per case ``<name>/``: input, weight, bias, offset, mask, grad_out (float32) and out, grad_input, grad_offset,
grad_mask, grad_weight, grad_bias (float64).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import dcn_ref, dcn_train_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "dcn_train.npz")
NAMES = ("edges", "pile", "one", "random")
GRADS = ("grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias")


def _targets(n):
    """Constructed sample coordinates along an axis of length n."""
    return np.array([-1.0, -0.75, -0.5, -0.125, 0.0, 1.0, 1.25, n - 1, n - 0.5, n - 0.0625, n, n + 4.5, -6.25, 2.5,
                     -1.0625, 0.5], np.float64)


def _base(H, W):
    """(9, H, W) integer sample positions of the taps before the offset: ho - 1 + i, wo - 1 + j."""
    i, j = np.divmod(np.arange(9), 3)
    hb = np.arange(H)[None, :, None] - 1 + i[:, None, None]
    wb = np.arange(W)[None, None, :] - 1 + j[:, None, None]
    return np.broadcast_to(hb, (9, H, W)), np.broadcast_to(wb, (9, H, W))


def make_case(name):
    rng = np.random.default_rng({"edges": 11, "pile": 12, "one": 13, "random": 14}[name])
    B, C, Co, H, W = {"edges": (1, 3, 2, 4, 5), "pile": (1, 2, 3, 5, 4), "one": (2, 3, 2, 1, 1),
                      "random": (2, 4, 3, 5, 7)}[name]
    hb, wb = _base(H, W)
    offset = np.zeros((B, 18, H, W))
    if name == "edges":
        th, tw = _targets(H), _targets(W)
        t = np.arange(B * 9 * H * W).reshape(B, 9, H, W)
        offset[:, 0::2] = th[t % len(th)] - hb
        offset[:, 1::2] = tw[(7 * t + 3) % len(tw)] - wb
    elif name == "pile":
        t = np.arange(B * 9 * H * W).reshape(B, 9, H, W)
        spots = np.array([[1.25, 2.5], [2.0, 1.0], [1.25, 2.5], [2.0, 1.5]])
        offset[:, 0::2] = spots[t % 4, 0] - hb
        offset[:, 1::2] = spots[t % 4, 1] - wb
    elif name == "one":
        offset = np.round(rng.normal(0, 0.75, offset.shape) * 16) / 16
    else:
        offset = rng.normal(0, 1.5, offset.shape)
    mask = rng.uniform(0, 1, (B, 9, H, W))
    if name == "edges":
        mask.reshape(-1)[::5] = 0.0
    f32 = lambda a: np.asarray(a, np.float32)
    return dict(input=f32(rng.normal(0, 1, (B, C, H, W))), weight=f32(rng.uniform(-0.5, 0.5, (Co, C, 3, 3))),
                bias=f32(rng.normal(0, 1, Co)), offset=f32(offset), mask=f32(mask),
                grad_out=f32(rng.normal(0, 1, (B, Co, H, W))))


def literal(c):
    out = dcn_ref.dcn_v2_forward_loops(c["input"], c["weight"], c["bias"], c["offset"], c["mask"])
    grads = dcn_train_ref.dcn_v2_backward_loops(c["input"], c["weight"], c["bias"], c["offset"], c["mask"],
                                                c["grad_out"])
    return dict(out=out, **dict(zip(GRADS, grads)))


def vectorised(c):
    t = {k: torch.from_numpy(v.astype(np.float64)) for k, v in c.items()}
    out = dcn_ref.dcn_v2_forward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"])
    grads = dcn_train_ref.dcn_v2_backward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], t["grad_out"])
    return dict(out=out.numpy(), **{k: g.numpy() for k, g in zip(GRADS, grads)})


def torchvision_f64(c):
    from torchvision.ops import deform_conv2d
    t = {k: torch.from_numpy(v.astype(np.float64)) for k, v in c.items()}
    leaves = [t[k].clone().requires_grad_(True) for k in ("input", "offset", "mask", "weight", "bias")]
    x, o, m, w, b = leaves
    out = deform_conv2d(x, o, w, b, stride=1, padding=1, dilation=1, mask=m)
    gi, go, gm, gw, gb = torch.autograd.grad(out, leaves, t["grad_out"])
    return dict(out=out.detach().numpy(), grad_input=gi.numpy(), grad_offset=go.numpy(), grad_mask=gm.numpy(),
                grad_weight=gw.numpy(), grad_bias=gb.numpy())


def on_minus_one(c):
    """(B, 18, H, W) bool: offset entries of taps whose sample sits exactly at -1 on either axis.  There torchvision's
    coordinate weight ignores the reference's ``<= -1`` range test (dcn_v2_im2col_cuda.cu:86) and sees the corner at
    0, so only there its grad_offset differs from the reference's 0."""
    B, _, H, W = c["offset"].shape
    hb, wb = _base(H, W)
    o = c["offset"].astype(np.float64)
    edge = ((hb + o[:, 0::2]) == -1) | ((wb + o[:, 1::2]) == -1)
    return np.repeat(edge, 2, axis=1)


def check_close(what, got, want, rtol=1e-12, skip=None):
    for k, v in want.items():
        scale = max(1.0, float(np.abs(v).max()))
        d = np.abs(np.asarray(got[k]) - v)
        if skip is not None and k in skip:
            d = np.where(skip[k], 0.0, d)
        err = float(d.max())
        if err > rtol * scale:
            raise AssertionError("%s: %s differs by %.3g (scale %.3g)" % (what, k, err, scale))


def check_reference_module():
    """The product's DCN against the unmodified reference's dcn_v2.py DCN: names, shapes and seeded init."""
    from oracle import ref_harness
    if not ref_harness.reference_available():
        print("reference absent: module structure not checked")
        return
    ref_harness.load_reference()
    from models.backbones.DCNv2.dcn_v2 import DCN as RefDCN
    from centerpose_b200 import dcn
    for ci, co in ((64, 64), (40, 24), (960, 24)):
        torch.manual_seed(7)
        ref = RefDCN(ci, co, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
        torch.manual_seed(7)
        mine = dcn.DCN(ci, co, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
        rs, ms = ref.state_dict(), mine.state_dict()
        assert list(rs) == list(ms), (list(rs), list(ms))
        for k in rs:
            assert rs[k].shape == ms[k].shape and torch.equal(rs[k], ms[k]), k
        mine.load_state_dict(rs)
    print("reference DCN module: names, shapes and seeded init match for (64,64), (40,24), (960,24)")


def main():
    check_reference_module()
    arrays = {}
    for name in NAMES:
        c = make_case(name)
        lit = literal(c)
        check_close(name + " vectorised", vectorised(c), lit)
        check_close(name + " torchvision", torchvision_f64(c), lit, skip={"grad_offset": on_minus_one(c)})
        for k, v in c.items():
            arrays[name + "/" + k] = v
        for k, v in lit.items():
            arrays[name + "/" + k] = np.asarray(v, np.float64)
        print(name, {k: float(np.abs(v).max()) for k, v in lit.items()})
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

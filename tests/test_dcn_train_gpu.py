"""GPU tests of the training DCNv2 (centerpose_b200.dcn, csrc/dcn_train.cu) against float64 autograd through the
restatement (oracle/dcn_ref.py, oracle/dcn_train_ref.py) on the device, and against tests/golden/dcn_train.npz.

Accuracy: for the output and each of the five gradients, max|dev - f64| / max|f64| and the relative L2 error must be
at most max(4 * e32, 1e-6), where e32 is the same statistic of torch's fp32 autograd through the same restatement.
"""
import math
import os

import numpy as np
import pytest
import torch
from torch import nn

from centerpose_b200 import dcn
from oracle import dcn_ref, dcn_train_ref

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dcn_train.npz")
NAMES = ("out", "grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias")
PRECISIONS = ("default", "fp32")

# (C, Co, H, W): every DCN of DLA-34 and MobileNetV3 at its map size for a 512x512 input, then odd shapes
DLA34 = [(512, 256, 16, 16), (256, 256, 32, 32), (256, 128, 32, 32), (128, 128, 64, 64), (128, 64, 64, 64),
         (256, 64, 32, 32), (64, 64, 128, 128)]
MOBILENETV3 = [(40, 24, 64, 64), (160, 24, 32, 32), (960, 24, 16, 16), (24, 24, 128, 128), (24, 24, 64, 64),
               (24, 24, 32, 32)]
ODD = [(8, 8, 7, 13), (8, 8, 1, 1), (64, 8, 7, 13), (8, 64, 13, 7), (3, 5, 2, 3), (24, 24, 1, 9)]
CFG = (3, 3, 1, 1, 1, 1, 1, 1, 1)


def make_inputs(B, C, Co, H, W, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    stdv = 1.0 / math.sqrt(9 * C)
    t = dict(input=torch.randn(B, C, H, W, generator=g), weight=(torch.rand(Co, C, 3, 3, generator=g) * 2 - 1) * stdv,
             bias=torch.randn(Co, generator=g) * 0.1, offset=torch.randn(B, 18, H, W, generator=g) * 2,
             mask=torch.rand(B, 9, H, W, generator=g), grad_out=torch.randn(B, Co, H, W, generator=g))
    return {k: v.to(DEV) for k, v in t.items()}


def restated(t, dtype):
    c = {k: v.to(dtype) for k, v in t.items()}
    out = dcn_ref.dcn_v2_forward(c["input"], c["weight"], c["bias"], c["offset"], c["mask"])
    grads = dcn_train_ref.dcn_v2_backward(c["input"], c["weight"], c["bias"], c["offset"], c["mask"], c["grad_out"])
    return [out.detach()] + [g.detach() for g in grads]


def device(t, precision):
    out = dcn.dcn_v2_forward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], *CFG, precision=precision)
    grads = dcn.dcn_v2_backward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], t["grad_out"], *CFG,
                                precision=precision)
    return [out] + list(grads)


def stats(got, want):
    d = (got.double() - want).abs()
    mx = want.abs().max().item()
    l2 = want.norm().item()
    return (d.max().item() / mx if mx > 0 else d.max().item(),
            (d.norm().item() / l2) if l2 > 0 else d.norm().item())


def check_accuracy(got, ref64, ref32, label):
    bad = []
    for name, g, r, r32 in zip(NAMES, got, ref64, ref32):
        assert g.shape == r.shape and g.dtype == torch.float32, name
        assert torch.isfinite(g).all(), "%s %s: not finite" % (label, name)
        e_dev, e32 = stats(g, r), stats(r32, r)
        for what, a, b in zip(("max", "l2"), e_dev, e32):
            if a > max(4 * b, 1e-6):
                bad.append("%s %s %s: %.3g > max(4 * %.3g, 1e-6)" % (label, name, what, a, b))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("shape", DLA34 + MOBILENETV3 + ODD, ids=lambda s: "%dx%d_%dx%d" % s)
def test_accuracy(shape):
    C, Co, H, W = shape
    t = make_inputs(2, C, Co, H, W, seed=C * 7919 + Co * 31 + H)
    ref64 = restated(t, torch.float64)
    ref32 = restated(t, torch.float32)
    for p in PRECISIONS:
        check_accuracy(device(t, p), ref64, ref32, "%s %s" % (shape, p))


@pytest.mark.parametrize("case", ("edges", "pile", "one", "random"))
def test_golden(case):
    z = np.load(GOLD)
    t = {k: torch.from_numpy(z[case + "/" + k]).to(DEV) for k in ("input", "weight", "bias", "offset", "mask",
                                                                 "grad_out")}
    ref64 = [torch.from_numpy(z[case + "/" + n]).to(DEV) for n in NAMES]
    ref32 = restated(t, torch.float32)
    for p in PRECISIONS:
        check_accuracy(device(t, p), ref64, ref32, "%s %s" % (case, p))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_scaling_is_exact(precision):
    t = make_inputs(2, 64, 64, 24, 20, seed=5)
    base = device(t, precision)
    for k in (-30, -10, 10):
        s = 2.0 ** k
        ts = dict(t, grad_out=t["grad_out"] * s)
        got = device(ts, precision)
        for name, a, b in zip(NAMES[2:], got[2:], base[2:]):
            assert torch.equal(a, b * s), "grad_output * 2^%d: %s is not scaled exactly" % (k, name)
        gi, gi0 = got[1] / s, base[1]
        assert (gi - gi0).abs().max().item() <= 1e-6 * gi0.abs().max().item(), "grad_input * 2^%d" % k
        tf = dict(t, input=t["input"] * s, bias=t["bias"] * s)
        out = dcn.dcn_v2_forward(tf["input"], tf["weight"], tf["bias"], tf["offset"], tf["mask"], *CFG,
                                 precision=precision)
        assert torch.equal(out, base[0] * s), "input, bias * 2^%d: output is not scaled exactly" % k


def test_small_magnitudes_keep_their_precision():
    """Gradients of 1e-9 reaching a neck: the tensor-core split keeps fp32's relative precision."""
    t = make_inputs(2, 64, 64, 16, 16, seed=9)
    t["grad_out"] = t["grad_out"] * 1e-9
    ref64 = restated(t, torch.float64)
    ref32 = restated(t, torch.float32)
    check_accuracy(device(t, "default"), ref64, ref32, "grad_output 1e-9")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_deterministic(precision):
    t = make_inputs(2, 128, 64, 33, 29, seed=3)
    a, b = device(t, precision), device(t, precision)
    for name, x, y in zip(NAMES, a, b):
        if name != "grad_input":
            assert torch.equal(x, y), name


def test_memory():
    """Forward + backward at B = 8, 64 -> 64 on 128x128 maps allocate less than one image's column matrix beyond the
    inputs, the output and the gradients."""
    B, C, Co, H, W = 8, 64, 64, 128, 128
    t = make_inputs(B, C, Co, H, W, seed=1)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    res = device(t, "default")
    torch.cuda.synchronize()
    kept = sum(r.numel() * r.element_size() for r in res)
    extra = torch.cuda.max_memory_allocated(DEV) - base - kept
    column = C * 9 * H * W * 4
    assert extra < column, "extra allocation %d bytes >= one image's column matrix %d" % (extra, column)


def test_autograd_noncontiguous_grad_and_retain_graph():
    t = make_inputs(2, 16, 24, 9, 11, seed=4)
    leaves = [t[k].clone().requires_grad_(True) for k in ("input", "offset", "mask", "weight", "bias")]
    out = dcn.dcn_v2_conv(*leaves, 1, 1, 1, 1)
    g = t["grad_out"].permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)     # same values, NHWC strides
    assert not g.is_contiguous()
    out.backward(g, retain_graph=True)
    first = [x.grad.clone() for x in leaves]
    want = device(t, "default")
    for name, a, b in zip(NAMES[1:], first, want[1:]):
        if name == "grad_input":
            assert (a - b).abs().max() <= 1e-6 * b.abs().max(), name
        else:
            assert torch.equal(a, b), name
    out.backward(g)
    for name, x, a in zip(NAMES[1:], leaves, first):
        assert torch.allclose(x.grad, 2 * a, rtol=1e-6, atol=1e-6 * a.abs().max().item()), name


def test_reference_state_dict_loads():
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):    # the offset conv in fp32, not TF32
        _state_dict_loads()


def _state_dict_loads():
    C, Co = 40, 24
    sd = {"weight": torch.randn(Co, C, 3, 3), "bias": torch.randn(Co),
          "conv_offset_mask.weight": torch.randn(27, C, 3, 3) * 0.01, "conv_offset_mask.bias": torch.randn(27) * 0.1}
    m = dcn.DCN(C, Co, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
    m.load_state_dict(sd)
    m = m.to(DEV)
    x = torch.randn(2, C, 12, 10, device=DEV)
    got = m(x)
    want = dcn_ref.dcn_module_forward(x.double(), *(sd[k].to(DEV).double() for k in
                                                    ("weight", "bias", "conv_offset_mask.weight",
                                                     "conv_offset_mask.bias")))
    assert (got.double() - want).abs().max().item() <= 1e-5 * want.abs().max().item()


class _RestatedDCN(dcn.DCN):
    """dcn.DCN whose deformable conv is torch autograd through the restatement (run in float64 below)."""

    def forward(self, input):
        o1, o2, mask = torch.chunk(self.conv_offset_mask(input), 3, dim=1)
        return dcn_ref.dcn_v2_forward(input, self.weight, self.bias, torch.cat((o1, o2), 1), torch.sigmoid(mask))


def _stack(cls, ch):
    up = [nn.ConvTranspose2d(ch, ch, 4, stride=2, padding=1, groups=ch, bias=False) for _ in range(2)]
    return nn.Sequential(cls(ch, ch, 3, 1, 1), nn.BatchNorm2d(ch), nn.ReLU(), up[0], up[1], cls(ch, ch, 3, 1, 1))


def test_training_matches_restatement():
    """Five Adam steps of DCN -> BN -> ReLU -> two depthwise 2x up-convs -> DCN at 64 channels on 32x32 maps, with
    dcn.DCN, with the restatement in fp32 and with the restatement in float64, from the same init and batch.  Adam's
    first steps are close to lr * sign(g), so an element whose gradient is near 0 moves by up to a step on any fp32
    rounding; each parameter tensor must therefore agree with float64 within 1e-4 of its largest value, or within
    4 times the fp32 restatement's own difference where that is larger.  cuDNN runs the offset and up-convs in fp32
    rather than its default TF32, so the stacks differ only in the DCN and in fp32 versus float64."""
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        _train_five_steps()


def _train_five_steps():
    torch.manual_seed(0)
    stacks = [_stack(dcn.DCN, 64), _stack(_RestatedDCN, 64), _stack(_RestatedDCN, 64)]
    for m in stacks[1:]:
        m.load_state_dict(stacks[0].state_dict())
    dts = (torch.float32, torch.float32, torch.float64)
    stacks = [m.to(DEV).to(dt) for m, dt in zip(stacks, dts)]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 64, 32, 32, generator=g).to(DEV)
    target = torch.randn(2, 64, 128, 128, generator=g).to(DEV)
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in stacks]
    for _ in range(5):
        for m, opt, dt in zip(stacks, opts, dts):
            opt.zero_grad()
            loss = ((m(x.to(dt)) - target.to(dt)) ** 2).mean()
            loss.backward()
            opt.step()
    mine, fp32, f64 = ([p.detach().double() for p in m.parameters()] for m in stacks)
    names = [n for n, _ in stacks[0].named_parameters()]
    bad = []
    for name, a, b, r in zip(names, mine, fp32, f64):
        scale = r.abs().max().item()
        err, err32 = (a - r).abs().max().item() / scale, (b - r).abs().max().item() / scale
        if err > max(4 * err32, 1e-4):
            bad.append("%s: %.3g > max(4 * %.3g, 1e-4)" % (name, err, err32))
    assert not bad, "\n".join(bad)

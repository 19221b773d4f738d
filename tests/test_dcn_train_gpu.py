"""GPU tests of the training DCNv2 (centerpose_b200.dcn, csrc/dcn_train.cu) against float64 autograd through the
restatement (oracle/dcn_ref.py, oracle/dcn_train_ref.py) on the device, and against tests/golden/dcn_train.npz.

Accuracy: for the output and each of the five gradients, max|dev - f64| / max|f64| and the relative L2 error must be
at most max(4 * e32, 1e-6), where e32 is the same statistic of torch's fp32 autograd through the same restatement.
The restatement runs image-chunk by image-chunk (tests/dcn_train_cases.restated), so the float64 reference fits at the
training batches; e32 sums the same chunks' weight and bias gradients in fp32.
"""
import os

import numpy as np
import pytest
import torch
from torch import nn

from centerpose_b200 import dcn
from oracle import dcn_ref
from tests.dcn_train_cases import (ACCURACY, CFG, DEV, NAMES, PRECISIONS, case_id, check_accuracy, device,
                                   make_inputs, restated)

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dcn_train.npz")


def _accuracy(t, label):
    ref64 = restated(t, torch.float64)
    ref32 = restated(t, torch.float32)
    report = {}
    try:
        for p in PRECISIONS:
            check_accuracy(device(t, p), ref64, ref32, "%s %s" % (label, p), report)
    finally:
        for (lab, name), (e_dev, e32) in report.items():
            print("%s %s: max %.3g (e32 %.3g), l2 %.3g (e32 %.3g)" % (lab, name, e_dev[0], e32[0], e_dev[1], e32[1]))


@pytest.mark.parametrize("case", ACCURACY, ids=case_id)
def test_accuracy(case):
    """Every DCN of DLA-34 and MobileNetV3 at B = 2 and at its training batch, the odd shapes, and a case of one
    weight-gradient split of several K steps (tests/dcn_train_cases.py: every regime of the split rule)."""
    B, C, Co, H, W = case
    seed = C * 7919 + Co * 31 + H + (0 if B == 2 else 104729 * B)
    _accuracy(make_inputs(B, C, Co, H, W, seed=seed), case_id(case))


@pytest.mark.parametrize("stats", ("same_sign", "sparse"))
def test_accuracy_training_statistics(stats):
    """At B = 32, 64 -> 64 on 128x128: post-ReLU inputs, 0.5 px offsets, saturated masks, and a same-sign or sparse
    grad_output (tests/dcn_train_cases.make_inputs)."""
    _accuracy(make_inputs(32, 64, 64, 128, 128, seed=11, stats=stats), "b32_64x64_128x128 " + stats)


@pytest.mark.parametrize("case", ("edges", "pile", "one", "random"))
def test_golden(case):
    z = np.load(GOLD)
    t = {k: torch.from_numpy(z[case + "/" + k]).to(DEV) for k in ("input", "weight", "bias", "offset", "mask",
                                                                 "grad_out")}
    ref64 = [torch.from_numpy(z[case + "/" + n]).to(DEV) for n in NAMES]
    ref32 = restated(t, torch.float32)
    for p in PRECISIONS:
        check_accuracy(device(t, p), ref64, ref32, "%s %s" % (case, p))


TRAINING_SHAPE = (32, 64, 64, 128, 128)      # DLA-34's widest DCN at its training batch: 53 splits of 619 K steps


def _bit_cases(small):
    """(precision, shape) over both precisions at ``small`` (id: the precision) and at TRAINING_SHAPE."""
    return [pytest.param(p, small, id=p) for p in PRECISIONS] + \
        [pytest.param(p, TRAINING_SHAPE, id="%s-%s" % (p, case_id(TRAINING_SHAPE))) for p in PRECISIONS]


@pytest.mark.parametrize("precision,shape", _bit_cases((2, 64, 64, 24, 20)))
def test_scaling_is_exact(precision, shape):
    B, C, Co, H, W = shape
    t = make_inputs(B, C, Co, H, W, seed=5)
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


@pytest.mark.parametrize("precision,shape", _bit_cases((2, 128, 64, 33, 29)))
def test_deterministic(precision, shape):
    B, C, Co, H, W = shape
    t = make_inputs(B, C, Co, H, W, seed=3)
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

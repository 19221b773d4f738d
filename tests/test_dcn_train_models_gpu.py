"""GPU tests of the training DCNv2 (centerpose_b200.dcn) inside the networks it exists for: DLA-34 and MobileNetV3,
whose IDAUp necks are built from DCN, through a training step's loss and backward.

Three arms evaluate the same functions, oracle/dla_ref.dla34_backbone or oracle/mobilenet_ref.mobilenetv3_backbone
(both necks go through dla_ref._ida) and dla_ref.keypoint_head, then oracle/train_loss_ref.loss_torch on a TrainData
batch of seeded JPEG files (INPUT_RES 256, so 64x64 head maps, B = 4):
  (a) fp32 with the device DCN (``dcn.DCN.forward``'s offset conv, chunk / cat / sigmoid, then ``dcn.dcn_v2_conv``),
      in each precision;
  (b) fp32 with the restatement's DCN (the same steps, then oracle/dcn_ref.dcn_v2_forward);
  (c) float64 with the restatement's DCN.
Every arm's DCNs sample at arm (c)'s offsets rounded to fp32 (``dcn_arm``): the bilinear sample's derivative jumps
at integer positions, and without the pin arms (a) and (b) would each take a different side at a different handful of
the some 10^6 samples that lie within fp32's rounding of one, which no kernel error causes.
The weights are the conditioned seed-317 state dict; every floating-point entry is a leaf that requires grad, except
BN's running mean and variance, which batch_norm does not differentiate.  BN uses its running statistics, as the
oracles do: what is under test is the DCN drop-in, not BN's train mode.  cuDNN runs the convs in fp32 rather than its
default TF32, so arms (a) and (b) differ only in the DCN.

Bound: the loss and every parameter tensor's gradient within max(4 * e32, 1e-6) of arm (c), on max|err| / max|ref|
and the relative L2 error, e32 being arm (b)'s own error: the same bound as the op's (tests/test_dcn_train_gpu.py).
Each DCN call of arm (c) is also replayed at op level, under the op bound, so a failure names the layer.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from centerpose_b200 import dcn
from centerpose_b200.config import default_cfg
from centerpose_b200.model import create_model
from oracle import dcn_ref, dla_ref, mobilenet_ref, train_loss_ref
from oracle.init_recipe import conditioned_state_dict
from tests.dcn_train_cases import DEV, NAMES, PRECISIONS, bound_failures, device, restated, stats
from tests.train_cases import seeded_jpeg_batch

pytestmark = pytest.mark.gpu

ARCHS = ("dla_34", "mobilenetv3")
BACKBONE = {"dla_34": dla_ref.dla34_backbone, "mobilenetv3": mobilenet_ref.mobilenetv3_backbone}
# A backbone conv whose output reaches the loss only through one DCN module: the deepest level feeds nothing but the
# first IDAUp's proj DCN (DLA-34: level5, into dla_up.ida_0.proj_1; MobileNetV3: conv2, into ida_up.proj_3).
ONLY_THROUGH_DCN = {"dla_34": "backbone_model.base.level5.tree2.conv2.weight",
                    "mobilenetv3": "backbone_model.conv2.weight"}
NOT_DIFFERENTIATED = (".running_mean", ".running_var")


@contextlib.contextmanager
def _dcn_module_forward(fn):
    """dla_ref._deform (both necks) with ``fn`` in place of dcn_ref.dcn_module_forward."""
    old = dla_ref.dcn_module_forward
    dla_ref.dcn_module_forward = fn
    try:
        yield
    finally:
        dla_ref.dcn_module_forward = old


def dcn_arm(pins, conv, calls=None, names=None):
    """One arm's DCN module forward: ``dcn.DCN.forward``'s offset conv, chunk / cat / sigmoid, then ``conv(input,
    offset, mask, weight, bias)``, with each call's offsets pinned to ``pins``.  Where a sample lies within fp32's
    rounding of an integer row or column, arms whose offsets differ by rounding take different corners, and the
    bilinear sample's derivative jumps there; so every arm takes the float64 arm's offset values rounded to fp32
    (the offset conv's gradient is unchanged), and the fp32 arms then sample at the same positions.  The float64 arm
    (``calls`` given) appends its offsets to ``pins`` and records each call's layer, operands and incoming gradient
    in ``calls``; ``names`` maps id(weight) to the layer."""
    k = [0]

    def fwd(x, weight, bias, om_weight, om_bias):
        o1, o2, m = torch.chunk(F.conv2d(x, om_weight, om_bias, stride=1, padding=1), 3, dim=1)
        offset, mask = torch.cat((o1, o2), dim=1), torch.sigmoid(m)
        if calls is not None:
            pins.append(offset.detach().float())
        offset = pins[k[0]].to(offset.dtype) + (offset - offset.detach())
        k[0] += 1
        out = conv(x, offset, mask, weight, bias)
        if calls is not None:
            rec = dict(layer=names[id(weight)], input=x.detach(), offset=offset.detach(), mask=mask.detach(),
                       weight=weight.detach(), bias=bias.detach())
            out.register_hook(lambda g: rec.__setitem__("grad_out", g.detach()))
            calls.append(rec)
        return out
    return fwd


def device_conv(precision):
    return lambda x, o, m, w, b: dcn.dcn_v2_conv(x, o, m, w, b, 1, 1, 1, 1, precision)


def restated_conv(x, o, m, w, b):
    return dcn_ref.dcn_v2_forward(x, w, b, o, m, 1, 1, 1)


def weights(arch):
    cfg = default_cfg(arch)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    return {k: v for k, v in conditioned_state_dict(m.state_dict(), 317).items() if v.dtype.is_floating_point}


def run_arm(arch, sd, cfg, batch, dtype, conv, pins, calls=None):
    """(loss, {parameter: gradient}) of one arm, its DCNs ``dcn_arm(pins, conv, calls)``."""
    leaves = {k: v.to(DEV, dtype).requires_grad_(not k.endswith(NOT_DIFFERENTIATED)) for k, v in sd.items()}
    b = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
    fwd = dcn_arm(pins, conv, calls, {id(v): k[:-len(".weight")] for k, v in leaves.items()})
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False), _dcn_module_forward(fwd):
        heads = dla_ref.keypoint_head(leaves, BACKBONE[arch](leaves, b["input"]))
        loss, _ = train_loss_ref.loss_torch(heads, b, cfg.LOSS)
        params = [k for k, v in leaves.items() if v.requires_grad]
        grads = torch.autograd.grad(loss, [leaves[k] for k in params], allow_unused=True)
    return loss.detach(), {k: g for k, g in zip(params, grads) if g is not None}


@pytest.fixture(scope="module")
def jpeg_batch(tmp_path_factory):
    return seeded_jpeg_batch(tmp_path_factory.mktemp("dcn_models"), B=4, res=256)


_REFERENCE = {}


@pytest.fixture(scope="module")
def reference(jpeg_batch):
    """Per arch: the weights, arms (b) and (c), arm (c)'s DCN calls and the pinned offsets."""
    cfg, batch = jpeg_batch

    def get(arch):
        if arch not in _REFERENCE:
            sd = weights(arch)
            calls, pins = [], []
            c = run_arm(arch, sd, cfg, batch, torch.float64, restated_conv, pins, calls)
            b = run_arm(arch, sd, cfg, batch, torch.float32, restated_conv, pins)
            _REFERENCE[arch] = (sd, b, c, calls, pins)
        return _REFERENCE[arch]
    yield get
    _REFERENCE.clear()


def group(name):
    """The parameter group the errors are reported by."""
    for suffix, g in ((".conv.conv_offset_mask.weight", "offset conv weight"),
                      (".conv.conv_offset_mask.bias", "offset conv bias"), (".conv.weight", "DCN weight"),
                      (".conv.bias", "DCN bias")):
        if name.endswith(suffix) and (".proj_" in name or ".node_" in name):
            return g
    if name.startswith("head_model."):
        return "head"
    return "neck BN and up-convs" if ".ida_" in name else "backbone"


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("arch", ARCHS)
def test_network_gradients(reference, jpeg_batch, arch, precision):
    sd, (loss_b, grad_b), (loss_c, grad_c), _, pins = reference(arch)
    cfg, batch = jpeg_batch
    loss_a, grad_a = run_arm(arch, sd, cfg, batch, torch.float32, device_conv(precision), pins)
    # coverage: every DCN weight and bias, every offset conv, and a backbone conv behind a DCN have a gradient
    dcns = [k[:-len(".conv_offset_mask.weight")] for k in sd if k.endswith(".conv_offset_mask.weight")]
    assert len(dcns) == {"dla_34": 16, "mobilenetv3": 6}[arch]
    need = [p + s for p in dcns for s in (".weight", ".bias", ".conv_offset_mask.weight", ".conv_offset_mask.bias")]
    need.append(ONLY_THROUGH_DCN[arch])
    missing = [k for k in need if k not in grad_c or not grad_c[k].any()]
    assert not missing, missing
    assert set(grad_a) == set(grad_b) == set(grad_c)
    bad = bound_failures("loss", loss_a, loss_c, loss_b)
    worst = {}
    for k, r in grad_c.items():
        assert torch.isfinite(grad_a[k]).all(), k
        bad += bound_failures(k, grad_a[k], r, grad_b[k])
        e_dev, e32 = stats(grad_a[k], r), stats(grad_b[k], r)
        w = worst.setdefault(group(k), [0.0, 0.0, 0.0, 0.0])
        w[:] = [max(w[0], e_dev[0]), max(w[1], e32[0]), max(w[2], e_dev[1]), max(w[3], e32[1])]
    print("%s %s loss: %s (e32 %s)" % (arch, precision, stats(loss_a, loss_c), stats(loss_b, loss_c)))
    for g, w in sorted(worst.items()):
        print("%s %s %s: worst max %.3g (e32 %.3g), worst l2 %.3g (e32 %.3g)" % (arch, precision, g, *w))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("arch", ARCHS)
def test_replay_dcn_calls(reference, arch):
    """Each DCN call of the float64 arm, its operands rounded to fp32, through dcn_v2_forward / dcn_v2_backward in
    both precisions against the float64 restatement, under the op bound."""
    _, _, _, calls, _ = reference(arch)
    assert len(calls) == {"dla_34": 16, "mobilenetv3": 6}[arch] and all("grad_out" in c for c in calls)
    bad = []
    for c in calls:
        t = {k: c[k].float() for k in ("input", "weight", "bias", "offset", "mask", "grad_out")}
        ref64, ref32 = restated(t, torch.float64), restated(t, torch.float32)
        for p in PRECISIONS:
            for name, g, r, r32 in zip(NAMES, device(t, p), ref64, ref32):
                assert torch.isfinite(g).all(), (c["layer"], p, name)
                bad += bound_failures("%s %s %s" % (c["layer"], p, name), g, r, r32)
    assert not bad, "\n".join(bad)

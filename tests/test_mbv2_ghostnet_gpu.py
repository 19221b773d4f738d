"""GPU tests of the device work the MobileNetV2 and GhostNet backbones (centerpose_b200/archs/mobilenetv2.py,
archs/ghostnet.py) added: the ReLU6 / clip01 epilogue activations (CPB200_FLAG_RELU6 / CPB200_FLAG_CLIP01), the bias
form of CPB200_OP_DWDECONV_ADD (k 2 / stride 2 deconv + folded BN + ReLU + skip) and the 4x bilinear upscale.  The
network-level checks of both backbones are in tests/test_backbones_gpu.py.

Tolerances:
  ops, "int" data : exact, element by element (tests/replay.py: integers that every format holds exactly)
  ops, randn data : tests/util.py::check_op
"""
import pytest
import torch
import torch.nn.functional as F

from tests.kernel_routes import CASES
from tests.layer_census import Record
from tests.replay import _data, _reference, _replay
from tests.util import builder, check_op, external, run_op

pytestmark = pytest.mark.gpu
PRECS = ["fp32", "bf16", "bf16x2", "fp16x2"]


def _precision(p):
    return ("bf16", False) if p == "bf16-simt" else (p, None)


def _launched(plan, stream, names):
    import ctypes
    from centerpose_b200 import _lib
    from tests.kernel_routes import kernel_key
    L = _lib.lib()
    L.cpb200_route_log_start()
    try:
        plan.run(stream)
        torch.cuda.synchronize()
    finally:
        buf = ctypes.create_string_buffer(1 << 16)
        n = L.cpb200_route_log_read(buf, len(buf))
        assert n >= 0
        names.update(kernel_key(k) for k in buf.value.decode().splitlines() if k)


def _with_act(rec, act):
    return Record(rec.method, tuple((k, act if k == "act" else (False if k == "relu" else v)) for k, v in rec.args), ())


# ------------------------------------------------------------------------------------------- epilogue activations
_ACT_CASES = [(i, p, act) for act in ("relu6", "clip01") for i, c in enumerate(CASES)
              if c.rec.method in (("conv", "stem", "dwconv") if act == "relu6" else ("conv",)) and not c.error
              for p in c.precisions()]


@pytest.mark.parametrize("idx,pkey,act", _ACT_CASES, ids=[f"{i}-{p}-{CASES[i].rec.method}-{a}" for i, p, a in _ACT_CASES])
def test_clamp_activation_on_every_route(idx, pkey, act, monkeypatch):
    """ReLU6 on every conv, stem and depthwise route of tests/kernel_routes.py, clip01 on every conv route: integer
    data whose results straddle 0, 1 and 6, so the clamp must be exact in every format (the split epilogues clamp
    before the hi / lo re-split).  The program launches the kernels the route table declares for the case."""
    case = CASES[idx]
    precision, tc = _precision(pkey)
    rec = _with_act(case.rec, act)
    data = _data(rec, "int", case.B)
    names = set()
    with monkeypatch.context() as mp:
        mp.setenv("CPB200_RZ_COMP", "0")
        got, problems = _replay(rec, precision, data, B=case.B, tc=tc, run=lambda plan, st: _launched(plan, st, names))
    assert names == set(case.routes_for(pkey)), (sorted(names), sorted(case.routes_for(pkey)))
    top = 6 if act == "relu6" else 1
    lin = _reference(_with_act(case.rec, None), data)
    assert (lin <= 0).any() and (lin >= top).any() and (act == "clip01" or ((lin > 0) & (lin < top)).any())
    ref = lin.clamp(0, top)
    assert not problems, problems
    diff = (got - ref).abs()
    assert bool((diff == 0).all()), f"{case.label()} {pkey} {act}: {int((diff != 0).sum())} elements differ"


# ------------------------------------------------------------------------------------------- element-wise ops
def _rnd(t, precision):
    return t.bfloat16().float() if precision == "bf16" else t


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("C", [24, 32, 64])
def test_dwdeconv_bias_form_matches_torch(precision, C):
    """relu(conv_transpose2d(x, w, stride 2, groups C) + b) (+ skip): MobileNetV2's IDAUp step, one DWDECONV_ADD op
    natively in every format.  Integer data must come out exact; randn data within the precision's bound."""
    from centerpose_b200.plan import OP_DWDECONV_ADD
    B = 2
    for i, (H, W, skip_on) in enumerate([(3, 5, True), (16, 16, True), (12, 20, False), (1, 1, True)]):
        g = torch.Generator().manual_seed(100 * C + i)
        for leg in ("int", "randn"):
            if leg == "int":
                x = torch.randint(-2, 3, (B, C, H, W), generator=g).float()
                w = torch.randint(-2, 3, (C, 1, 2, 2), generator=g).float()
                b = torch.randint(-3, 4, (C,), generator=g).float()
                skip = torch.randint(-3, 4, (B, C, 2 * H, 2 * W), generator=g).float()
            else:
                x = _rnd(torch.randn(B, C, H, W, generator=g) * 2, precision)
                w = torch.randn(C, 1, 2, 2, generator=g)
                b = torch.randn(C, generator=g)
                skip = _rnd(torch.randn(B, C, 2 * H, 2 * W, generator=g), precision)
            pb = builder(B, precision)
            y = pb.up_add(external(pb, x, precision), external(pb, skip, precision) if skip_on else None, w, b=b,
                          act="relu", stride=2, pad=0)
            assert [o.type for o in pb.ops] == [OP_DWDECONV_ADD] and (y.H, y.W) == (2 * H, 2 * W)
            ref = F.relu(F.conv_transpose2d(x.double(), w.double(), b.double(), stride=2, groups=C))
            if skip_on:
                ref = ref + skip.double()
            got = run_op(pb, y)
            if leg == "int":
                assert torch.equal(got, ref), (precision, C, H, W)
            else:
                check_op(got, ref, precision, what=(C, H, W))


def test_dwdeconv_activation_needs_bias():
    """An activation flag on the bias-less form is rejected (CPB200_ERR_ARG) before anything is launched."""
    pb = builder(1, "fp32")
    x = torch.randn(1, 16, 4, 4)
    pb.up_add(external(pb, x, "fp32"), None, torch.randn(16, 1, 4, 4))
    plan = pb.build()
    plan.ops[0].flags = 1
    with pytest.raises(RuntimeError, match="bias form"):
        plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


@pytest.mark.parametrize("precision", PRECS)
def test_se_clip01_gate_matches_torch(precision):
    """GhostNet's SE: x * clamp(fc2(relu(fc1(avgpool(x)))), 0, 1) with the FCs as 1x1 convs on the 1x1 map and the
    clamp as the second conv's clip01 epilogue; the biases push about half the gates outside [0, 1]."""
    B, C, H, W, mid = 3, 48, 9, 13, 16
    g = torch.Generator().manual_seed(7)
    x = _rnd(torch.randn(B, C, H, W, generator=g) * 2, precision)
    w1 = torch.randn(mid, C, 1, 1, generator=g) / C ** 0.5
    b1 = torch.randn(mid, generator=g) * 0.1
    w2 = torch.randn(C, mid, 1, 1, generator=g) / mid ** 0.5
    b2 = torch.randn(C, generator=g) + 0.5
    pb = builder(B, precision)
    xs = external(pb, x, precision)
    h = pb.conv([pb.avgpool(xs)], w1, b1, act="relu")
    gate = pb.conv([h], w2, b2, act="clip01")
    y = pb.scale_add(xs, gate)
    s = F.relu(F.conv2d(x.double().mean(dim=(2, 3), keepdim=True), w1.double(), b1.double()))
    gd = F.conv2d(s, w2.double(), b2.double())
    assert (gd < 0).any() and (gd > 1).any()
    ref = x.double() * gd.clamp(0, 1)
    check_op(run_op(pb, y), ref, precision, what="se")


@pytest.mark.parametrize("precision", PRECS)
def test_resize_bilinear_4x_upscale(precision):
    """GhostNet's fixed 128 x 128 resize: 2x (512 input), 4x (256 input) and a non-square 4x / 3.2x, in every format."""
    B, C = 1, 80
    for i, (H, W) in enumerate([(64, 64), (32, 32), (32, 40)]):
        x = _rnd(torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(i)) * 3, precision)
        pb = builder(B, precision)
        y = pb.resize_bilinear(external(pb, x, precision), 128, 128)
        ref = F.interpolate(x.double(), size=(128, 128), mode="bilinear", align_corners=True)
        check_op(run_op(pb, y), ref, precision, what=(H, W))

"""The fused keypoint-head op (OP_HEADS, csrc/net_heads.cu) against the 3x3 + 1x1 conv pairs it replaces.  Both sum
the same products in the same order, so the head maps must be bit-identical."""
import pytest
import torch

from centerpose_b200 import plan as plan_mod
from centerpose_b200.synth import synth_images
from tests.util import model

DEV = torch.device("cuda:0")
_MODELS = {}


def _cached_model(arch):
    if arch not in _MODELS:
        _MODELS[arch] = model(arch, "fp32")[0]
    return _MODELS[arch]


def _forward(m, xs, precision, fused, monkeypatch):
    """the head maps of each input in turn (fresh output tensors per forward, i.e. re-bound outputs)"""
    with monkeypatch.context() as mp:
        if not fused:
            mp.setattr(plan_mod.Plan, "_fuse_heads", lambda self, pb: None)
        m.set_precision(precision)
        outs = [m(x) for x in xs]
        plan = m._plan(xs[0].shape[0], xs[0].shape[2], xs[0].shape[3], DEV)
        assert any(o.type == plan_mod.OP_HEADS for o in plan.pb.ops) == fused
        torch.cuda.synchronize()
        m.invalidate()
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16x2", "bf16x2", "bf16"])
@pytest.mark.parametrize("B,H,W", [(1, 512, 512), (3, 512, 512), (1, 96, 160), (3, 96, 160)])
def test_fused_heads_bit_identical(precision, B, H, W, monkeypatch):
    m = _cached_model("dla_34")
    xs = [synth_images(B, H, W, 317 + k).to(DEV) for k in range(2)]
    got = _forward(m, xs, precision, True, monkeypatch)
    want = _forward(m, xs, precision, False, monkeypatch)
    for k in range(2):
        for g, w in zip(got[k], want[k]):
            assert torch.equal(g, w), (k, (g - w).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16x2", "bf16"])
def test_fused_heads_bit_identical_mobilenetv3(precision, monkeypatch):
    """32-channel head input: 32-wide K slab with the 64-byte swizzle"""
    m = _cached_model("mobilenetv3")
    xs = [synth_images(2, 96, 160, 317).to(DEV)]
    got = _forward(m, xs, precision, True, monkeypatch)
    want = _forward(m, xs, precision, False, monkeypatch)
    for g, w in zip(got[0], want[0]):
        assert torch.equal(g, w), (g - w).abs().max().item()

"""Plan-level fusion of the keypoint heads (Plan._fuse_heads -> OP_HEADS): which programs take it and which stay as they
were.  Plans are built on the host (no kernel runs)."""
import pytest
import torch

from centerpose_b200 import plan as plan_mod
from centerpose_b200.config import default_cfg
from centerpose_b200.model import HEADS, create_model

CPU = torch.device("cpu")


def _programs(arch, precision, monkeypatch):
    cfg = default_cfg(arch)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).set_precision(precision)
    fused = m._plan(1, 128, 128, CPU)
    with monkeypatch.context() as mp:
        mp.setattr(plan_mod.Plan, "_fuse_heads", lambda self, pb: None)
        m.invalidate()
        plain = m._plan(1, 128, 128, CPU)
    return fused, plain


def _ops(plan):
    return [(o.type, o.flags, o.act_dtype, o.cout, o.kh, o.kw, o.Ho, o.Wo) for o in plan.ops]


@pytest.mark.parametrize("arch", ["dla_34", "mobilenetv3"])
@pytest.mark.parametrize("precision", ["bf16", "bf16x2", "fp16x2"])
def test_heads_become_one_op(arch, precision, monkeypatch):
    fused, plain = _programs(arch, precision, monkeypatch)
    assert plain.n == fused.n + 11
    assert _ops(fused)[:-1] == _ops(plain)[:-12]
    tail = plain.ops[plain.n - 12:]
    assert [o.kh for o in tail] == [3, 1] * 6 and all(tail[k].flags & plan_mod.FLAG_OUT_NCHW_F32 for k in range(1, 12, 2))
    o = fused.ops[fused.n - 1]
    assert o.type == plan_mod.OP_HEADS and o.flags & plan_mod.FLAG_TC and o.aux_pitch == len(HEADS)
    assert o.cout == sum(c for _, c in HEADS) and o.cin[0] == tail[0].cin[0]
    tab = fused._head_tables[fused.n - 1]
    assert [(e.hidden, e.cout) for e in tab] == [(256, c) for _, c in HEADS]
    assert [e.acc_scale3 for e in tab] == pytest.approx([tail[k].acc_scale for k in range(0, 12, 2)], rel=0, abs=0)
    assert [e.acc_scale1 for e in tab] == pytest.approx([tail[k].acc_scale for k in range(1, 12, 2)], rel=0, abs=0)
    # no op of the fused program writes a hidden map
    assert not any(po.type == plan_mod.OP_CONV and po.dst.C == 256 and po.dst.H == 32 for po in fused.pb.ops)


@pytest.mark.parametrize("arch,precision", [("dla_34", "fp32"), ("mobilenetv3", "fp32")] +
                         [(a, p) for a in ("res_50", "hrnet", "hardnet") for p in ("fp32", "bf16", "bf16x2", "fp16x2")])
def test_other_programs_unchanged(arch, precision, monkeypatch):
    fused, plain = _programs(arch, precision, monkeypatch)
    assert _ops(fused) == _ops(plain)
    assert not any(o.type == plan_mod.OP_HEADS for o in fused.ops)


def test_outputs_rebind_through_the_table(monkeypatch):
    fused, _ = _programs("dla_34", "fp16x2", monkeypatch)
    outs = {name: torch.empty(1, c, 32, 32) for name, c in HEADS}
    fused.bind(torch.zeros(1), outs)
    tab = fused._head_tables[fused.n - 1]
    assert [e.dst for e in tab] == [outs[name].data_ptr() for name, _ in HEADS]

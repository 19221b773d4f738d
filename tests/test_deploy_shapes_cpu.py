"""The eight network configurations lowered on the host at the input shapes the detector builds at deployment
(tests/util.py: DEPLOY_SHAPES, B = 1), checked before anything is launched:

  * every op of every program has positive extents, and reads only activations whose buffer still holds them (the
    liveness-based buffer reuse at odd extents: no later op has written the buffer in between, and it is large enough);
  * the inputs the reference cannot run (TOO_SMALL) are refused with a Python error when the plan is built, and the
    float64 oracle raises on them too;
  * the routes the table reaches that the golden sizes (the inputs of tests/golden/<arch>_*.npz) do not: each op as
    (type, tensor-core / fp32-island, class of Ho, class of Wo), the classes 1, 2-7, 8-15 and 16 or more (the
    tensor-core tiles take 8 output columns or more; fewer go to an fp32 island).  They are printed per row, and the
    table must keep reaching the regimes of NEW_ROUTES.

The GPU side of the same table is tests/test_backbones_gpu.py::test_forward_matches_oracle.
"""
import pytest
import torch

from tests.util import ARCHS, DEPLOY_SHAPES, TOO_SMALL, config

PRECISIONS = ["fp32", "bf16", "bf16x2", "fp16x2"]
CPU = torch.device("cpu")
# (B, H, W) of each configuration's golden inputs (HRNet-W48: W32's)
GOLDEN_INPUTS = {"dla_34": [(1, 128, 128), (2, 96, 160), (1, 512, 512)], "res_50": [(2, 128, 128), (1, 512, 512)],
                 "hrnet": [(2, 128, 128), (1, 256, 320), (1, 512, 512)],
                 "hrnet_w48": [(2, 128, 128), (1, 256, 320), (1, 512, 512)],
                 "mobilenetv3": [(2, 128, 160), (1, 512, 512)],
                 "hardnet": [(2, 128, 128), (2, 96, 160), (1, 512, 512)],
                 "mobilenetv2": [(1, 512, 512), (2, 96, 160)], "ghostnet": [(1, 512, 512)]}
# regimes only the deployment shapes reach, in fp16x2 (the default precision)
NEW_ROUTES = {
    "conv/tc 2-7x16+": "tensor-core conv tiles with fewer than 8 output rows and 8 or more columns (Ho < 8 <= Wo)",
    "conv/tc 1x16+": "tensor-core conv on a map one pixel high",
    "conv/f32 16+x2-7": "fp32-island conv on a tall map fewer than 8 pixels wide (Wo < 8 <= Ho)",
    "conv/f32 16+x1": "fp32-island conv on a map one pixel wide",
    "convert 16+x2-7": "CONVERT ops into and out of those islands",
    "dcn/tc 2-7x16+": "tensor-core DCN with fewer than 8 rows",
    "dcn/f32 16+x2-7": "CUDA-core DCN between tensor-core ones (MobileNetV3 / DLA-34 at 640x224)",
    "heads/tc 8-15x16+": "the fused heads on an 8 x N map",
    "upsample_add 2-7x16+": "HRNet's nearest upsample-add into a map fewer than 8 rows high",
    "dwdeconv_add 16+x2-7": "IDAUp's depthwise deconv-add into a map fewer than 8 wide",
    "resize_bilinear 2-7x16+": "HarDNet's align-corners resize into a map fewer than 8 rows high",
    "scale_add 2-7x16+": "the SE scale-add on a map fewer than 8 rows high",
}


def _cls(n):
    return "1" if n == 1 else "2-7" if n < 8 else "8-15" if n < 16 else "16+"


def _lower(m, B, H, W):
    m.invalidate()
    return m._plan(B, H, W, CPU)


def _routes(plan):
    from centerpose_b200 import plan as P
    names = {v: k[3:].lower() for k, v in vars(P).items() if k.startswith("OP_") and isinstance(v, int)}
    out = set()
    for o in plan.pb.ops:
        kind = names[o.type]
        if o.flags & P.FLAG_TC:
            kind += "/tc"
        elif plan.pb.split and o.dtype == P.F32:
            kind += "/f32"
        out.add(f"{kind} {_cls(o.HoWo[0])}x{_cls(o.HoWo[1])}")
    return out


def _check_program(plan, what):
    """positive extents; every operand still in its buffer when read"""
    pb = plan.pb
    owner = {}                                       # id(buffer) -> the root Sym last written into it
    for i, po in enumerate(pb.ops):
        for s in (*po.operands(), po.dst):
            assert min(s.C, s.H, s.W) > 0, (what, i, po.type, s.C, s.H, s.W)
        assert min(po.HoWo) > 0 and po.cout > 0, (what, i, po.type, po.HoWo, po.cout)
        for s in po.operands():
            r = plan._root(s)
            if r.fixed:
                continue
            assert owner.get(id(r.buf)) is r, f"{what}: op {i} (type {po.type}) reads a buffer a later op overwrote"
            assert r.buf.numel() >= pb.B * r.H * r.W * r.C * pb._storage(r.kind)[0], (what, i)
        d = plan._root(po.dst)
        if not d.fixed:
            assert d.buf.numel() >= pb.B * d.H * d.W * d.C * pb._storage(d.kind)[0], (what, i)
            owner[id(d.buf)] = d


def _model(arch, precision):
    from centerpose_b200.model import create_model
    cfg = config(arch)
    torch.manual_seed(0)
    return create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).set_precision(precision)


@pytest.mark.parametrize("arch", ARCHS)
def test_deploy_shapes_lower_with_positive_extents(arch):
    for precision in PRECISIONS:
        m = _model(arch, precision)
        for H, W in DEPLOY_SHAPES:
            if (arch, H, W) in TOO_SMALL:
                with pytest.raises(ValueError, match="too small"):
                    _lower(m, 1, H, W)
                continue
            _check_program(_lower(m, 1, H, W), (arch, precision, H, W))


def test_too_small_inputs_are_refused_by_the_oracle():
    """the reason of every TOO_SMALL entry: the float64 oracle (as the reference) raises at that input"""
    from oracle import hardnet_ref
    from oracle.init_recipe import conditioned_state_dict, synth_images
    from centerpose_b200.model import create_model
    assert {a for a, _, _ in TOO_SMALL} == {"hardnet"}
    cfg = config("hardnet")
    sd = conditioned_state_dict(create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).state_dict(), 317)
    for _, H, W in TOO_SMALL:
        with pytest.raises(RuntimeError, match="too small"):
            hardnet_ref.forward(sd, synth_images(1, H, W, 317).double())


def test_deploy_shapes_reach_routes_the_goldens_do_not():
    new_all = set()
    for arch in ARCHS:
        m = _model(arch, "fp16x2")
        golden = set()
        for B, H, W in GOLDEN_INPUTS[arch]:
            golden |= _routes(_lower(m, B, H, W))
        for H, W in DEPLOY_SHAPES:
            if (arch, H, W) in TOO_SMALL:
                continue
            new = _routes(_lower(m, 1, H, W)) - golden
            print(f"{arch} {H}x{W}: {sorted(new)}")
            new_all |= new
    missing = sorted(set(NEW_ROUTES) - new_all)
    assert not missing, missing

"""GPU tests of HarDNet's two element-wise ops, CPB200_OP_AVGPOOL2 and CPB200_OP_RESIZE_BILINEAR, against a float64
torch evaluation in every format (bounds: tests/util.py::check_op; inputs already bf16-representable in bf16).  The
network-level checks of HarDNet (centerpose_b200/archs/hardnet.py) are in tests/test_backbones_gpu.py.
"""
import pytest
import torch
import torch.nn.functional as F

from tests.util import builder, check_op, external, run_op

pytestmark = pytest.mark.gpu
PRECS = ["fp32", "bf16", "bf16x2", "fp16x2"]

POOL_IN = [(13, 18), (3, 5), (6, 10), (16, 16), (24, 40), (12, 20), (2, 2)]
RESIZE = [((13, 18), (6, 9)), ((1, 2), (3, 5)), ((3, 5), (6, 10)), ((8, 8), (16, 16)), ((12, 20), (24, 40)),
          ((12, 20), (12, 20)), ((2, 3), (1, 1))]


def _input(B, C, H, W, seed, precision):
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(seed)) * 3
    return x.bfloat16().float() if precision == "bf16" else x


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("C", [16, 48, 320])
def test_avgpool2_op_matches_torch(precision, C):
    """2x2 / stride-2 average pool, floor mode (odd sizes drop the last row / column), natively in every dtype: the
    program is the one op, with no CONVERT around it in the split precisions."""
    from centerpose_b200.plan import OP_AVGPOOL2
    B = 2
    for i, (H, W) in enumerate(POOL_IN):
        x = _input(B, C, H, W, 100 * C + i, precision)
        pb = builder(B, precision)
        y = pb.avgpool2(external(pb, x, precision))
        assert [o.type for o in pb.ops] == [OP_AVGPOOL2] and (y.H, y.W) == (H // 2, W // 2)
        check_op(run_op(pb, y), F.avg_pool2d(x.double(), 2, 2), precision, what=(H, W))


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("C", [16, 48, 320])
def test_resize_bilinear_op_matches_torch(precision, C):
    """bilinear resize, align_corners=True, to arbitrary sizes (up, down, same size, from a 1-pixel-high map, to 1x1)."""
    from centerpose_b200.plan import OP_RESIZE_BILINEAR
    B = 2
    for i, ((H, W), (Ho, Wo)) in enumerate(RESIZE):
        x = _input(B, C, H, W, 200 * C + i, precision)
        pb = builder(B, precision)
        y = pb.resize_bilinear(external(pb, x, precision), Ho, Wo)
        assert [o.type for o in pb.ops] == [OP_RESIZE_BILINEAR]
        ref = F.interpolate(x.double(), size=(Ho, Wo), mode="bilinear", align_corners=True)
        check_op(run_op(pb, y), ref, precision, what=((H, W), (Ho, Wo)))
    if precision == "fp32":                 # fp32: PyTorch's own fp32 arithmetic, to within a couple of ulps
        x = _input(B, C, 12, 20, 7, precision)
        pb = builder(B, precision)
        y = pb.resize_bilinear(external(pb, x, precision), 24, 40)
        ref = F.interpolate(x, size=(24, 40), mode="bilinear", align_corners=True).double()
        assert (run_op(pb, y) - ref).abs().max().item() <= 4 * 2.0 ** -23 * ref.abs().max().item()


def _expect_error(pb, edit, match):
    plan = pb.build()
    edit(plan.ops[0])
    with pytest.raises(RuntimeError, match=match):
        plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_avgpool2_and_resize_reject_unsupported_shapes(precision):
    """Shapes the kernels do not handle return CPB200_ERR_ARG with a message before anything is launched."""
    B, C = 2, 16
    x = _input(B, C, 5, 6, 1, precision)

    def pool():
        pb = builder(B, precision)
        pb.avgpool2(external(pb, x, precision))
        return pb

    def resize():
        pb = builder(B, precision)
        pb.resize_bilinear(external(pb, x, precision), 9, 11)
        return pb

    def second_input(o):
        o.nsrc = 2; o.src[1] = o.src[0]; o.cin[1] = o.cin[0]

    def set_(**kw):
        def f(o):
            for k, v in kw.items():
                setattr(o, k, v)
        return f

    def pitch(o):
        o.src_pitch[0] = 2 * C

    _expect_error(pool(), set_(H=1, Ho=0), "bad shape")                   # H < 2 (floor mode gives an empty output)
    _expect_error(pool(), set_(W=1), "avgpool2")                          # W < 2
    _expect_error(pool(), set_(Ho=3), "avgpool2")                         # Ho != H/2
    _expect_error(pool(), set_(Wo=2), "avgpool2")                         # Wo != W/2
    _expect_error(pool(), second_input, "avgpool2")                       # nsrc != 1
    _expect_error(pool(), pitch, "channel-slice")                         # a src_pitch slice
    _expect_error(resize(), set_(Ho=0), "bad shape")                      # Ho < 1
    _expect_error(resize(), set_(Wo=-1), "bad shape")                     # Wo < 1
    _expect_error(resize(), second_input, "resize_bilinear")
    _expect_error(resize(), pitch, "channel-slice")

"""GPU tests of max-pool's 2x2 / stride 2 form (csrc/net_eltwise.cu: pool2_fast) at both sides of each of its shape
conditions, in all four activation formats.  Max-pooling is exact in every format: the result equals torch's max_pool2d
of the values the format holds (bf16-rounded inputs for bf16, hi + lo of the planes for the split precisions)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

CASES = [
    # C, H, W, B, form
    (8, 6, 10, 2, "2x2 form: C = 8, the smallest channel count"),
    (72, 4, 60, 1, "2x2 form: C / VEC not a power of two, an output row of more than 256 items"),
    (64, 32, 32, 3, "2x2 form: a DLA-34 shape"),
    (4, 6, 10, 2, "generic form: C = 4"),
    (12, 6, 10, 1, "generic form: C % 8 != 0"),
    (8, 7, 10, 1, "generic form: odd H"),
    (16, 6, 11, 2, "generic form: odd W"),
]


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x2", "fp16x2"])
@pytest.mark.parametrize("C,H,W,B,form", CASES, ids=[c[4] for c in CASES])
def test_maxpool_2x2_is_exact_in_both_forms(precision, C, H, W, B, form):
    from centerpose_b200.plan import OP_MAXPOOL, PlanBuilder, split_planes
    g = torch.Generator().manual_seed(C * 1000 + H * 10 + W)
    t = torch.randn(B, C, H, W, generator=g) * 3
    pb = PlanBuilder(B, 1, 1, precision, torch.device(DEV), tc=None if precision != "bf16" else False)
    if precision in ("bf16x2", "fp16x2"):
        held = split_planes(t, pb.torch16).float().sum(0)
        x = pb.external(t.permute(0, 2, 3, 1).contiguous().to(DEV))
    else:
        dt = torch.float32 if precision == "fp32" else torch.bfloat16
        held = t.to(dt).float()
        x = pb.external(t.permute(0, 2, 3, 1).contiguous().to(DEV, dt))
    y = pb.maxpool(x, 2, 2, 0)
    assert [o.type for o in pb.ops] == [OP_MAXPOOL], "the pool runs on the format's own planes, without an fp32 island"
    plan = pb.build()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = plan.tensor(y).float().permute(0, 3, 1, 2).cpu()
    assert torch.equal(got, F.max_pool2d(held, 2, 2, 0)), form

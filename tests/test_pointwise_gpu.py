"""Pointwise convs (1x1 / stride 1 / pad 0, NHWC output, cout % 16 == 0) on the tap-per-stage kernel's 1 x 128 pixel
tiles with the 16-byte epilogue, against the same ops on 2-D tiles (CPB200_NO_PW=1), bit for bit.

The two layouts issue the same products in the same order and finish them with the same epilogue arithmetic, so the
stored outputs must be equal element for element, on integer-exact data and on randn data, in bf16, bf16x2 and fp16x2.
The cases are the route table's pointwise convs (tests/kernel_routes.py) and the edges below: three and four inputs
with a channel slice and a residual, cout 512, fp32 output, pixel counts that leave a partial last tile."""
import pytest
import torch

from tests.kernel_routes import CASES, Case, record, sym, tcr, tensor
from tests.replay import _data, _replay

pytestmark = pytest.mark.gpu


def _pointwise(c):
    kw = dict(c.rec.args)
    w = kw.get("w")
    return (c.rec.method == "conv" and not c.error and w[1][2:] == (1, 1) and kw["stride"] == 1 and kw["out"] != "nchw"
            and w[1][0] % 16 == 0 and "bf16" in c.routes)


def _conv(srcs, cout, routes, reason, B=1, res=False, relu=False, out="act"):
    cin = sum(s[1] for s in srcs)
    H, W = srcs[0][2], srcs[0][3]
    rec = record("conv", srcs=tuple(srcs), w=tensor(cout, cin, 1, 1), b=tensor(cout), stride=1, pad=0, relu=relu,
                 res=sym(cout, H, W) if res else None, out=out)
    return Case(rec, {k: frozenset(v) for k, v in routes.items()}, reason, B)


EDGES = [
    _conv([sym(64, 9, 11)], 32, tcr(32, 32), "NHWC fp32 output, cout 32", out="f32"),
    _conv([sym(64, 9, 9)], 512, tcr(256, 128), "cout 512: 2 (bf16) / 4 (split) N tiles, residual", res=True),
    _conv([sym(16, 9, 13), sym(64, 9, 13), sym(32, 9, 13)], 48, tcr(64, 64), "three inputs (bk 16), 351 pixels", B=3),
    _conv([sym(64, 8, 9), sym(64, 8, 9, pc=192, off=128), sym(32, 8, 9), sym(128, 8, 9)], 128, tcr(128, 128),
          "four inputs, a channel slice at offset 128 of 192, residual + relu", res=True, relu=True),
    _conv([sym(256, 5, 14)], 16, tcr(16, 16), "cin 256 (four K slabs), 70 pixels"),
]
PW_CASES = [c for c in CASES if _pointwise(c)] + EDGES


def test_cases_exist():
    assert len(PW_CASES) >= 15


@pytest.mark.parametrize("precision", ["bf16", "bf16x2", "fp16x2"])
@pytest.mark.parametrize("case", PW_CASES, ids=[c.rec.label() for c in PW_CASES])
def test_pointwise_tiles_equal_2d_tiles(case, precision, monkeypatch):
    legs = (["int"] if case.exact else []) + ["bf16" if precision == "bf16" else "f32"]
    for leg in legs:
        data = _data(case.rec, leg, case.B)
        got = {}
        for layout in ("2d", "pw"):
            with monkeypatch.context() as mp:
                if leg == "int":
                    mp.setenv("CPB200_RZ_COMP", "0")
                if layout == "2d":
                    mp.setenv("CPB200_NO_PW", "1")
                else:
                    mp.delenv("CPB200_NO_PW", raising=False)
                got[layout], problems = _replay(case.rec, precision, data, B=case.B)
            assert not problems, (layout, leg, problems)
        a, b = got["2d"], got["pw"]
        assert a.shape == b.shape
        diff = int((a.view(torch.int64) != b.view(torch.int64)).sum())
        assert diff == 0, f"{case.label()} {precision} [{leg}]: {diff} elements differ between the tile layouts"


@pytest.mark.parametrize("precision", ["bf16", "fp16x2"])
def test_pointwise_refuses_unaligned_output(precision, monkeypatch):
    """The 16-byte epilogue needs a 16-byte aligned dst: an 8-byte offset is refused before the launch, and the same op on
    2-D tiles (4-byte stores) runs.  Also shows that the pointwise layout is the one prepared for such an op."""
    from centerpose_b200.plan import PlanBuilder
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    adt = torch.bfloat16 if precision == "bf16" else torch.float32
    raw = torch.empty(1 << 20, dtype=torch.uint8, device=dev)
    for layout in ("2d", "pw"):
        with monkeypatch.context() as mp:
            if layout == "2d":
                mp.setenv("CPB200_NO_PW", "1")
            else:
                mp.delenv("CPB200_NO_PW", raising=False)
            pb = PlanBuilder(1, 8, 16, precision, dev, tc=True)
            x = pb.external(torch.randn(1, 8, 16, 64, generator=g).to(dev, adt))
            pb.conv([x], torch.randn(32, 64, 1, 1, generator=g).to(dev), torch.zeros(32, device=dev), stride=1, pad=0)
            plan = pb.build()
            plan.ops[plan.n - 1].dst = raw.data_ptr() + 8
            stream = torch.cuda.current_stream().cuda_stream
            if layout == "pw":
                with pytest.raises(RuntimeError, match="16-byte aligned"):
                    plan.run(stream)
            else:
                plan.run(stream)
                torch.cuda.synchronize()
